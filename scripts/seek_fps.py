#!/usr/bin/env python3
"""VideoReader seek cost on a 4K YUV444 file of 60 frames, keyframe_interval=30 (two GOPs), for both entropy coders: milliseconds
and d2h_bytes of read(i, i + 1) at GOP positions 0, 1, 15 and 29 (frames 30 + i: the second GOP, whose keyframe is frame 30), of
read(0, 60) and of the whole decompress_video, and of read(i, i + 1, out=<torch CUDA tensor>).  Each time is the median of `--runs`
host-clock runs of a call that ends in a device synchronisation.  Prints the card's name and power limit first, then one JSON
line per coder."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import new_bloom_filter_repo_b200 as pkg  # noqa: E402
from new_bloom_filter_repo_b200 import _cabi  # noqa: E402
from tests.util import synth_stream  # noqa: E402

POSITIONS = (0, 1, 15, 29)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else _cabi.device_info()["name"]


def measure(fn, runs):
    """-> (median ms, d2h_bytes of one call, d2d_bytes of one call, result of the last call)."""
    L, ctx = _cabi.lib(), _cabi.ctx()
    ms, res = [], None
    for _ in range(runs):
        L.rbf_reset_counters(ctx)
        t0 = time.perf_counter()
        res = fn()
        ms.append((time.perf_counter() - t0) * 1e3)
    return round(statistics.median(ms), 2), L.rbf_get_counter(ctx, b"d2h_bytes"), L.rbf_get_counter(ctx, b"d2d_bytes"), res


def run(frames, coder, runs):
    import torch
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=30)
    comp.entropy_coder = coder
    comp.compress_video(list(frames), input_color_space="YUV")
    payloads = list(comp._last_compressed_frames)
    fb = frames[0].data.nbytes
    full = comp.decompress_video(compressed_frames=payloads)          # warm-up: context, kernels, pool
    data = [np.asarray(f.data) for f in full]
    out = {"config": "3840x2160 YUV444 x 60 frames, keyframe_interval=30, lossless, batch_size=%d" % comp.batch_size,
           "entropy_coder": coder, "frame_bytes": fb, "runs": runs}
    with pkg.VideoReader(payloads, comp) as r:
        r.read(0, 60)
        dev = torch.empty((1,) + data[0].shape, dtype=torch.uint8, device="cuda")
        r.read(31, 32, out=dev)
        for pos in POSITIONS:
            i = 30 + pos
            ms, d2h, _, got = measure(lambda: r.read(i, i + 1), runs)
            assert np.array_equal(got[0].data, data[i]), i
            out[f"read({i},{i + 1})"] = {"ms": ms, "d2h_bytes": d2h}
            ms, d2h, d2d, _ = measure(lambda: r.read(i, i + 1, out=dev), runs)
            assert np.array_equal(dev[0].cpu().numpy(), data[i]), i
            out[f"read({i},{i + 1},out=cuda)"] = {"ms": ms, "d2h_bytes": d2h, "d2d_bytes": d2d}
        ms, d2h, _, got = measure(lambda: r.read(0, 60), runs)
        assert all(np.array_equal(g.data, d) for g, d in zip(got, data))
        out["read(0,60)"] = {"ms": ms, "d2h_bytes": d2h}
    del got
    ms, d2h, _, _ = measure(lambda: comp.decompress_video(compressed_frames=payloads), runs)
    out["decompress_video"] = {"ms": ms, "d2h_bytes": d2h}
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    frames = [pkg.YUVFrame(f) for f in synth_stream(2160, 3840, 60, 2, [0.01, 0.05, 0.15, 0.30])]
    for coder in ("zlib", "gpu"):
        print(json.dumps(run(frames, coder, args.runs)), flush=True)
