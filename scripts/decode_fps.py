#!/usr/bin/env python3
"""decompress_video frames per second (batched group decode) against the per-frame route it replaced, rebuilt here from public
calls -- BloomFilterCompressor.decompress, FrameStream.apply_diff and FrameStream.download per inter frame -- on the same payloads:
1080p x 30 and 4K x 30 YUV444, one GOP of 30, lossless mode, both entropy coders.  The two routes alternate, 3 runs each, and must
give identical frames.  Also prints the device-event time of decode_masks and apply_chain per group, and the card (GPU box only).
One JSON line per case."""
import ctypes
import json
import os
import subprocess
import sys
import time
import zlib

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import new_bloom_filter_repo_b200 as pkg  # noqa: E402
from new_bloom_filter_repo_b200 import _cabi  # noqa: E402
from new_bloom_filter_repo_b200 import improved_video_compressor as ivcmod  # noqa: E402
from tests.util import synth_stream  # noqa: E402


def per_frame_decode(comp, payloads):
    """The per-frame route: keyframes one by one, each inter frame decoded, applied and downloaded on its own."""
    frames, st = [], None
    for c in payloads:
        if not c.startswith((ivcmod._INTER_TAG, ivcmod._INTER_TAG_V1)):
            frames.append(comp.compressor.decompress_frame(c))
            continue
        p = ivcmod.ImprovedVideoCompressor._parse_inter(c)
        dtype = np.uint8 if p.isz == 1 else np.uint16
        values = np.frombuffer(zlib.decompress(p.vz), dtype=dtype)[:p.vcount]
        n = p.h * p.w
        if p.raw:
            mask = np.unpackbits(np.frombuffer(zlib.decompress(p.mask_bytes), dtype=np.uint8))[:n]
        else:
            bitmap = np.unpackbits(np.frombuffer(p.mask_bytes, dtype=np.uint8))[:p.l]
            witness = np.unpackbits(np.frombuffer(p.witness_bytes, dtype=np.uint8))[:p.wlen]
            mask = pkg.BloomFilterCompressor().decompress(bitmap, witness, n, p.k)
        prev = frames[-1]
        if st is None:
            st = pkg.FrameStream(p.h, p.w, p.ch, dtype, max_frames=2, max_pairs=1, k1_only=True)
        st.upload(np.ascontiguousarray(prev.data if hasattr(prev, "yuv_info") else prev)[None], first=0)
        assert st.apply_diff(0, mask, values) == p.ones
        out = st.download(1)
        frames.append(pkg.YUVFrame(out) if hasattr(prev, "yuv_info") else out)
    if st is not None:
        st.close()
    return frames


class StageTimer:
    """Device-event time (rbf_timer_start / rbf_timer_stop_ms on the context's stream) of FrameStream.decode_masks and
    FrameStream.apply_chain -- and, for GPU-coded files, inflate_values -- per call."""

    def __init__(self):
        self.ms = {"inflate_values": [], "decode_masks": [], "apply_chain": []}
        self._orig = {}

    def __enter__(self):
        L, ctx = _cabi.lib(), _cabi.ctx()
        for name in self.ms:
            fn = getattr(pkg.FrameStream, name)
            self._orig[name] = fn

            def timed(st, *a, _fn=fn, _name=name, **k):
                _cabi.check(L.rbf_timer_start(ctx), ctx)
                r = _fn(st, *a, **k)
                ms = ctypes.c_double()
                _cabi.check(L.rbf_timer_stop_ms(ctx, ctypes.byref(ms)), ctx)
                self.ms[_name].append(ms.value)
                return r
            setattr(pkg.FrameStream, name, timed)
        return self

    def __exit__(self, *exc):
        for name, fn in self._orig.items():
            setattr(pkg.FrameStream, name, fn)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else _cabi.device_info()["name"]


def data(frames):
    return [np.asarray(f.data if hasattr(f, "yuv_info") else f) for f in frames]


def run(h, w, coder, runs=3):
    frames = [pkg.YUVFrame(f) for f in synth_stream(h, w, 30, 2, [0.01, 0.05, 0.15, 0.30])]
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=30)
    comp.entropy_coder = coder
    comp.compress_video(list(frames), input_color_space="YUV")
    payloads = list(comp._last_compressed_frames)
    comp.decompress_video(compressed_frames=payloads[:4])                  # warm-up: context, kernels, pool
    per_frame_decode(comp, payloads[:4])
    t_new, t_old = [], []
    for _ in range(runs):
        t0 = time.perf_counter()
        new = comp.decompress_video(compressed_frames=payloads)
        t1 = time.perf_counter()
        old = per_frame_decode(comp, payloads)
        t2 = time.perf_counter()
        t_new.append(t1 - t0)
        t_old.append(t2 - t1)
        assert all(np.array_equal(a, b) for a, b in zip(data(new), data(old))), "the routes disagree"
        assert all(np.array_equal(a, b) for a, b in zip(data(new), data(frames))), "not lossless"
    with StageTimer() as tm:
        comp.decompress_video(compressed_frames=payloads)
    ni = sum(p.startswith(ivcmod._INTER_TAG) for p in payloads)
    return {"config": "%dx%d YUV444 x 30 frames, keyframe_interval=30, lossless, batch_size=%d" % (w, h, comp.batch_size),
            "entropy_coder": coder, "inter_frames": ni, "threads": comp.num_threads,
            "decompress_fps": [round(30 / t, 2) for t in t_new], "per_frame_route_fps": [round(30 / t, 2) for t in t_old],
            "identical_frames": True,
            "decode_masks_ms_per_group": [round(x, 3) for x in tm.ms["decode_masks"]],
            "apply_chain_ms_per_group": [round(x, 3) for x in tm.ms["apply_chain"]],
            "inflate_values_ms_per_group": [round(x, 3) for x in tm.ms["inflate_values"]]}


if __name__ == "__main__":
    import faulthandler
    faulthandler.dump_traceback_later(600, repeat=True)          # a stuck run shows where
    print(json.dumps({"card": card()}), flush=True)
    for (h, w) in ((1080, 1920), (2160, 3840)):
        for coder in ("zlib", "gpu"):
            print(json.dumps(run(h, w, coder)), flush=True)
