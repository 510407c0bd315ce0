#!/usr/bin/env python3
"""Input GB/s and output/input ratio of the device zlib coder (deflate.compress_many, FrameStream.zlib_changed) next to CPU
zlib at levels 1 and 9 on one thread and on the default pool, all in one run (GPU box only).  One JSON line per case.
Workloads: the four blobs of one 4K YUV444 keyframe (frame + Y/U/V planes) and the changed values of 29 4K pairs at p = 0.05.
Device times are CUDA events around the whole call (host<->device copies included) after a warm-up."""
import json
import os
import subprocess
import sys
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import new_bloom_filter_repo_b200 as pkg  # noqa: E402
from new_bloom_filter_repo_b200 import _cabi  # noqa: E402
from tests.util import synth_stream  # noqa: E402


def gpu_ms(fn, reps):
    L, h = _cabi.lib(), _cabi.ctx()
    fn()                                                        # warm-up
    best, out = [], None
    for _ in range(reps):
        _cabi.check(L.rbf_timer_start(h), h)
        out = fn()
        ms = _cabi.C.c_double()
        _cabi.check(L.rbf_timer_stop_ms(h, _cabi.C.byref(ms)), h)
        best.append(ms.value)
    return float(np.median(best)), out


def cpu_s(bufs, level, threads):
    t0 = time.perf_counter()
    if threads == 1:
        out = [zlib.compress(b, level) for b in bufs]
    else:
        with ThreadPoolExecutor(threads) as pool:
            out = list(pool.map(lambda b: zlib.compress(b, level), bufs))
    return time.perf_counter() - t0, sum(len(z) for z in out)


def card():
    """name and power limit of the card, read in the same run as the measurement"""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", os.environ.get("RBF_DEVICE", "0")],
                           capture_output=True, text=True)
        if q.returncode == 0 and q.stdout.strip():
            return q.stdout.strip().splitlines()[0]
    except OSError:
        pass
    return _cabi.device_info()["name"] + ", power limit not readable"


def report(workload, nbytes, rows):
    for coder, secs, outb in rows:
        print(json.dumps({"workload": workload, "coder": coder, "input_bytes": nbytes, "seconds": secs,
                          "input_GBps": nbytes / secs / 1e9, "ratio": outb / nbytes, "card": CARD}), flush=True)


if __name__ == "__main__":
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 5
    CARD = card()
    pool_threads = max(1, min(32, os.cpu_count() or 2))
    # the four blobs of one 4K YUV444 keyframe
    f = pkg.YUVFrame(synth_stream(2160, 3840, 1, 2, [0.05])[0])
    raws = pkg.fixed_video_compressor.keyframe_raws(f)
    nb = sum(len(r) for r in raws)
    ms, zs = gpu_ms(lambda: pkg.deflate.compress_many(raws), reps)
    for z, r in zip(zs, raws):
        assert zlib.decompress(z) == r
    rows = [("gpu", ms / 1e3, sum(len(z) for z in zs))]
    for level in (1, 9):
        for th in (1, pool_threads):
            s, ob = cpu_s(raws, level, th)
            rows.append(("zlib-%d x%d threads" % (level, th), s, ob))
    report("4K YUV444 keyframe (frame + 3 planes)", nb, rows)
    del raws, zs
    # the changed values of 29 4K pairs at p = 0.05
    frames = synth_stream(2160, 3840, 30, 7, [0.05])
    st = pkg.FrameStream(2160, 3840, 3, np.uint8, max_frames=30)
    st.upload(frames)
    st.encode_consecutive(30, 3.0)
    vals = [g.tobytes() for g in st.gather_changed()]
    nb = sum(len(v) for v in vals)
    ms, zs = gpu_ms(lambda: st.zlib_changed(), reps)
    for z, v in zip(zs, vals):
        assert zlib.decompress(z) == v
    gms, _ = gpu_ms(lambda: st.gather_changed(), reps)
    rows = [("gpu gather+deflate (zlib_changed)", ms / 1e3, sum(len(z) for z in zs)),
            ("gpu gather only, raw copy (gather_changed)", gms / 1e3, nb)]
    for level in (1, 9):
        for th in (1, pool_threads):
            s, ob = cpu_s(vals, level, th)
            rows.append(("zlib-%d x%d threads" % (level, th), s, ob))
    report("changed values of 29 4K pairs, p=0.05", nb, rows)
    st.close()
