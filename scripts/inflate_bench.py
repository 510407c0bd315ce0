#!/usr/bin/env python3
"""GPU inflate of the device coder's zlib streams against zlib.decompress, and decompress_video with it against the host route.

1. GB/s of inflated output: the four blobs of a 4K YUV444 keyframe, and the value streams of 29 4K pairs, inflated with
   deflate.decompress_many (one batch), with zlib.decompress on one thread and on a pool of os.cpu_count() threads.
2. decompress_video frames/s of GPU-coded 1080p x 30 and 4K x 30 YUV444 GOPs: the device route and the host route (every value
   stream and keyframe blob inflated with zlib.decompress, forced here by substituting the host inflater), alternated, 3 runs
   each, identical frames required.
3. Per group of the device route: device-event time of inflate_values, decode_masks and apply_chain, and host wall time.
The card's name and power limit are read in the same command.  One JSON line per result."""
import ctypes
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
from new_bloom_filter_repo_b200 import _cabi, deflate  # noqa: E402
from new_bloom_filter_repo_b200 import improved_video_compressor as ivcmod  # noqa: E402
from tests.util import synth_stream  # noqa: E402

IVC = ivcmod.ImprovedVideoCompressor


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else _cabi.device_info()["name"]


def gop(h, w):
    frames = [pkg.YUVFrame(f) for f in synth_stream(h, w, 30, 2, [0.01, 0.05, 0.15, 0.30])]
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=30)
    comp.entropy_coder = "gpu"
    comp.compress_video(list(frames), input_color_space="YUV")
    return comp, frames, list(comp._last_compressed_frames)


def best_of(fn, reps=5):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return min(ts)


def inflate_rates(name, streams, bounds, pool):
    out = sum(len(x) for x in deflate.decompress_many(streams, bounds))
    got, dev = deflate.decompress_routed(streams, bounds)
    assert all(dev) and got == [zlib.decompress(s) for s in streams]
    t_gpu = best_of(lambda: deflate.decompress_many(streams, bounds))
    t_one = best_of(lambda: [zlib.decompress(s) for s in streams], 3)
    t_pool = best_of(lambda: list(pool.map(zlib.decompress, streams)), 3)
    return {"case": name, "streams": len(streams), "compressed_MB": round(sum(map(len, streams)) / 1e6, 2),
            "inflated_MB": round(out / 1e6, 2), "gpu_GBps": round(out / t_gpu / 1e9, 3), "zlib_1thread_GBps": round(out / t_one / 1e9, 3),
            "zlib_pool_GBps": round(out / t_pool / 1e9, 3), "pool_threads": pool._max_workers,
            "gpu_ms": round(t_gpu * 1e3, 2), "zlib_1thread_ms": round(t_one * 1e3, 2), "zlib_pool_ms": round(t_pool * 1e3, 2)}


class HostRoute:
    """decompress_video with every value stream and keyframe blob inflated by zlib.decompress (the default coder's route)."""

    def __enter__(self):
        self.saved = (IVC.__dict__["_inflate_group"], IVC.__dict__["_start_key"])

        def host_group(st, jobs, pool):
            for j in jobs:
                if j.p is not None and j.values is None:
                    j.values = pool.submit(zlib.decompress, j.p.vz)
        IVC._inflate_group = staticmethod(host_group)
        IVC._start_key = lambda self, payload, pool: pool.submit(self.compressor.decompress_frame, payload)
        return self

    def __exit__(self, *exc):
        IVC._inflate_group, IVC._start_key = self.saved


class StageTimer:
    """Device-event time per call of the named FrameStream methods, and host wall time of each decompress_video group."""
    NAMES = ("inflate_values", "decode_masks", "apply_chain")

    def __enter__(self):
        L, ctx = _cabi.lib(), _cabi.ctx()
        self.ms = {n: [] for n in self.NAMES}
        self.ms["group_wall"] = []
        self.saved = {n: getattr(pkg.FrameStream, n) for n in self.NAMES}
        self.saved_group = IVC._decode_group
        for n, fn in self.saved.items():
            def timed(st, *a, _fn=fn, _n=n, **k):
                _cabi.check(L.rbf_timer_start(ctx), ctx)
                r = _fn(st, *a, **k)
                ms = ctypes.c_double()
                _cabi.check(L.rbf_timer_stop_ms(ctx, ctypes.byref(ms)), ctx)
                self.ms[_n].append(round(ms.value, 3))
                return r
            setattr(pkg.FrameStream, n, timed)
        orig = self.saved_group

        def group(st, base, g):
            t0 = time.perf_counter()
            r = orig(st, base, g)
            self.ms["group_wall"].append(round((time.perf_counter() - t0) * 1e3, 3))
            return r
        IVC._decode_group = staticmethod(group)
        return self

    def __exit__(self, *exc):
        for n, fn in self.saved.items():
            setattr(pkg.FrameStream, n, fn)
        IVC._decode_group = staticmethod(self.saved_group)


def data(frames):
    return [np.asarray(f.data if hasattr(f, "yuv_info") else f) for f in frames]


def decode_fps(h, w, comp, frames, pls, runs=3):
    comp.decompress_video(compressed_frames=pls)                       # warm-up of both routes
    with HostRoute():
        comp.decompress_video(compressed_frames=pls)
    t_dev, t_host = [], []
    for _ in range(runs):
        t0 = time.perf_counter()
        a = comp.decompress_video(compressed_frames=pls)
        t1 = time.perf_counter()
        with HostRoute():
            b = comp.decompress_video(compressed_frames=pls)
        t2 = time.perf_counter()
        t_dev.append(t1 - t0)
        t_host.append(t2 - t1)
        assert all(np.array_equal(x, y) for x, y in zip(data(a), data(b))), "the routes disagree"
        assert all(np.array_equal(x, y) for x, y in zip(data(a), data(frames))), "not lossless"
    with StageTimer() as tm:
        t0 = time.perf_counter()
        comp.decompress_video(compressed_frames=pls)
        wall = time.perf_counter() - t0
    return {"case": "decompress_video %dx%d YUV444 x 30, GPU coder" % (w, h), "threads": comp.num_threads,
            "device_inflate_fps": [round(30 / t, 2) for t in t_dev], "host_inflate_fps": [round(30 / t, 2) for t in t_host],
            "identical_frames": True, "timed_run_wall_ms": round(wall * 1e3, 2),
            "per_group_ms": tm.ms}


if __name__ == "__main__":
    import faulthandler
    faulthandler.dump_traceback_later(900, repeat=True)
    print(json.dumps({"card": card()}), flush=True)
    pool = ThreadPoolExecutor(os.cpu_count() or 1)
    comp4k, frames4k, pls4k = gop(2160, 3840)
    blobs = pkg.FixedVideoCompressor.keyframe_blobs(pls4k[0])
    print(json.dumps(inflate_rates("4K YUV444 keyframe blobs", [b for b, _ in blobs], [n for _, n in blobs], pool)), flush=True)
    inter = [IVC._parse_inter(p) for p in pls4k[1:]]
    print(json.dumps(inflate_rates("value streams of 29 4K pairs", [bytes(p.vz) for p in inter], [p.vcount * p.isz for p in inter],
                                   pool)), flush=True)
    comp1k, frames1k, pls1k = gop(1080, 1920)
    print(json.dumps(decode_fps(1080, 1920, comp1k, frames1k, pls1k)), flush=True)
    print(json.dumps(decode_fps(2160, 3840, comp4k, frames4k, pls4k)), flush=True)
