#!/usr/bin/env python3
"""compress_video / decompress_video frames per second of the drop-in on BASELINE configs[1] (1080p x 30, keyframe_interval 30) and
on 4K x 30, with the entropy stage on one thread and on the default thread pool (GPU box only).  One JSON line per case."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import new_bloom_filter_repo_b200 as pkg  # noqa: E402
from tests.util import synth_stream  # noqa: E402


def run(h, w, nfr, threads, mode, coder="zlib"):
    frames = [f for f in synth_stream(h, w, nfr, 2, [0.01, 0.05, 0.15, 0.30])]
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=30, num_threads=threads)
    comp.entropy_coder = coder
    comp.inter_frame_mode = mode
    comp.inter_frame_threshold = 3.0
    comp.compress_video(list(frames[:4]), input_color_space="YUV")          # warm-up (context, streams, zlib)
    t0 = time.perf_counter()
    stats = comp.compress_video(list(frames), input_color_space="YUV")
    t1 = time.perf_counter()
    dec = comp.decompress_video(compressed_frames=comp._last_compressed_frames)
    t2 = time.perf_counter()
    ok = comp.verify_lossless(frames, dec)["lossless"]
    return {"config": "%dx%d YUV444 x %d frames, keyframe_interval=30, inter_frame_mode=%s" % (w, h, nfr, mode), "entropy_coder": coder,
            "zlib_threads": threads or "default(%d)" % comp.num_threads,
            "compress_fps": nfr / (t1 - t0), "decompress_fps": nfr / (t2 - t1), "keyframes": stats["keyframes"], "ratio": stats["compression_ratio"],
            "lossless": bool(ok)}


if __name__ == "__main__":
    import faulthandler
    faulthandler.dump_traceback_later(120, repeat=True)          # a stuck run shows where
    sizes = ((1080, 1920), (2160, 3840)) if "--4k" in sys.argv else ((1080, 1920),)
    for (h, w) in sizes:
        for coder, threads in (("zlib", 1), ("zlib", None), ("gpu", None)):
            for mode in ("lossless", "reference"):
                t0 = time.perf_counter()
                line = run(h, w, 30, threads, mode, coder)
                line["wall_s_incl_synthesis_and_warmup"] = time.perf_counter() - t0
                print(json.dumps(line), flush=True)
