#!/usr/bin/env python3
"""Compressed size and speed of value_coding "plain", "adaptive" (RBF3: residuals where they are shorter) and "motion" (RBF4: also
residuals against the block-motion-compensated previous frame), for both entropy coders, on seeded YUV444 8-bit content at 1080p and
4K in one lossless GOP:

  pan+noise    a textured pan of 1 px per frame plus Gaussian noise (sigma 1.5): the lossless mask flags nearly every pixel
  pan          the same pan without noise
  pan2d+noise  a textured pan of 3 px right and 2 px up per frame plus the same noise
  pan2d        the same 2-D pan without noise
  box          a static textured background with a flat box moving 4 px per frame: few changed pixels
  synth        tests/util.synth_stream: Bernoulli-chosen pixels change by +64 on every channel

Per row: total and inter-payload bytes, how many inter frames chose residuals (vmode 1) and motion residuals (vmode 2), and compress /
decompress frames/s (host clock around calls that end in a device synchronisation; best of --reps after a warm-up).  Every decode is
checked against the input.  Per size, the device time of FrameStream.motion_search per YUV444 pair (CUDA events around one call over
7 pairs, field copy included; best of 5).  The card name, power limit and max SM clock are read in the same run.  One JSON line per
row, then a markdown table."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import new_bloom_filter_repo_b200 as pkg  # noqa: E402
from new_bloom_filter_repo_b200 import improved_video_compressor as ivcmod  # noqa: E402
from tests.util import synth_stream  # noqa: E402


def texture(h, w, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    f1, f2, f3 = rng.uniform(20, 45, 3)
    t = 128 + 60 * np.sin(xx / f1) * np.cos(yy / f2) + 30 * np.sin((xx + yy) / (f3 / 3))
    return np.stack([t, 128 + 0.3 * (t - 128), 128 - 0.2 * (t - 128)], -1)


def content(kind, h, w, nfr, seed):
    rng = np.random.default_rng(seed)
    if kind == "synth":
        return [x for x in synth_stream(h, w, nfr, seed, [0.01, 0.05, 0.15, 0.30])]
    big = texture(h + 2 * nfr, w + 3 * nfr, seed)         # texture() is a function of the coordinates: tex is the same as texture(h, w + nfr)
    tex = big[:h, :w + nfr]
    out = []
    for t in range(nfr):
        if kind.startswith("pan2d"):                      # frame t+1 (y, x) = frame t (y + 2, x - 3)
            f = big[2 * t:2 * t + h, 3 * (nfr - t):3 * (nfr - t) + w] + (rng.normal(0, 1.5, (h, w, 3)) if kind == "pan2d+noise" else 0)
            f = np.clip(np.rint(f), 0, 255).astype(np.uint8)
        elif kind == "box":
            f = np.clip(np.rint(tex[:, :w]), 0, 255).astype(np.uint8)
            x0 = w // 8 + 4 * t
            f[h // 5:h // 5 + h // 10, x0:x0 + w // 16] = (200, 90, 60)
        else:
            f = tex[:, t:t + w] + (rng.normal(0, 1.5, (h, w, 3)) if kind == "pan+noise" else 0)
            f = np.clip(np.rint(f), 0, 255).astype(np.uint8)
        out.append(np.ascontiguousarray(f))
    return out


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else pkg._cabi.device_info()["name"]


def run(frames, coder, coding, reps):
    best_c = best_d = float("inf")
    for _ in range(reps):
        comp = pkg.ImprovedVideoCompressor(keyframe_interval=30)
        comp.entropy_coder, comp.value_coding = coder, coding
        yuv = [pkg.YUVFrame(f) for f in frames]
        t0 = time.perf_counter()
        comp.compress_video(yuv, input_color_space="YUV")
        t1 = time.perf_counter()
        pls = list(comp._last_compressed_frames)
        dec = comp.decompress_video(compressed_frames=pls)
        t2 = time.perf_counter()
        assert all(np.array_equal(np.asarray(d.data if hasattr(d, "yuv_info") else d), f) for d, f in zip(dec, frames)), "not lossless"
        best_c, best_d = min(best_c, t1 - t0), min(best_d, t2 - t1)
    inter = [p for p in pls if p.startswith(ivcmod._INTER_TAGS)]
    vmodes = [ivcmod.ImprovedVideoCompressor._parse_inter(p).vmode for p in inter]
    return {"total_bytes": sum(len(p) for p in pls), "inter_bytes": sum(len(p) for p in inter), "inter_frames": len(inter),
            "residual_frames": vmodes.count(1), "motion_frames": vmodes.count(2), "compress_fps": round(len(frames) / best_c, 2), "decompress_fps": round(len(frames) / best_d, 2)}


def motion_search_ms(h, w, reps=5):
    """Device time (CUDA events) of one motion_search call over 7 YUV444 8-bit pairs of the 2-D pan, per pair."""
    import ctypes as C
    frames = content("pan2d+noise", h, w, 8, 7)
    st = pkg.FrameStream(h, w, 3, np.uint8, max_frames=8, max_pairs=7, k1_only=True, mask_mode=1)
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    try:
        st.upload(np.stack(frames))
        st.encode_consecutive(8, 0.0)
        st.motion_search()                                                   # warm-up
        best = float("inf")
        for _ in range(reps):
            ms = C.c_double()
            pkg._cabi.check(L.rbf_timer_start(ctx), ctx)
            st.motion_search()
            pkg._cabi.check(L.rbf_timer_stop_ms(ctx, C.byref(ms)), ctx)
            best = min(best, ms.value / 7)
        return best
    finally:
        st.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--sizes", default="1080p,4k")
    ap.add_argument("--kinds", default="pan+noise,pan,pan2d+noise,pan2d,box,synth")
    a = ap.parse_args()
    sizes = {"1080p": (1080, 1920), "4k": (2160, 3840)}
    print(json.dumps({"card": card(), "threads": pkg.ImprovedVideoCompressor().num_threads}), flush=True)
    rows = []
    for size in a.sizes.split(","):
        h, w = sizes[size]
        print(json.dumps({"size": size, "motion_search_ms_per_pair": round(motion_search_ms(h, w), 4)}), flush=True)
        warm = content("synth", h, w, 3, 0)
        for coder in ("zlib", "gpu"):
            run(warm, coder, "adaptive", 1)                                   # context, kernels, pool
        for i, kind in enumerate(a.kinds.split(",")):
            frames = content(kind, h, w, a.frames, 100 + i)
            raw = sum(f.nbytes for f in frames)
            for coder in ("zlib", "gpu"):
                for coding in ("plain", "adaptive", "motion"):
                    r = {"size": size, "content": kind, "coder": coder, "value_coding": coding, "frames": a.frames, "raw_bytes": raw}
                    r.update(run(frames, coder, coding, a.reps))
                    rows.append(r)
                    print(json.dumps(r), flush=True)
    print("| size | content | coder | coding | total / raw | inter bytes | vmode 1 / 2 frames | compress fps | decompress fps |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %s | %s | %s | %s | %.4f | %d | %d / %d of %d | %.2f | %.2f |" % (
            r["size"], r["content"], r["coder"], r["value_coding"], r["total_bytes"] / r["raw_bytes"], r["inter_bytes"],
            r["residual_frames"], r["motion_frames"], r["inter_frames"], r["compress_fps"], r["decompress_fps"]))


if __name__ == "__main__":
    main()
