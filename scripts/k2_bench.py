#!/usr/bin/env python3
"""K2 (insert) alone, timed by the library's stage events, on one resident stream (GPU box only).
    python scripts/k2_bench.py [--pairs 1,8,31,299] [--reps 10] [--height 2160 --width 3840]
The frames are bench.py's synthetic stream.  For each pair count F: 2 warm-up encodes of pairs 0..F-1, then --reps timed
encodes; prints one JSON line per F with the K2 times and a sha256 over the bitmaps, so that two builds can be compared."""
import argparse
import hashlib
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", default="1,8,31,299")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--width", type=int, default=3840)
    args = ap.parse_args()
    import new_bloom_filter_repo_b200 as pkg
    cabi = pkg._cabi
    counts = [int(x) for x in args.pairs.split(",")]
    H, W, nfr = args.height, args.width, max(counts) + 1
    frames, pin = bench.pinned_array(cabi, (nfr, H, W, 3))
    bench.fill_stream(frames, seed=3)
    st = pkg.FrameStream(H, W, 3, np.uint8, max_frames=nfr)
    st.upload(frames)
    info = cabi.device_info()
    for F in counts:
        for _ in range(2):
            st.encode_consecutive(F + 1, 3.0)
        k2 = []
        for _ in range(args.reps):
            res = st.encode_consecutive(F + 1, 3.0)
            k2.append(st.stage_ms()["k2_insert"])
        bms, _, _ = st.fetch_batch(0, F)
        h = hashlib.sha256()
        for t, r in enumerate(res):
            h.update(bms[t, :(r.l + 7) // 8].tobytes())
        print(json.dumps({"gpu": info["name"], "pairs": F, "height": H, "width": W, "k2_ms_min": round(min(k2), 4),
                          "k2_ms_median": round(float(np.median(k2)), 4), "k2_ms_max": round(max(k2), 4),
                          "max_l": max(r.l for r in res), "bitmap_sha16": h.hexdigest()[:16]}), flush=True)
    st.close()


if __name__ == "__main__":
    main()
