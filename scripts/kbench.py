#!/usr/bin/env python3
"""A/B timing of kernel variants and pipeline settings on ONE resident 4K stream (GPU box only).
    python scripts/kbench.py [--frames 120] [--out kbench.jsonl]
Each configuration: 2 warm-up encodes, 3 timed; prints one JSON line per configuration with the stage times (CUDA events
inside the library) and a sha256 over all bitmaps + witnesses, so that a variant that changes a single bit is visible at once."""
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
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--out", default=None)
    ap.add_argument("--one-in", type=int, default=20, help="change density 1/one_in of the synthetic stream (20 -> p = 0.05)")
    ap.add_argument("--configs", default=None, help="JSON list of option dicts; default: the built-in sweep")
    args = ap.parse_args()
    import new_bloom_filter_repo_b200 as pkg
    cabi = pkg._cabi
    L, ctx = cabi.lib(), cabi.ctx()
    F, H, W = args.frames, args.height, args.width
    frames, pin = bench.pinned_array(cabi, (F, H, W, 3))
    bench.fill_stream(frames, seed=3, one_in=args.one_in)
    st = pkg.FrameStream(H, W, 3, np.uint8, max_frames=F)
    st.upload(frames)
    base = {"query_variant": 5, "insert_variant": 1, "encode_ranges": 1, "pipe_k1_sms": 66, "query_smem_bytes": 0, "query_warps": 0, "kq_ranges": 1}
    sweep = json.loads(args.configs) if args.configs else [
        {}, {"query_variant": 1}, {"query_variant": 6}, {"insert_variant": 0}, {"encode_ranges": 4},
        {"query_smem_bytes": 200000}, {"query_smem_bytes": 170000}, {"query_smem_bytes": 140000}, {"query_smem_bytes": 110000},
    ]
    out = open(args.out, "w") if args.out else None
    ref_sha = None
    for cfg in sweep:
        opts = dict(base, **cfg)
        for k, v in opts.items():
            cabi.check(L.rbf_set_option(ctx, k.encode(), int(v)), ctx)
        for _ in range(2):
            res = st.encode_consecutive(F, 3.0)
        acc, tot = {}, []
        for _ in range(3):
            res = st.encode_consecutive(F, 3.0)
            ms = st.stage_ms()
            tot.append(ms["encode_total"])
            for k, v in ms.items():
                acc[k] = acc.get(k, 0.0) + v / 3
        bms, wts, _ = st.fetch_batch(0, F - 1)
        h = hashlib.sha256()
        for t, r in enumerate(res):
            h.update(bms[t, :(r.l + 7) // 8].tobytes())
            h.update(wts[t, :(r.wlen + 7) // 8].tobytes())
        sha = h.hexdigest()[:16]
        ref_sha = ref_sha or sha
        px = (F - 1) * H * W
        line = {"cfg": cfg, "stage_ms": {k: round(v, 4) for k, v in acc.items()}, "total_ms_min": round(min(tot), 4),
                "gpx_s": round(px / min(tot) / 1e6, 2), "us_per_pair_k3": round(acc["k3_query"] * 1e3 / (F - 1), 3),
                "sha16": sha, "same_bits_as_first": sha == ref_sha}
        print(json.dumps(line), flush=True)
        if out:
            out.write(json.dumps(line) + "\n")
            out.flush()
    for k, v in base.items():
        L.rbf_set_option(ctx, k.encode(), int(v))
    st.close()


if __name__ == "__main__":
    main()
