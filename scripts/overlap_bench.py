#!/usr/bin/env python3
"""What bounds the pipelined encode (encode_ranges = R, pipe_k1_sms = S) on ONE resident 4K stream (GPU box only).
    python scripts/overlap_bench.py [--frames 300] [--out overlap.json]

1. K1 alone (a k1_only stream, no K2 beside it): every k_threshold_sweep launch under torch.profiler, range 0 over the whole GPU
   and ranges 1.. on S SMs, as GB/s of distinct frame bytes (each frame of a range's chain is read once).
2. The overlapped encode under torch.profiler: per range, the K1 and K2 (k_insert_cluster) kernel times, so that the longer of
   the two shows which one bounds the overlap.
3. A sweep of (R, S) against the serial encode (R = 1): the library's stage events (rbf_stream_stage_ms), mean of 3 timed encodes
   after 2 warm-up encodes each, and a sha256 over every bitmap, witness and result field (every row must equal the serial one)."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402


def set_opts(cabi, **opts):
    L, ctx = cabi.lib(), cabi.ctx()
    for k, v in opts.items():
        cabi.check(L.rbf_set_option(ctx, k.encode(), int(v)), ctx)


def profiled(fn):
    """-> [(name, grid, block, start us, duration us)] of the library's kernels that fn ran, in start order."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device="cuda").add_(1)
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            ev = json.load(f)["traceEvents"]
    ks = sorted((e for e in ev if e.get("cat") == "kernel" and "rbf::" in e["name"]), key=lambda e: e["ts"])
    return [(e["name"], tuple(e["args"].get("grid", ())), tuple(e["args"].get("block", ())), float(e["ts"]), float(e["dur"])) for e in ks]


def bounds(P, R):
    return [P * r // R for r in range(R + 1)]


def digest(st, res):
    bms, wts, _ = st.fetch_batch(0, len(res))
    h = hashlib.sha256()
    for t, r in enumerate(res):
        h.update(repr((r.ones, r.resid, r.raw, r.l, r.wlen, r.k.hex(), r.p.hex())).encode())
        h.update(bms[t, :(r.l + 7) // 8].tobytes())
        h.update(wts[t, :(r.wlen + 7) // 8].tobytes())
    return h.hexdigest()[:16]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--ranges", default="2,3,4,6,8")
    ap.add_argument("--sms", default="22,33,44,55,66")
    ap.add_argument("--k1-sms", default="16,22,33,44,55,66,88,110")
    ap.add_argument("--profile", default="4:44", help="R:S of parts 1 and 2")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import new_bloom_filter_repo_b200 as pkg
    cabi = pkg._cabi
    info = cabi.device_info()
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                 # the card's name and power limit belong beside every number
        smi = "nvidia-smi failed: %r" % e
    F, H, W = args.frames, 2160, 3840
    P, fbytes = F - 1, H * W * 3
    frames, pin = bench.pinned_array(cabi, (F, H, W, 3))
    bench.fill_stream(frames, seed=3)
    st = pkg.FrameStream(H, W, 3, np.uint8, max_frames=F)
    st.upload(frames)
    out = {"device": info["name"], "sm_count": info["sm_count"], "nvidia_smi": smi, "frames": F}
    R0, S0 = (int(x) for x in args.profile.split(":"))

    # 1. K1 alone
    st.set_option("k1_only", 1)
    k1 = []
    for S in [int(x) for x in args.k1_sms.split(",")]:
        set_opts(cabi, encode_ranges=R0, pipe_k1_sms=S, kq_ranges=1)
        st.encode_consecutive(F, 3.0)
        ks = [k for k in profiled(lambda: st.encode_consecutive(F, 3.0)) if "k_threshold_sweep" in k[0]]
        b = bounds(P, R0)
        for r, k in enumerate(ks):
            gb = (b[r + 1] - b[r] + 1) * fbytes / (k[4] * 1e-6) / 1e9
            k1.append({"S": S, "range": r, "grid": k[1], "block": k[2], "us": round(k[4], 1), "GBps": round(gb, 1)})
    st.set_option("k1_only", 0)
    out["k1_alone"] = k1
    print(json.dumps({"k1_alone": k1}), flush=True)

    # 2. the overlapped encode, kernel by kernel
    set_opts(cabi, encode_ranges=R0, pipe_k1_sms=S0)
    st.encode_consecutive(F, 3.0)
    ks = profiled(lambda: st.encode_consecutive(F, 3.0))
    t0 = ks[0][3]
    tl = [{"kernel": k[0].split("(")[0].replace("void ", "")[:40], "grid": k[1], "block": k[2], "start_us": round(k[3] - t0, 1),
           "us": round(k[4], 1)} for k in ks if "k_threshold_sweep" in k[0] or "k_insert" in k[0] or "k_query" in k[0]]
    out["timeline"] = tl
    print(json.dumps({"timeline": tl}), flush=True)

    # 3. the (R, S) sweep
    configs = [(1, S0)] + [(R, S) for R in [int(x) for x in args.ranges.split(",")] for S in [int(x) for x in args.sms.split(",")]]
    ref = None
    sweep = []
    for R, S in configs:
        set_opts(cabi, encode_ranges=R, pipe_k1_sms=S, kq_ranges=1)
        for _ in range(2):
            res = st.encode_consecutive(F, 3.0)
        acc = {}
        for _ in range(3):
            res = st.encode_consecutive(F, 3.0)
            for k, v in st.stage_ms().items():
                acc[k] = acc.get(k, 0.0) + v / 3
        d = digest(st, res)
        ref = ref or d
        line = {"R": R, "S": S, "stage_ms": {k: round(v, 3) for k, v in acc.items()}, "same_as_serial": d == ref}
        sweep.append(line)
        print(json.dumps(line), flush=True)
    out["sweep"] = sweep
    set_opts(cabi, encode_ranges=1, pipe_k1_sms=S0)
    st.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
