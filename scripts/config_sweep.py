"""GPU: throughput of the other BASELINE.json configs (1080p 30-frame stream; 8K 16-bit k* sweep) and of the N1 / N2 kernels
(ordered gather of the changed values, one-pair apply), one JSON line each.  Parity for these shapes is covered by
tests/test_gpu_parity.py; this script only times them (CUDA events inside the library)."""
import ctypes as C, json, math, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import new_bloom_filter_repo_b200 as pkg
from new_bloom_filter_repo_b200 import _cabi as cabi
L, ctx = cabi.lib(), cabi.ctx()


def timed(st, fn, reps=5, warm=2):
    for _ in range(warm):
        fn()
    cabi.check(L.rbf_timer_start(ctx), ctx)
    for _ in range(reps):
        res = fn()
    ms = C.c_double(); cabi.check(L.rbf_timer_stop_ms(ctx, C.byref(ms)), ctx)
    return ms.value / reps, res


ONLY = os.environ.get("RBF_SWEEP_ONLY", "")         # "gather": just the N1/N2 section (for an ncu launch list of its kernels)

# ---- config[1]: 1080p YUV444 30-frame stream, keyframe_interval=30 -> 29 inter-frame pairs, mixed densities
if not ONLY:
    h, w, F = 1080, 1920, 30
    rng = np.random.default_rng(2)
    frames = np.empty((F, h, w, 3), np.uint8)
    frames[0] = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    dens = [0.01, 0.05, 0.15, 0.30]
    for t in range(1, F):
        p = dens[(t - 1) % 4]
        d = (np.random.default_rng(2 + t).random((h, w)) < p).astype(np.uint8) * np.uint8(64)
        np.add(frames[t - 1], d[:, :, None], out=frames[t])
    st = pkg.FrameStream(h, w, 3, np.uint8, max_frames=F)
    st.upload(frames)
    ms, res = timed(st, lambda: st.encode_consecutive(F, 3.0))
    print(json.dumps({"config": "1080p YUV444 30 frames, 29 inter-frame pairs, p cycling 0.01/0.05/0.15/0.30", "ms_per_step": ms,
                      "Mpixels_per_s": 29 * h * w / ms / 1e3, "stage_ms": st.stage_ms(), "raw_pairs": sum(r.raw for r in res)}), flush=True)
    st.close()

# ---- N1 / N2 at 4K: gather of the changed values of 16 pairs (p = 0.05) and one apply_diff, device time incl. the D2H of the values
h, w, F = 2160, 3840, 17
import bench as _bench
frames = np.empty((F, h, w, 3), np.uint8)
_bench.fill_stream(frames, seed=3)
st = pkg.FrameStream(h, w, 3, np.uint8, max_frames=F + 1)
st.upload(frames)
res = st.encode_consecutive(F, 3.0)
ms, vals = timed(st, lambda: st.gather_changed(F - 1), reps=5, warm=2)
nbytes = sum(v.nbytes for v in vals)
mask = np.unpackbits(st.fetch_batch(0, 1, want_masks=True)[2][0], bitorder="little")[: h * w]
ms2, _ = timed(st, lambda: st.apply_diff(F - 1, mask, vals[0]), reps=5, warm=2)        # into the spare slot F
print(json.dumps({"config": "N1 gather_changed, 4K YUV444, %d pairs, p=0.05 (incl. D2H of %.1f MB of values and the host-side offsets)" % (F - 1, nbytes / 1e6),
                  "ms_per_call": ms, "us_per_pair": ms * 1e3 / (F - 1),
                  "N2_apply_diff_one_4K_frame_ms (incl. H2D of mask + values)": ms2}), flush=True)
st.close()

if not ONLY:
    # ---- config[4]: 8K 16-bit, 16 frames, explicit k* sweep (l = int(p*n*k/ln2))
    h, w, F = 4320, 7680, 8
    frames = None
    n = h * w
    rng = np.random.default_rng(5)
    frames = np.empty((F, h, w, 3), np.uint16)
    frames[0] = rng.integers(0, 65536, (h, w, 3), dtype=np.uint16)
    for t in range(1, F):
        d = (np.random.default_rng(50 + t).integers(0, 20, (h, w), dtype=np.uint8) == 0).astype(np.uint16) * np.uint16(16384)
        np.add(frames[t - 1], d[:, :, None], out=frames[t])
    st = pkg.FrameStream(h, w, 3, np.uint16, max_frames=F)
    st.upload(frames)
    base = st.encode_consecutive(F, 3.0)
    for ks in (0.0, 1.5, 2.0, 2.5, 3.0, 3.5, 4.0):
        if ks == 0.0:
            fn = lambda: st.encode_consecutive(F, 3.0)
        else:
            lo = [int((np.uint64(r.ones) / n) * n * ks / math.log(2)) for r in base]
            fn = (lambda ks=ks, lo=lo: st.encode_consecutive(F, 3.0, k_override=[ks] * (F - 1), l_override=lo))
        ms, res = timed(st, fn, reps=3, warm=1)
        print(json.dumps({"config": "8K (7680x4320) 16-bit YUV444, %d pairs, k*=%s" % (F - 1, "auto" if ks == 0 else ks), "ms_per_step": ms,
                          "Mpixels_per_s": (F - 1) * n / ms / 1e3, "l_bits": res[0].l, "stage_ms": st.stage_ms(),
                          "roundtrip_mismatch_words": int(st.decode_verify().sum())}), flush=True)
    st.close()
