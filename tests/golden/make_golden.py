#!/usr/bin/env python3
"""
Generates tests/golden/*.json|*.npz from the REAL reference
(ross39/new_bloom_filter_repo @ 7e37ed8, imported from $RBF_REFERENCE_DIR through
oracle/refshim.py).  Needs that checkout and cv2; the fixtures it writes are
committed and are what pins the oracle (the reference's own tests hold no golden
vectors -- SURVEY.md section 8c).

    RBF_REFERENCE_DIR=<checkout of the reference> python tests/golden/make_golden.py

Everything stored is an output of unmodified reference code:
  * xxhash.xxh64_intdigest / xxhash.xxh64(...).intdigest()  (the reference's L0)
  * ivc.RationalBloomFilter, ivc.BloomFilterCompressor, ivc.VideoFrameCompressor pieces
  * rbf.RationalBloomFilter / rbf.StandardBloomFilter, bc nested filter seeds
"""
import hashlib
import json
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))
from oracle import refshim  # noqa: E402

ivc, rbf, bc, fvc = refshim.load()
import xxhash  # noqa: E402  (the reference's dependency)


def sha(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def dump(name, obj):
    with open(os.path.join(HERE, name), "w") as f:
        json.dump(obj, f, indent=0, sort_keys=True)
    print("wrote", name)


# ---------------------------------------------------------------- xxh64 KATs
def gen_xxh64():
    seeds = [0x12345678, 0x87654321, 999, 0, 1, 2, 3, 4, 2 ** 32 - 1]
    items = set([0, 1, 7, 9, 10, 11, 42, 99, 100, 101, 999, 1000, 1001, 1234, 9999, 10000, 12345,
                 65535, 65536, 99999, 100000, 123456, 999999, 1000000, 1234567, 2073599, 2073600,
                 8294399, 8294400, 9999999, 10000000, 12345678, 33177599, 33177600, 99999999,
                 100000000, 123456789, 999999999, 1000000000, 2147483647, 4294967295])
    rng = random.Random(7)
    for digits in range(1, 11):
        lo, hi = (0 if digits == 1 else 10 ** (digits - 1)), min(10 ** digits - 1, 2 ** 32 - 1)
        for _ in range(40):
            items.add(rng.randint(lo, hi))
    dec = [{"item": it, "digests": [format(xxhash.xxh64_intdigest(str(it), s), "016x") for s in seeds]}
           for it in sorted(items)]
    # arbitrary strings (string API, rbf:115): lengths 0..100 incl. the >=32 B stripe loop
    strs = []
    for n in list(range(0, 70)) + [95, 96, 97, 100, 127, 128, 129, 255, 1000]:
        s = "".join(rng.choice("abcdefghijklmnopqrstuvwxyzABC0123456789 _-") for _ in range(n))
        strs.append({"s": s, "digests": [format(xxhash.xxh64(s, seed=sd).intdigest(), "016x") for sd in seeds]})
    strs.append({"s": "héllo wörld ✓", "digests": [format(xxhash.xxh64("héllo wörld ✓", seed=sd).intdigest(), "016x")
                                                   for sd in seeds]})
    dump("xxh64_kat.json", {"seeds": seeds, "decimal": dec, "strings": strs})


# ---------------------------------------------------------------- filter probes / activation
def gen_filter():
    out = []
    for size, k in [(1000, 2.3), (971, 3.1023850821971357), (476516, 3.1946), (1908872, 3.19), (7, 0.5),
                    (1, 1.0), (123457, 0.1), (2 ** 31 - 1, 4.75), (2 ** 32 - 5, 2.5), (65536, 12.99)]:
        f = ivc.RationalBloomFilter(size, k)
        items = [0, 1, 7, 10, 99, 100, 4095, 12345, 99999, 100000, 1234567, 8294399, 33177599, 123456789]
        rec = {"size": size, "k": k, "floor_k": f.floor_k, "p_activation": float(f.p_activation).hex(),
               "items": items,
               "probes": [[int(f._get_hash_indices(it, i)) for i in range(f.floor_k + 1)] for it in items],
               "activation": [bool(f._determine_activation(it)) for it in items]}
        out.append(rec)
    # activation rate KAT (SURVEY 8c): items 0..19999 with k*=2.3
    f = ivc.RationalBloomFilter(1000, 2.3)
    act = [bool(f._determine_activation(i)) for i in range(20000)]
    dump("filter_kat.json", {"filters": out, "act_count_k2.3_0..19999": int(sum(act)),
                             "act_bits_sha256": sha(np.packbits(np.array(act, dtype=np.uint8)))})


# ---------------------------------------------------------------- activation thresholds
def gen_threshold():
    """T(p) = #{h : h/(2**64-1) < p} found with the reference expression (ivc:95-97)."""
    d = 2 ** 64 - 1

    def T(p):
        lo, hi = 0, 2 ** 64
        while lo < hi:
            mid = (lo + hi) // 2
            if mid / d < p:
                lo = mid + 1
            else:
                hi = mid
        return lo

    rng = random.Random(11)
    ps = [2.3 - 2, 3.1023850821971357 - 3, 0.5, 0.25, 0.1, 0.75, 1 / 3, 0.999999, 1e-3, 1e-9, 2.0 ** -52,
          2.0 ** -53, 1 - 2.0 ** -53, 0.0, 5e-324, 1e-300, 2.0 ** -64, 2.0 ** -63, 3 * 2.0 ** -65]
    for _ in range(200):
        k = rng.uniform(0.1, 13.0)
        ps.append(k - int(k))
    for _ in range(50):
        ps.append(rng.random() * 10 ** rng.uniform(-18, 0))
    recs = [{"p": float(p).hex(), "T": format(T(p), "x")} for p in ps]
    # unit-division samples: h / (2**64-1)
    hs = [0, 1, 2, 2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1, 2 ** 54 + 1, 2 ** 54 + 2, 2 ** 54 + 3, 2 ** 63, 2 ** 64 - 1,
          2 ** 64 - 2, 2 ** 64 - 1025, 2 ** 64 - 2048, 0x4cccccccccccbe00, 0x4cccccccccccbdff]
    for _ in range(300):
        hs.append(rng.getrandbits(rng.randint(1, 64)))
    divs = [{"h": format(h, "x"), "q": float(h / d).hex()} for h in hs]
    dump("activation_kat.json", {"thresholds": recs, "unit_div": divs})


# ---------------------------------------------------------------- _calculate_optimal_params
def gen_params():
    c = ivc.BloomFilterCompressor()
    rng = random.Random(13)
    recs = []
    ns = [1, 2, 10, 100, 4096, 65536, 100000, 230400, 2073600, 8294400, 33177600]
    for n in ns:
        cand = {0, 1, 2, n // 10000, n // 10000 + 1, n // 1000, n // 100, n // 20, n // 10, n // 5, n // 4,
                int(n * 0.32452), int(n * 0.32453), int(n * 0.32453) + 1, int(n * 0.32454), n // 3, n // 2, n}
        for _ in range(40):
            cand.add(rng.randint(0, max(1, int(n * 0.35))))
        for ones in sorted(x for x in cand if 0 <= x <= n):
            p = np.uint64(ones) / n                       # as compress(): np.sum(uint8)/len  (ivc:211-212)
            k, l = c._calculate_optimal_params(n, p)
            recs.append({"n": n, "ones": ones, "p": float(p).hex(), "k": float(k).hex(), "l": int(l)})
    dump("params_kat.json", {"cases": recs})


# ---------------------------------------------------------------- compress / decompress
def mask_for(case):
    rng = np.random.default_rng(case["seed"])
    return (rng.random(case["n"]) < case["p_gen"]).astype(np.uint8)


def gen_compress():
    cases = [
        {"name": "survey_4096", "n": 4096, "seed": 0, "p_gen": 0.05},
        {"name": "n4096_p01", "n": 4096, "seed": 1, "p_gen": 0.01},
        {"name": "n4096_p15", "n": 4096, "seed": 2, "p_gen": 0.15},
        {"name": "n4096_p30", "n": 4096, "seed": 3, "p_gen": 0.30},
        {"name": "n4096_p40_raw", "n": 4096, "seed": 4, "p_gen": 0.40},
        {"name": "n4096_p0_raw", "n": 4096, "seed": 5, "p_gen": 0.0},
        {"name": "n4096_tiny_raw", "n": 40960, "seed": 6, "p_gen": 0.00005},
        {"name": "n1000_p05", "n": 1000, "seed": 7, "p_gen": 0.05},
        {"name": "n10_p2", "n": 10, "seed": 8, "p_gen": 0.2},
        {"name": "n101_p3", "n": 101, "seed": 9, "p_gen": 0.3},
        {"name": "n12345_p02", "n": 12345, "seed": 10, "p_gen": 0.02},
        {"name": "n100000_p05", "n": 100000, "seed": 11, "p_gen": 0.05},
        {"name": "n100000_p0005", "n": 100000, "seed": 12, "p_gen": 0.0005},
        {"name": "n230400_p05", "n": 230400, "seed": 13, "p_gen": 0.05},
        {"name": "n230400_p25", "n": 230400, "seed": 14, "p_gen": 0.25},
        {"name": "n1100000_p03", "n": 1100000, "seed": 15, "p_gen": 0.03},
    ]
    comp = ivc.BloomFilterCompressor()
    arrays = {}
    recs = []
    for cs in cases:
        m = mask_for(cs)
        bitmap, witness, p, n, ratio = comp.compress(m)
        k, l = comp._calculate_optimal_params(n, p)
        raw = len(witness) == 0 and len(bitmap) == n and (l == 0 or l >= n or p >= comp.P_STAR)
        w = np.array(witness, dtype=np.uint8)
        rec = dict(cs, ones=int(m.sum()), p=float(p).hex(), k=float(k).hex(), l=int(l), raw=bool(raw),
                   bitmap_len=int(len(bitmap)), witness_len=int(len(w)), ratio=float(ratio).hex(),
                   mask_sha256=sha(np.packbits(m)), bitmap_sha256=sha(np.packbits(bitmap)),
                   witness_sha256=sha(np.packbits(w)))
        if not raw:
            dec = comp.decompress(bitmap, witness, n, k)
            rec["roundtrip"] = bool(np.array_equal(dec, m))
            # the reference's own decode receives k rounded to float32 (ivc:938, ivc:986)
            k32 = float(np.float32(k))
            dec32 = comp.decompress(bitmap, witness[:] + [0] * 64, n, k32)
            rec["k_f32"] = float(k32).hex()
            rec["decoded_f32k_sha256"] = sha(np.packbits(dec32))
            rec["roundtrip_f32k"] = bool(np.array_equal(dec32, m))
        if cs["n"] <= 12345:
            arrays[cs["name"] + "/mask"] = np.packbits(m)
            arrays[cs["name"] + "/bitmap"] = np.packbits(bitmap)
            arrays[cs["name"] + "/witness"] = np.packbits(w)
        recs.append(rec)
        print(cs["name"], rec["ones"], rec["l"], rec["witness_len"], rec.get("roundtrip"), rec.get("roundtrip_f32k"))

    # explicit k*=2.3 filter on the survey mask (SURVEY 8c KAT)
    m = mask_for(cases[0])
    f = ivc.RationalBloomFilter(1000, 2.3)
    for i in np.nonzero(m)[0]:
        f.add_index(int(i))
    wit = [int(m[i]) for i in range(len(m)) if f.check_index(i)]
    explicit = {"size": 1000, "k": 2.3, "ones": int(m.sum()), "bits_set": int(f.bit_array.sum()),
                "witness_len": len(wit), "bitmap_sha256": sha(np.packbits(f.bit_array)),
                "witness_sha256": sha(np.packbits(np.array(wit, dtype=np.uint8)))}
    # k* sweep of BASELINE config 5 on a small mask: l = int(p*n*k/ln2)
    sweep = []
    m2 = mask_for({"n": 20000, "seed": 21, "p_gen": 0.05})
    import math
    p2 = np.sum(m2) / len(m2)
    for ks in [1.5, 2.0, 2.5, 3.0, 3.5, 4.0, 0.1, 0.7, 1.0, 7.25]:
        l2 = int(p2 * len(m2) * ks / math.log(2))
        f = ivc.RationalBloomFilter(l2, ks)
        for i in np.nonzero(m2)[0]:
            f.add_index(int(i))
        wit = [int(m2[i]) for i in range(len(m2)) if f.check_index(i)]
        sweep.append({"k": ks, "l": l2, "bitmap_sha256": sha(np.packbits(f.bit_array)),
                      "witness_len": len(wit),
                      "witness_sha256": sha(np.packbits(np.array(wit, dtype=np.uint8)))})
    dump("compress_kat.json", {"cases": recs, "explicit_k2.3": explicit,
                               "k_sweep": {"n": 20000, "seed": 21, "p_gen": 0.05, "p": float(p2).hex(), "cases": sweep}})
    np.savez_compressed(os.path.join(HERE, "compress_arrays.npz"), **arrays)


# ---------------------------------------------------------------- frame diff + payload
def synth_pair(h, w, seed, p_change, dtype=np.uint8):
    rng = np.random.default_rng(seed)
    hi = 256 if dtype == np.uint8 else 65536
    prev = rng.integers(0, hi, (h, w, 3)).astype(dtype)
    curr = prev.copy()
    ch = rng.random((h, w)) < p_change
    delta = 64 if dtype == np.uint8 else 16384
    curr[ch] = (curr[ch].astype(np.int64) + delta) % hi
    return prev, curr


def gen_frames():
    vfc = refshim.make_vfc(ivc, use_direct_yuv=True)
    recs = []
    arrays = {}
    for name, h, w, seed, pc, dt, thr in [
        ("cfg1_64x64", 64, 64, 1234, 0.05, np.uint8, 3.0),
        ("u8_thr0", 48, 80, 31, 0.10, np.uint8, 0.0),
        ("u8_thr_frac", 48, 80, 32, 0.10, np.uint8, 63.5),
        ("u8_thr64", 48, 80, 32, 0.10, np.uint8, 64.0),
        ("u8_thr_neg", 16, 16, 33, 0.10, np.uint8, -1.0),
        ("u8_thr_big", 16, 16, 33, 0.10, np.uint8, 300.0),
        ("u16_wrap", 40, 72, 34, 0.05, np.uint16, 3.0),
        ("u16_wrap_thr30000", 40, 72, 35, 0.20, np.uint16, 30000.0),
        ("u8_360p", 360, 640, 36, 0.05, np.uint8, 3.0),
    ]:
        prev, curr = synth_pair(h, w, seed, pc, dt)
        if dt == np.uint16:   # force int16-wrap corner cases (SURVEY hard part 2)
            prev[0, 0, 0], curr[0, 0, 0] = 0, 40000
            prev[0, 1, 0], curr[0, 1, 0] = 65535, 0
            prev[0, 2, 0], curr[0, 2, 0] = 0, 32768
            prev[0, 3, 0], curr[0, 3, 0] = 32768, 0
            prev[0, 4, 0], curr[0, 4, 0] = 32767, 65535
        pf = vfc_wrap(prev)
        cf = vfc_wrap(curr)
        mask, changed, dens = vfc._calculate_frame_diff(pf, cf, threshold=thr)
        rec = {"name": name, "h": h, "w": w, "seed": seed, "p_change": pc, "dtype": np.dtype(dt).name,
               "threshold": thr, "ones": int(mask.sum()), "density": float(dens).hex(),
               "mask_sha256": sha(np.packbits(mask.reshape(-1))), "changed_len": int(len(changed)),
               "changed_sha256": sha(changed)}
        if dt == np.uint16:
            rec["wrap_mask_head"] = [int(x) for x in mask[0, :5]]
        if h * w <= 4096:
            # full inter-frame payload of the reference (ivc:911-967) and its decode + apply
            payload, ratio = vfc._compress_frame_differences(mask, changed)
            dmask, dchanged = vfc._decompress_frame_differences(payload, curr.shape)
            recon = vfc._apply_frame_diff(pf, dmask, dchanged)
            arrays[name + "/payload"] = np.frombuffer(payload, dtype=np.uint8)
            rec.update(payload_len=len(payload), payload_sha256=hashlib.sha256(payload).hexdigest(),
                       decoded_mask_equal=bool(np.array_equal(dmask, mask)),
                       recon_equal_curr=bool(np.array_equal(np.asarray(recon.data if hasattr(recon, "data") else recon), curr)),
                       recon_sha256=sha(np.asarray(recon.data if hasattr(recon, "data") else recon)))
        recs.append(rec)
        print(name, rec["ones"], rec.get("payload_len"), rec.get("decoded_mask_equal"), rec.get("recon_equal_curr"))
    dump("frames_kat.json", {"cases": recs})
    np.savez_compressed(os.path.join(HERE, "frames_arrays.npz"), **arrays)


def vfc_wrap(frame):
    return fvc.FixedVideoCompressor(verbose=False).add_yuv_info_to_frame(frame)


# ---------------------------------------------------------------- string API (rbf / bc seeds)
def gen_strings():
    rng = random.Random(42)
    items = ["".join(rng.choices("abcdefghijklmnopqrstuvwxyz", k=10)) for _ in range(400)]
    probes = ["".join(rng.choices("abcdefghijklmnopqrstuvwxyz", k=10)) for _ in range(600)] + items[:50]
    long_items = ["x" * n + str(n) for n in (0, 1, 31, 32, 33, 63, 64, 65, 200)]
    recs = []
    for m, k in [(4000, 2.3), (5000, 6.93), (3000, 0.4), (4001, 3.0)]:
        f = rbf.RationalBloomFilter(m, k)
        for it in items + long_items:
            f.add(it)
        res = [bool(f.contains(p)) for p in probes + long_items]
        recs.append({"kind": "rational", "m": m, "k": k, "ceil_k": f.ceil_k, "bits_set": int(sum(f.bit_array)),
                     "bitmap_sha256": sha(np.packbits(np.array(f.bit_array, dtype=np.uint8))),
                     "contains_sha256": sha(np.packbits(np.array(res, dtype=np.uint8))), "contains_true": int(sum(res))})
    for m, k in [(4000, 3), (5000, 7), (100, 1)]:
        f = rbf.StandardBloomFilter(m, k)
        for it in items + long_items:
            f.add(it)
        res = [bool(f.contains(p)) for p in probes + long_items]
        recs.append({"kind": "standard", "m": m, "k": k, "bits_set": int(sum(f.bit_array)),
                     "bitmap_sha256": sha(np.packbits(np.array(f.bit_array, dtype=np.uint8))),
                     "contains_sha256": sha(np.packbits(np.array(res, dtype=np.uint8))), "contains_true": int(sum(res))})
    # bc nested filter (seeds 0/1/999, int items) via bc.BloomFilterCompressor.compress
    m = mask_for({"n": 5000, "seed": 17, "p_gen": 0.1})
    bitmap, witness, p, n, ratio = bc.BloomFilterCompressor().compress(m)
    recs.append({"kind": "bc_compress", "n": 5000, "seed": 17, "p_gen": 0.1, "l": int(len(bitmap)),
                 "witness_len": len(witness), "bitmap_sha256": sha(np.packbits(bitmap)),
                 "witness_sha256": sha(np.packbits(np.array(witness, dtype=np.uint8)))})
    opt = [{"n": n, "p": p, "size": rbf.RationalBloomFilter.get_optimal_size(n, p)} for n, p in
           [(1000, 0.01), (12345, 0.001), (7, 0.5), (10 ** 6, 1e-6)]]
    hc = [{"m": m, "n": n, "k": float(rbf.RationalBloomFilter.get_optimal_hash_count(m, n)).hex(),
           "k_std": rbf.StandardBloomFilter.get_optimal_hash_count(m, n)} for m, n in
          [(9586, 1000), (100, 1000), (5000, 400), (1, 10 ** 6)]]
    dump("strings_kat.json", {"items_seed": 42, "filters": recs, "optimal_size": opt, "optimal_hash_count": hc})


# ---------------------------------------------------------------- keyframe payloads (host glue, fvc:27-74)
def gen_keyframes():
    comp = fvc.FixedVideoCompressor(verbose=False)
    arrays, recs = {}, []
    for name, shape, dt, yuv in [("bgr_u8", (24, 40, 3), np.uint8, False), ("yuv_u8", (24, 40, 3), np.uint8, True),
                                 ("gray_u8", (16, 16), np.uint8, False), ("yuv_u16", (8, 12, 3), np.uint16, False)]:
        rng = np.random.default_rng(77)
        hi = 256 if dt == np.uint8 else 65536
        f = (rng.integers(0, hi, shape) // 16 * 16).astype(dt)
        fr = comp.add_yuv_info_to_frame(f) if yuv else f
        payload = comp.compress_frame(fr)
        arrays[name + "/frame"] = f
        arrays[name + "/payload"] = np.frombuffer(payload, dtype=np.uint8)
        recs.append({"name": name, "yuv": yuv, "payload_sha256": hashlib.sha256(payload).hexdigest()})
    dump("keyframe_kat.json", {"cases": recs})
    np.savez_compressed(os.path.join(HERE, "keyframe_arrays.npz"), **arrays)


# ---------------------------------------------------------------- adaptive threshold (ivc:727-766), SURVEY 8f N3
def gen_adaptive():
    recs = []
    for name, h, w, seed, pc, dt, noise_amp in [("u8_smooth", 72, 96, 61, 0.05, np.uint8, 2), ("u8_noisy", 72, 96, 62, 0.05, np.uint8, 40),
                                                  ("u8_edge", 7, 9, 63, 0.3, np.uint8, 10), ("u16", 40, 56, 64, 0.05, np.uint16, 300),
                                                  ("u8_tiny", 64, 80, 65, 0.002, np.uint8, 1), ("u8_mid", 64, 80, 66, 0.004, np.uint8, 2)]:
        rng = np.random.default_rng(seed)
        hi = 256 if dt == np.uint8 else 65536
        yy, xx = np.mgrid[0:h, 0:w]
        base = ((yy * 5 + xx * 3) * (hi // 512) % (hi - 2 * noise_amp - 1)).astype(np.int64)
        if name in ("u8_tiny", "u8_mid"):
            base = ((yy + xx) // 4 + 20).astype(np.int64)      # no wrap edges: the noise estimate stays below the clamp
        prev = np.stack([base + rng.integers(0, noise_amp + 1, (h, w)) for _ in range(3)], axis=-1).astype(dt)
        curr = prev.copy()
        ch = rng.random((h, w)) < pc
        delta = {"u8_tiny": 20, "u8_mid": 30}.get(name, hi // 4)
        curr[ch] = (curr[ch].astype(np.int64) + delta) % hi
        vfc = refshim.make_vfc(ivc, use_direct_yuv=True)
        y = curr[:, :, 0].copy()
        nl = vfc._estimate_noise_level(y)
        thr = vfc._adaptive_diff_threshold(y)
        mask, changed, dens = vfc._calculate_frame_diff(vfc_wrap(prev), vfc_wrap(curr), threshold=None)
        import cv2
        recs.append({"name": name, "h": h, "w": w, "seed": seed, "p_change": pc, "dtype": np.dtype(dt).name, "noise_amp": noise_amp, "delta": int(delta),
                     "noise_level": float(nl).hex(), "noise_level_type": type(nl).__name__, "threshold": float(thr).hex(),
                     "median_sha256": sha(cv2.medianBlur(y, 5)), "ones": int(mask.sum()), "mask_sha256": sha(np.packbits(mask.reshape(-1)))})
        print(name, nl, thr, int(mask.sum()))
    dump("adaptive_kat.json", {"cases": recs})


def gen_gray():
    """The reference's non-YUV colour branch: cv2.COLOR_BGR2GRAY before the diff (ivc:792-795), fixed and adaptive thresholds."""
    import cv2
    recs = []
    for name, h, w, seed, pc, dt, thr in [("bgr_u8_thr3", 48, 80, 71, 0.10, np.uint8, 3.0), ("bgr_u8_thr0", 37, 53, 72, 0.10, np.uint8, 0.0),
                                           ("bgr_u8_thr20", 64, 96, 73, 0.30, np.uint8, 20.5), ("bgr_u16_thr3", 40, 72, 74, 0.05, np.uint16, 3.0),
                                           ("bgr_u16_thr9000", 40, 72, 75, 0.20, np.uint16, 9000.0), ("bgr_u8_360p", 360, 640, 76, 0.05, np.uint8, 3.0),
                                           ("bgr_u8_adaptive", 72, 96, 77, 0.05, np.uint8, None), ("bgr_u16_adaptive", 40, 56, 78, 0.05, np.uint16, None)]:
        prev, curr = synth_pair(h, w, seed, pc, dt)
        if thr is None:                                   # smooth content so that the adaptive threshold is not clamped
            rng = np.random.default_rng(seed)
            hi = 256 if dt == np.uint8 else 65536
            yy, xx = np.mgrid[0:h, 0:w]
            base = ((yy + xx) // 4 + 20).astype(np.int64) * (1 if dt == np.uint8 else 200)
            prev = np.stack([base + rng.integers(0, 3, (h, w)) for _ in range(3)], axis=-1).astype(dt)
            curr = prev.copy()
            ch = rng.random((h, w)) < pc
            curr[ch] = (curr[ch].astype(np.int64) + hi // 4) % hi
        # single-channel changes that move the gray value by exactly the rounding boundary
        curr[0, 0] = prev[0, 0]; curr[0, 0, 0] = (int(prev[0, 0, 0]) + 9) % (256 if dt == np.uint8 else 65536)
        vfc = refshim.make_vfc(ivc, use_direct_yuv=False)
        mask, changed, dens = vfc._calculate_frame_diff(prev, curr, threshold=thr)
        g = cv2.cvtColor(curr, cv2.COLOR_BGR2GRAY)
        rec = {"name": name, "h": h, "w": w, "seed": seed, "p_change": pc, "dtype": np.dtype(dt).name, "threshold": thr,
               "ones": int(mask.sum()), "density": float(dens).hex(), "mask_sha256": sha(np.packbits(mask.reshape(-1))),
               "changed_len": int(len(changed)), "changed_dtype": changed.dtype.name, "changed_sha256": sha(changed),
               "gray_curr_sha256": sha(g)}
        if thr is None:
            rec["adaptive_threshold"] = float(vfc._adaptive_diff_threshold(g)).hex()
        recs.append(rec)
        print(name, rec["ones"], rec["changed_len"])
    # exhaustive corner sweep of the fixed-point conversion: every (b, g, r) with two channels on a coarse grid
    grid = np.array(sorted(set(list(range(0, 256, 5)) + [1, 2, 254, 255])), dtype=np.uint8)
    bb, gg, rr = np.meshgrid(grid, grid, grid, indexing="ij")
    cube = np.stack([bb, gg, rr], axis=-1).reshape(1, -1, 3)
    cube16 = (cube.astype(np.uint16) * 257)
    dump("gray_kat.json", {"cases": recs, "cube_u8_sha256": sha(cv2.cvtColor(cube, cv2.COLOR_BGR2GRAY)),
                           "cube_u16_sha256": sha(cv2.cvtColor(cube16, cv2.COLOR_BGR2GRAY)), "cv2_version": cv2.__version__})


def enc(a: np.ndarray) -> dict:
    """An array as {"shape", "dtype", "hex"} (read back by tests/test_gpu_frame_api.py)."""
    a = np.ascontiguousarray(a)
    return {"shape": list(a.shape), "dtype": a.dtype.name, "hex": a.tobytes().hex()}


def outcome(fn):
    """-> ("ok", result) or ("error", the exception's type name)."""
    try:
        return "ok", fn()
    except Exception as e:                                # the reference's own exception is the recorded outcome
        return "error", type(e).__name__


def gen_frame_api():
    """VideoFrameCompressor's per-frame API (ivc:727-909) at its mask value, value count, layout and adaptive-threshold edges:
    inputs, and the SHA-256 of every result or the name of the exception the reference raises."""
    import cv2
    rng = np.random.default_rng(2026)
    h, w = 6, 7
    apply_cases, diff_cases, noise_cases = [], [], []

    def base_for(shape, dt):
        return rng.integers(0, 256 if dt == np.uint8 else 65536, shape).astype(dt)

    # mask values: only entries == 1 are applied (ivc:869)
    masks = {}
    m = np.zeros((h, w), np.uint8); m[1, 1] = 1; m[3, 4] = 1; m[5, 6] = 1; masks["bin"] = m
    m = np.zeros((h, w), np.uint8); m[1, 1] = 1; m[2, 2] = 255; masks["u8_255"] = m
    m = np.zeros((h, w), np.uint8); m[1, 1] = 1; m[4, 0] = 2; m[0, 6] = 1; masks["u8_2"] = m
    m = np.zeros((h, w), np.int16); m[1, 1] = 1; m[2, 2] = 257; m[3, 3] = -1; masks["i16"] = m
    m = np.zeros((h, w), np.float64); m[1, 1] = 1.0; m[2, 2] = 0.5; m[5, 0] = 1.0; masks["f64"] = m
    m = np.zeros((h, w), bool); m[0, 0] = True; m[2, 3] = True; masks["bool"] = m
    masks["empty"] = np.zeros((h, w), np.uint8)

    def counts(n):                                        # value counts in pixels: exact, short, long, none, one
        return {"exact": n, "short": n - 1, "long": n + 1, "zero": 0, "one": 1}

    layouts = [("g8", (h, w), np.uint8, False), ("g16", (h, w), np.uint16, False), ("g1", (h, w, 1), np.uint8, False),
               ("c8", (h, w, 3), np.uint8, False), ("c16", (h, w, 3), np.uint16, False), ("c4", (h, w, 4), np.uint8, False),
               ("yuv8", (h, w, 3), np.uint8, True), ("yuv16", (h, w, 3), np.uint16, True)]
    picks = [("g8", "bin", ["exact", "short", "long", "zero", "one"]), ("g8", "u8_255", ["exact", "long"]),
             ("g8", "empty", ["long", "zero"]), ("g16", "i16", ["exact", "one"]), ("g16", "f64", ["exact", "long"]),
             ("g1", "bin", ["exact", "short", "one"]), ("g1", "u8_2", ["exact"]), ("c8", "bin", ["exact", "short", "one"]),
             ("c8", "u8_255", ["exact", "long"]), ("c16", "i16", ["exact"]), ("c16", "bool", ["exact", "zero"]),
             ("c4", "u8_2", ["exact", "short"]), ("yuv8", "bin", ["exact", "short"]), ("yuv8", "f64", ["exact"]),
             ("yuv16", "bin", ["exact"]), ("yuv16", "u8_255", ["long"])]
    lay = {name: (shape, dt, yuv) for name, shape, dt, yuv in layouts}
    for lname, mname, cnames in picks:
        shape, dt, yuv = lay[lname]
        base = base_for(shape, dt)
        mask = masks[mname]
        if len(shape) == 3 and shape[2] == 1:
            mask = mask[:, :, None]                       # the (h, w, 1) mask _calculate_frame_diff returns for such frames
        ch = shape[2] if len(shape) == 3 and shape[2] > 1 else 1
        n = int(np.sum(mask == 1))
        for cname in cnames:
            k = counts(n)[cname]
            vdt = np.uint8 if yuv else dt                 # YUV values are u8 (ivc:825)
            vals = rng.integers(0, 256 if vdt == np.uint8 else 65536, max(0, k) * ch).astype(vdt)
            vfc = refshim.make_vfc(ivc, use_direct_yuv=yuv)
            frame = vfc_wrap(base.copy()) if yuv else base.copy()
            status, res = outcome(lambda: vfc._apply_frame_diff(frame, mask, vals))
            rec = {"name": f"{lname}/{mname}/{cname}", "use_direct_yuv": yuv, "yuv": yuv, "base": enc(base), "mask": enc(mask),
                   "values": enc(vals)}
            if status == "error":
                rec["error"] = res
            else:
                d = np.asarray(res.data if hasattr(res, "yuv_info") else res)
                rec.update(result_shape=list(d.shape), result_dtype=d.dtype.name, result_sha256=sha(d))
                if yuv:
                    rec["planes_sha256"] = [sha(res.yuv_info[p]) for p in ("y_plane", "u_plane", "v_plane")]
                rec["base_unchanged"] = bool(np.array_equal(np.asarray(frame.data if yuv else frame), base))
            apply_cases.append(rec)

    # _calculate_frame_diff across its branches (ivc:768-847)
    def pair(shape, dt, p=0.3):
        prev = base_for(shape, dt)
        curr = prev.copy()
        sel = rng.random(shape[:2]) < p
        hi = 256 if dt == np.uint8 else 65536
        curr[sel] = (curr[sel].astype(np.int64) + rng.integers(1, 8, curr[sel].shape)) % hi
        return prev, curr

    for name, shape, dt, yuv, thr in [("yuv8_thr3", (9, 11, 3), np.uint8, True, 3.0), ("yuv16_thr3.5", (9, 11, 3), np.uint16, True, 3.5),
                                      ("arr3_direct_thr0", (9, 11, 3), np.uint8, "array", 0.0), ("bgr8_thr3", (9, 11, 3), np.uint8, False, 3.0),
                                      ("bgr16_thr3.5", (9, 11, 3), np.uint16, False, 3.5), ("g8_thr0", (9, 11), np.uint8, False, 0.0),
                                      ("g16_none", (12, 17), np.uint16, False, None), ("g1_thr3", (9, 11, 1), np.uint8, False, 3.0),
                                      ("g1_none", (9, 11, 1), np.uint8, False, None), ("g1_square_none", (6, 6, 1), np.uint8, False, None),
                                      ("yuv8_none", (12, 17, 3), np.uint8, True, None), ("bgr8_none", (12, 17, 3), np.uint8, False, None)]:
        prev, curr = pair(shape, dt)
        vfc = refshim.make_vfc(ivc, use_direct_yuv=bool(yuv))
        pf, cf = (vfc_wrap(prev), vfc_wrap(curr)) if yuv is True else (prev, curr)
        status, res = outcome(lambda: vfc._calculate_frame_diff(pf, cf, threshold=thr))
        rec = {"name": name, "use_direct_yuv": bool(yuv), "yuv": yuv is True, "threshold": thr, "prev": enc(prev), "curr": enc(curr)}
        if status == "error":
            rec["error"] = res
        else:
            mask, changed, dens = res
            rec.update(mask_shape=list(mask.shape), mask_sha256=sha(mask.astype(np.uint8)), changed_dtype=changed.dtype.name,
                       changed_sha256=sha(changed), changed_len=int(len(changed)), density=float(dens).hex())
        diff_cases.append(rec)

    # noise level and adaptive threshold where cv2.medianBlur is the reference's median (ivc:727-766)
    for name, plane, tol in [("u8_random", base_for((9, 11), np.uint8), 10.0), ("u16_high", (base_for((8, 13), np.uint16) | 0x8000), 0.001),
                             ("u8_ties", rng.choice(np.array([0, 128, 255], np.uint8), (16, 33)), 0.05),
                             ("u16_ties", rng.choice(np.array([0, 32767, 32768, 65535], np.uint16), (17, 31)), 0.0001),
                             ("u8_flat", np.full((7, 9), 200, np.uint8), 10.0), ("u8_1x1", np.array([[77]], np.uint8), 10.0)]:
        vfc = refshim.make_vfc(ivc, noise_tolerance=tol)
        nl = vfc._estimate_noise_level(plane)
        thr = vfc._adaptive_diff_threshold(plane)
        noise_cases.append({"name": name, "plane": enc(plane), "noise_tolerance": tol, "noise_level": float(nl).hex(),
                            "noise_level_type": type(nl).__name__, "threshold": float(thr).hex(),
                            "median_sha256": sha(cv2.medianBlur(plane, 5))})
    dump("frame_api_kat.json", {"apply": apply_cases, "diff": diff_cases, "noise": noise_cases, "cv2_version": cv2.__version__})


if __name__ == "__main__":
    if "--gray-only" in sys.argv:
        gen_gray()
        sys.exit(0)
    if "--frame-api-only" in sys.argv:
        gen_frame_api()
        sys.exit(0)
    gen_gray()
    gen_xxh64()
    gen_filter()
    gen_threshold()
    gen_params()
    gen_compress()
    gen_frames()
    gen_strings()
    gen_keyframes()
    gen_adaptive()
    gen_frame_api()
