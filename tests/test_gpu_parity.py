"""GPU parity tests (-m gpu): the CUDA path, called through the C ABI / the drop-in classes,
against (i) the golden fixtures generated from the real reference and (ii) the oracle on the
same seeded inputs.  Integer / bit work: every comparison is bit-exact."""
import math
import os
import random

import numpy as np
import pytest

from tests.util import golden_json, golden_npz, golden_pair, mask_for, sha, synth_pair, synth_stream

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    import new_bloom_filter_repo_b200 as p
    info = p._cabi.device_info()
    assert info["cc"] == (9, 0), info
    return p


@pytest.fixture(scope="module")
def co():
    from oracle import c_oracle
    c_oracle.build()
    return c_oracle


# ------------------------------------------------------------------ filter (ivc:39-138)
def test_index_filter_against_golden(pkg):
    g = golden_json("filter_kat.json")
    for rec in g["filters"]:
        f = pkg.IndexRationalBloomFilter(rec["size"], rec["k"])
        assert f.floor_k == rec["floor_k"] and float(f.p_activation).hex() == rec["p_activation"]
        if rec["size"] > 5_000_000:          # bit_array of 2^31 bytes is not worth materialising
            for it, probes in zip(rec["items"][:4], rec["probes"][:4]):
                assert [f._get_hash_indices(it, i) for i in range(f.floor_k + 1)] == probes
            continue
        for it, probes, act in zip(rec["items"], rec["probes"], rec["activation"]):
            ff = pkg.IndexRationalBloomFilter(rec["size"], rec["k"])
            ff.add_index(it)
            expect = set(probes[:rec["floor_k"]]) | ({probes[rec["floor_k"]]} if act else set())
            got = set(np.nonzero(ff.bit_array)[0].tolist())
            assert got == expect, (rec["size"], rec["k"], it)
            assert ff.check_index(it)
            assert [ff._get_hash_indices(it, i) for i in range(ff.floor_k + 1)] == probes
            assert ff._determine_activation(it) == act


def test_index_filter_survey_kat(pkg):
    """SURVEY.md 8c: mask inserted into RationalBloomFilter(1000, 2.3), all 4096 queried."""
    g = golden_json("compress_kat.json")
    e = g["explicit_k2.3"]
    m = mask_for(g["cases"][0])
    f = pkg.IndexRationalBloomFilter(1000, 2.3)
    f.add_indices(np.nonzero(m)[0])
    bits = f.bit_array
    assert int(bits.sum()) == e["bits_set"] == 382
    assert sha(np.packbits(bits)) == e["bitmap_sha256"]
    passed = f.check_indices(np.arange(4096))
    wit = m[passed]
    assert len(wit) == e["witness_len"] == 700 and sha(np.packbits(wit)) == e["witness_sha256"]
    # bit_array assignment (ivc:290)
    f2 = pkg.IndexRationalBloomFilter(1000, 2.3)
    f2.bit_array = bits
    assert np.array_equal(f2.check_indices(np.arange(4096)), passed)


# ------------------------------------------------------------------ BloomFilterCompressor (ivc:140-307)
def test_compress_against_golden(pkg):
    g = golden_json("compress_kat.json")
    arrays = golden_npz("compress_arrays.npz")
    comp = pkg.BloomFilterCompressor()
    for rec in g["cases"]:
        m = mask_for(rec)
        bitmap, witness, p, n, ratio = comp.compress(m)
        assert float(p).hex() == rec["p"] and n == rec["n"]
        if rec["raw"]:
            assert witness == [] and bitmap is m and ratio == 1.0
            continue
        w = np.array(witness, dtype=np.uint8)
        assert len(bitmap) == rec["bitmap_len"] and len(w) == rec["witness_len"], rec["name"]
        assert sha(np.packbits(bitmap)) == rec["bitmap_sha256"], rec["name"]
        assert sha(np.packbits(w)) == rec["witness_sha256"], rec["name"]
        assert float(ratio).hex() == rec["ratio"]
        assert float(comp.last_info.k).hex() == rec["k"]
        if rec["name"] + "/bitmap" in arrays:
            assert np.array_equal(np.packbits(bitmap), arrays[rec["name"] + "/bitmap"])
        k, l = comp._calculate_optimal_params(n, p)
        assert (float(k).hex(), l) == (rec["k"], rec["l"])
        dec = comp.decompress(bitmap, witness, n, k)
        assert np.array_equal(dec, m)
        # the reference's own decode uses k rounded to float32 (ivc:938/986): replicate, do not fix
        k32 = float.fromhex(rec["k_f32"])
        dec32 = comp.decompress(bitmap, witness + [0] * 64, n, k32)
        assert sha(np.packbits(dec32)) == rec["decoded_f32k_sha256"], rec["name"]


def test_compress_k_sweep_and_seed_variants(pkg, co):
    g = golden_json("compress_kat.json")
    sw = g["k_sweep"]
    m2 = mask_for(sw)
    p2 = np.sum(m2) / len(m2)
    comp = pkg.BloomFilterCompressor()
    for c in sw["cases"]:
        bitmap, witness, p, n, ratio = comp.compress(m2, k_l_override=(c["k"], c["l"]))
        assert sha(np.packbits(bitmap)) == c["bitmap_sha256"], c
        assert len(witness) == c["witness_len"]
        assert sha(np.packbits(np.array(witness, dtype=np.uint8))) == c["witness_sha256"]
    s = golden_json("strings_kat.json")
    rec = [r for r in s["filters"] if r["kind"] == "bc_compress"][0]
    m = mask_for(rec)
    bitmap, witness, *_ = pkg.BloomFilterCompressor(seeds=pkg._cabi.BC_SEEDS).compress(m)
    assert len(bitmap) == rec["l"] and sha(np.packbits(bitmap)) == rec["bitmap_sha256"]
    assert sha(np.packbits(np.array(witness, dtype=np.uint8))) == rec["witness_sha256"]


@pytest.mark.parametrize("n,p_gen,seed", [(1, 0.5, 1), (33, 0.2, 2), (99, 0.1, 3), (100, 0.1, 4), (101, 0.1, 5), (3199, 0.05, 6),
                                          (3200, 0.05, 7), (3201, 0.05, 8), (65536, 0.003, 9), (99999, 0.12, 10),
                                          (100001, 0.2, 11), (1000003, 0.05, 12), (2073600, 0.0499, 13), (10 ** 7 + 7, 0.01, 14)])
def test_compress_vs_oracle_ragged_sizes(pkg, co, n, p_gen, seed):
    m = mask_for({"n": n, "p_gen": p_gen, "seed": seed})
    ob, ow, op, on, oratio, ok, ol = co.compress(m)
    bitmap, witness, p, nn, ratio = pkg.BloomFilterCompressor().compress(m)
    assert float(p) == op and nn == on
    if ok == 0:
        assert witness == [] and np.array_equal(bitmap, m)
        return
    assert len(bitmap) == ol and np.array_equal(bitmap, ob)
    assert np.array_equal(np.array(witness, dtype=np.uint8), ow)
    assert ratio == oratio
    dec = pkg.BloomFilterCompressor().decompress(bitmap, witness, n, ok)
    assert np.array_equal(dec, m)


@pytest.mark.parametrize("variant", [0, 1, 5, 6])
@pytest.mark.parametrize("n,p_gen,seed", [(101, 0.1, 21), (99999, 0.12, 22), (2073600, 0.0499, 23), (8294400, 0.03, 24),
                                          (8294400, 0.19, 25), (33177600, 0.08, 26), (33177600, 0.2, 27)])
def test_query_kernel_variants_vs_oracle(pkg, co, variant, n, p_gen, seed):
    """Every K3 formulation (per-lane, staged rings, decade / half-decade tiles with carried batches) gives the oracle's bitmap
    and witness bit for bit; the last sizes have l > 2^23 (the tile kernel switches to half-decade tiles with 24-bit records)
    and l > 2^24 (rings)."""
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    m = mask_for({"n": n, "p_gen": p_gen, "seed": seed})
    ob, ow, op, on, oratio, ok, ol = co.compress(m)
    assert ok > 0
    pkg._cabi.check(L.rbf_set_option(ctx, b"query_variant", variant), ctx)
    try:
        comp = pkg.BloomFilterCompressor()
        bitmap, witness, p, nn, ratio = comp.compress(m)
        assert len(bitmap) == ol and np.array_equal(bitmap, ob)
        assert np.array_equal(np.array(witness, dtype=np.uint8), ow)
        assert np.array_equal(comp.decompress(bitmap, witness, n, ok), m)
    finally:
        L.rbf_set_option(ctx, b"query_variant", 5)


@pytest.mark.parametrize("variant", [0, 1, 5, 6])
@pytest.mark.parametrize("k,l", [(3.5, 16), (2.2, 5), (3.0, 64), (1.0, 7), (2.999, 2), (3.4, 40000)])
def test_query_saturated_filter_and_empty_regions(pkg, co, variant, k, l):
    """A tiny (saturated) Bloom array makes every position survive every stage -- the survivor buffers and the stage-C ring
    of the compacting kernels run full -- and the second half of the mask is empty, so whole slabs have no member to skip."""
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    n = 150000
    rng = np.random.default_rng(77)
    m = np.zeros(n, dtype=np.uint8)
    m[: n // 3] = rng.random(n // 3) < 0.15
    ob, ow, *_ = co.compress(m, k_l_override=(k, l))
    pkg._cabi.check(L.rbf_set_option(ctx, b"query_variant", variant), ctx)
    try:
        comp = pkg.BloomFilterCompressor()
        bitmap, witness, p, nn, ratio = comp.compress(m, k_l_override=(k, l))
        assert len(bitmap) == l and np.array_equal(bitmap, ob)
        assert np.array_equal(np.array(witness, dtype=np.uint8), ow)
        assert np.array_equal(comp.decompress(bitmap, witness, n, k), m)
    finally:
        L.rbf_set_option(ctx, b"query_variant", 5)


@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("n,p_gen,seed,kl", [(101, 0.1, 31, None), (99999, 0.12, 32, None), (8294400, 0.05, 33, None), (8294400, 0.31, 34, None),
                                             (33177600, 0.05, 35, None), (150000, 0.3, 36, (3.5, 16)), (2073600, 0.05, 37, (2.0, 2 ** 20)),
                                             (640000, 0.0004, 38, None)])
def test_insert_kernel_variants_vs_oracle(pkg, co, variant, n, p_gen, seed, kl):
    """K2 per-lane (0) and warp-compacted (1): the same bit array as the oracle -- dense slabs that need several list rounds
    (p = 0.31), power-of-two and saturated filters, nearly empty masks, 4K and 8K sizes."""
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    m = mask_for({"n": n, "p_gen": p_gen, "seed": seed})
    ob, ow, op, on, oratio, ok, ol = co.compress(m, k_l_override=kl)
    assert ok > 0
    pkg._cabi.check(L.rbf_set_option(ctx, b"insert_variant", variant), ctx)
    try:
        comp = pkg.BloomFilterCompressor()
        bitmap, witness, p, nn, ratio = comp.compress(m, k_l_override=kl)
        assert len(bitmap) == ol and np.array_equal(bitmap, ob)
        assert np.array_equal(np.array(witness, dtype=np.uint8), ow)
    finally:
        L.rbf_set_option(ctx, b"insert_variant", 1)


def test_decompress_short_witness_raises(pkg):
    m = mask_for({"n": 5000, "p_gen": 0.05, "seed": 3})
    comp = pkg.BloomFilterCompressor()
    bitmap, witness, p, n, _ = comp.compress(m)
    k, l = comp._calculate_optimal_params(n, p)
    with pytest.raises(IndexError):
        comp.decompress(bitmap, witness[:-5], n, k)
    assert comp.decompress(bitmap, [], n, k) is bitmap       # ivc:282-284


# ------------------------------------------------------------------ frame diff (ivc:768-847) + payload (ivc:911-1027)
def test_frame_diff_against_golden(pkg, co):
    g = golden_json("frames_kat.json")
    arrays = golden_npz("frames_arrays.npz")
    vfc = pkg.VideoFrameCompressor(use_direct_yuv=True)
    for rec in g["cases"]:
        prev, curr = golden_pair(rec)
        pf, cf = pkg.YUVFrame(prev), pkg.YUVFrame(curr)
        mask, changed, dens = vfc._calculate_frame_diff(pf, cf, threshold=rec["threshold"])
        assert mask.shape == (rec["h"], rec["w"]) and mask.dtype == np.uint8
        assert int(mask.sum()) == rec["ones"], rec["name"]
        assert sha(np.packbits(mask.reshape(-1))) == rec["mask_sha256"], rec["name"]
        assert float(dens).hex() == rec["density"]
        assert len(changed) == rec["changed_len"] and sha(changed) == rec["changed_sha256"]
        if "wrap_mask_head" in rec:
            assert [int(x) for x in mask[0, :5]] == rec["wrap_mask_head"]
        if "payload_len" in rec:
            payload, ratio = vfc._compress_frame_differences(mask, changed)
            assert payload == arrays[rec["name"] + "/payload"].tobytes(), rec["name"]
            dmask, dchanged = vfc._decompress_frame_differences(payload, curr.shape)
            assert np.array_equal(dmask, mask) == rec["decoded_mask_equal"]
            recon = vfc._apply_frame_diff(pf, dmask, dchanged)
            assert sha(recon.data) == rec["recon_sha256"]


@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("shape,dtype,thr", [((64, 64), np.uint8, 3.0), ((37, 53), np.uint8, 0.0), ((1080, 1920), np.uint8, 3.0),
                                             ((130, 4099), np.uint8, 10.5), ((270, 480), np.uint16, 3.0), ((33, 65), np.uint16, 20000.0),
                                             ((2160, 3840), np.uint8, 3.0)])
def test_threshold_kernel_variants_vs_oracle(pkg, co, variant, shape, dtype, thr):
    """K1 with vectorised loads (0) and with the TMA bulk-copy ring (1): same mask, same counts."""
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    prev, curr = synth_pair(shape[0], shape[1], 99, 0.05, dtype)
    curr[0, 0, 1] ^= 1          # chroma-only change: not in the Y mask, counted as residual
    omask, oones = co.frame_diff_mask(prev, curr, thr)
    st = pkg.FrameStream(shape[0], shape[1], 3, dtype, max_frames=2, max_pairs=1, k1_only=True)
    st.upload(np.stack([prev, curr]))
    pkg._cabi.check(L.rbf_set_option(ctx, b"k1_variant", variant), ctx)
    try:
        res = st.encode([0], [1], thr)[0]
    finally:
        L.rbf_set_option(ctx, b"k1_variant", 0)
    bm, wt, mask = st.fetch(0)
    assert res.wlen == 0 and bm.size == 0 and wt.size == 0      # k1_only: no coder outputs, never garbage lengths
    buf = np.full(16, 0xA5, dtype=np.uint8)
    with pytest.raises(pkg.RbfError):                              # the C ABI refuses a bitmap pointer after a k1_only encode
        pkg._cabi.check(L.rbf_stream_fetch_batch(st._h, 0, 1, pkg._cabi.ptr(buf), buf.size, None, 0, None, 0), ctx)
    assert (buf == 0xA5).all()                                     # and copies nothing
    assert res.ones == oones
    assert np.array_equal(mask.reshape(shape), omask)
    anyd = (prev != curr).any(axis=2)
    assert res.resid == int((anyd & (omask == 0)).sum())
    st.close()


# ------------------------------------------------------------------ batched stream (the bench path)
def _check_stream_vs_oracle(pkg, co, frames, thr, k_over=None):
    nfr, h, w = frames.shape[:3]
    st = pkg.FrameStream(h, w, 3, frames.dtype, max_frames=nfr)
    st.upload(frames)
    kw = {}
    n = h * w
    if k_over is not None:
        # BASELINE config 5: explicit k*, l = int(p*n*k/ln2)
        ones = [co.frame_diff_mask(frames[t], frames[t + 1], thr)[1] for t in range(nfr - 1)]
        kw = dict(k_override=[k_over] * (nfr - 1),
                  l_override=[int((np.uint64(o) / n) * n * k_over / math.log(2)) for o in ones])
    res = st.encode_consecutive(nfr, thr, **kw)
    for t, r in enumerate(res):
        omask, oones = co.frame_diff_mask(frames[t], frames[t + 1], thr)
        flat = omask.reshape(-1)
        over = None if k_over is None else (k_over, kw["l_override"][t])
        ob, ow, op, on, oratio, ok, ol = co.compress(flat, k_l_override=over)
        bm, wt, mask = st.fetch(t)
        assert r.ones == oones and np.array_equal(mask, flat), t
        assert r.p == op
        if ok == 0:
            assert r.raw and r.l == 0
            continue
        assert not r.raw and r.l == ol and r.k == ok and r.wlen == len(ow), (t, r, ol, len(ow))
        assert np.array_equal(bm, np.packbits(ob)), t
        assert np.array_equal(wt, np.packbits(ow)), t
    assert not st.decode_verify().any()
    st.close()
    return res


def test_stream_1080p_mixed_densities(pkg, co):
    """BASELINE config 2 shape: densities cycle through coded and raw-passthrough branches."""
    frames = synth_stream(1080, 1920, 7, 2, [0.01, 0.05, 0.15, 0.30, 0.0, 0.40])
    res = _check_stream_vs_oracle(pkg, co, frames, 3.0)
    assert [r.raw for r in res] == [False, False, False, False, True, True]


def test_stream_small_and_ragged(pkg, co):
    for (h, w) in [(64, 64), (7, 11), (100, 100), (123, 457)]:
        frames = synth_stream(h, w, 4, 5, [0.05, 0.2, 0.01])
        _check_stream_vs_oracle(pkg, co, frames, 3.0)


def test_stream_4k_full_size(pkg, co):
    """BASELINE config 3 frame size, p = 0.05: bit-exact against the C oracle."""
    frames = synth_stream(2160, 3840, 3, 3, [0.05])
    res = _check_stream_vs_oracle(pkg, co, frames, 3.0)
    assert all(1_850_000 < r.l < 1_970_000 for r in res)


def test_stream_8k_u16_k_sweep(pkg, co):
    """BASELINE config 5: 8K 16-bit samples (int16 wrap in the diff), explicit k*."""
    rng = np.random.default_rng(5)
    f0 = rng.integers(0, 65536, (4320, 7680, 3)).astype(np.uint16)
    f1 = f0.copy()
    ch = rng.random((4320, 7680)) < 0.05
    f1[ch] = (f1[ch].astype(np.int64) + 16384) % 65536
    frames = np.stack([f0, f1])
    for ks in (1.5, 3.5, 4.0):           # l(3.5) just below 2^23 (decade tiles), l(4.0) above (half-decade tiles, 24-bit records)
        _check_stream_vs_oracle(pkg, co, frames, 3.0, k_over=ks)


def test_stream_properties_at_scale(pkg):
    """Size-independent properties on a longer 4K stream: decode(encode) == mask, witness >= ones,
    no false negatives (every set mask bit passes), bitmap fill near 1/2 at the optimal k."""
    frames = synth_stream(2160, 3840, 9, 11, [0.05, 0.02, 0.1])
    st = pkg.FrameStream(2160, 3840, 3, np.uint8, max_frames=9)
    st.upload(frames)
    res = st.encode_consecutive(9, 3.0)
    assert not st.decode_verify().any()
    for t, r in enumerate(res):
        bm, wt, mask = st.fetch(t)
        assert r.ones == int(mask.sum()) and r.wlen >= r.ones
        assert int(np.unpackbits(wt)[:r.wlen].sum()) == r.ones           # witness ones == mask ones
        fill = np.unpackbits(bm)[:r.l].mean()
        assert 0.45 < fill < 0.55, fill
    st.close()


# ------------------------------------------------------------------ string API (rbf:9-214)
def test_string_filters_against_golden(pkg):
    g = golden_json("strings_kat.json")
    rng = random.Random(g["items_seed"])
    items = ["".join(rng.choices("abcdefghijklmnopqrstuvwxyz", k=10)) for _ in range(400)]
    probes = ["".join(rng.choices("abcdefghijklmnopqrstuvwxyz", k=10)) for _ in range(600)] + items[:50]
    long_items = ["x" * n + str(n) for n in (0, 1, 31, 32, 33, 63, 64, 65, 200)]
    for rec in g["filters"]:
        if rec["kind"] == "rational":
            f = pkg.RationalBloomFilter(rec["m"], rec["k"])
            assert f.ceil_k == rec["ceil_k"]
            for it in items[:5]:
                f.add(it)                       # one-item signature of the reference
            f.add_many(items[5:] + long_items)
        elif rec["kind"] == "standard":
            f = pkg.StandardBloomFilter(rec["m"], rec["k"])
            f.add_many(items + long_items)
        else:
            continue
        bits = np.array(f.bit_array, dtype=np.uint8)
        assert isinstance(f.bit_array, list)
        assert int(bits.sum()) == rec["bits_set"], rec
        assert sha(np.packbits(bits)) == rec["bitmap_sha256"], rec
        res = f.contains_many(probes + long_items).astype(np.uint8)
        assert int(res.sum()) == rec["contains_true"]
        assert sha(np.packbits(res)) == rec["contains_sha256"]
        assert f.contains(items[0]) and all(f.contains(x) for x in long_items)
    for rec in g["optimal_size"]:
        assert pkg.RationalBloomFilter.get_optimal_size(rec["n"], rec["p"]) == rec["size"]
    for rec in g["optimal_hash_count"]:
        assert float(pkg.RationalBloomFilter.get_optimal_hash_count(rec["m"], rec["n"])).hex() == rec["k"]
        assert pkg.StandardBloomFilter.get_optimal_hash_count(rec["m"], rec["n"]) == rec["k_std"]


# ------------------------------------------------------------------ ImprovedVideoCompressor (ivc:309-523)
def test_compress_video_roundtrip_gop(pkg, tmp_path):
    frames = [f for f in synth_stream(96, 160, 12, 21, [0.05, 0.2, 0.0, 0.4])]
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=5, use_direct_yuv=True)
    out = str(tmp_path / "clip.bfvc")
    stats = comp.compress_video(list(frames), output_path=out, input_color_space="YUV")
    assert set(stats) >= {"frame_count", "original_size", "compressed_size", "compression_ratio", "space_savings",
                          "compression_time", "frames_per_second", "keyframes", "keyframe_ratio", "output_path",
                          "color_space", "overall_ratio"}
    assert stats["frame_count"] == 12 and stats["keyframes"] == 3
    dec = comp.decompress_video(input_path=out)
    ver = comp.verify_lossless(frames, dec)
    assert ver["lossless"] and ver["exact_frame_matches"] == 12
    assert all(hasattr(f, "yuv_info") for f in dec)
    with pytest.raises(ValueError):
        comp.compress_video([])
    (tmp_path / "bad.bfvc").write_bytes(b"NOPE1234")
    with pytest.raises(ValueError):
        comp.decompress_video(input_path=str(tmp_path / "bad.bfvc"))


def test_compress_video_all_keyframes_matches_reference_bytes(pkg):
    g = golden_json("keyframe_kat.json")
    arr = golden_npz("keyframe_arrays.npz")
    rec = [r for r in g["cases"] if r["name"] == "bgr_u8"][0]
    f = arr["bgr_u8/frame"]
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=1)
    comp.compress_video([f, f.copy()])
    assert comp._last_compressed_frames[0] == arr["bgr_u8/payload"].tobytes()
    assert comp._last_compressed_frames[1] == arr["bgr_u8/payload"].tobytes()


def test_compress_video_reference_mode_falls_back_to_keyframe(pkg):
    frames = [f for f in synth_stream(64, 64, 4, 31, [0.05])]
    frames[2] = frames[2].copy()
    frames[2][5, 5, 2] ^= 1                       # chroma-only change: the Y mask cannot carry it (SURVEY hard part 3ii)
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=30)
    comp.inter_frame_mode = "reference"
    comp.inter_frame_threshold = 3.0
    stats = comp.compress_video(list(frames), input_color_space="YUV")
    dec = comp.decompress_video(compressed_frames=comp._last_compressed_frames)
    assert comp.verify_lossless(frames, dec)["lossless"]
    assert stats["keyframes"] >= 2


# ------------------------------------------------------------------ NCCL all-gather path (single rank here; N > 1 in bench.py)
def test_nccl_allgather_single_rank(pkg):
    import ctypes as C
    from new_bloom_filter_repo_b200 import distributed as rdist
    cabi = pkg._cabi
    frames = synth_stream(270, 480, 5, 41, [0.05, 0.1])
    st = pkg.FrameStream(270, 480, 3, np.uint8, max_frames=5)
    st.upload(frames)
    res = st.encode_consecutive(5, 3.0)
    ident = np.zeros(128, dtype=np.uint8)
    cabi.check(cabi.lib().rbf_nccl_unique_id(cabi.ptr(ident)))
    cabi.check(cabi.lib().rbf_nccl_init(cabi.ctx(), cabi.ptr(ident), 0, 1), cabi.ctx())
    slot = (max((r.l + 7) // 8 for r in res) + 15) // 16 * 16
    want = [st.fetch(t, want_mask=False)[0] for t in range(4)]
    send, recv = rdist.allgather_bitmaps(st, 4, slot, 1)
    # the exchange runs on the communication stream: an encode issued right behind it (other bit arrays) must not disturb it
    st.upload(synth_stream(270, 480, 5, 43, [0.1, 0.05]))
    res2 = st.encode_consecutive(5, 3.0)
    assert [r.ones for r in res2] != [r.ones for r in res]
    cabi.check(cabi.lib().rbf_sync(cabi.ctx()), cabi.ctx())
    got = recv.to_host().reshape(4, slot)
    for t in range(4):
        assert np.array_equal(got[t, : len(want[t])], want[t])
    send.free(); recv.free()
    cabi.check(cabi.lib().rbf_nccl_destroy(cabi.ctx()), cabi.ctx())
    st.close()


# ------------------------------------------------------------------ SURVEY 8(f) N1 / N2 on the device
@pytest.mark.parametrize("shape,dtype", [((64, 64), np.uint8), ((37, 53), np.uint8), ((270, 480), np.uint16), ((1080, 1920), np.uint8),
                                         ((2160, 3840), np.uint8), ((1080, 1920), np.uint16)])
def test_gather_changed_and_apply_diff_into_next_slot_vs_oracle(pkg, shape, dtype):
    from oracle import rbf_oracle as po
    frames = synth_stream(shape[0], shape[1], 4, 77, [0.05, 0.3, 0.0], dtype)
    st = pkg.FrameStream(shape[0], shape[1], 3, dtype, max_frames=6)
    st.upload(frames)
    res = st.encode_consecutive(4, 3.0)
    gathered = st.gather_changed()
    for t in range(3):
        mask = po.frame_diff_mask(frames[t], frames[t + 1], 3.0)
        rows, cols = np.where(mask == 1)
        expect = frames[t + 1][rows, cols, :].reshape(-1)                 # ivc:810-842, native sample type
        assert gathered[t].dtype == frames.dtype and np.array_equal(gathered[t], expect), t
        assert res[t].ones == len(rows)
        # N2: rebuild frame t+1 from frame t on the device (slot 5 <- slot 4, which holds frame t; slot 5 holds another frame)
        want = po.apply_frame_diff(frames[t], mask, expect)
        st.upload(frames[t], first=4)
        st.upload(want ^ dtype(1), first=5)
        applied = st.apply_diff(4, mask, gathered[t])
        assert applied == len(rows)
        assert np.array_equal(st.download(5), want)
        assert np.array_equal(want, frames[t + 1])                        # every channel moves together in this stream
    # value-count mismatch leaves the base frame unchanged (ivc:882): slot 1 holds frame 1 before the call
    mask = po.frame_diff_mask(frames[0], frames[1], 3.0)
    assert not np.array_equal(st.download(1), frames[0])
    assert st.apply_diff(0, mask, gathered[0][:-3]) == 0
    assert np.array_equal(st.download(1), frames[0])
    st.close()


def test_vfc_apply_frame_diff_device_path(pkg):
    vfc = pkg.VideoFrameCompressor(use_direct_yuv=True)
    prev, curr = synth_pair(96, 128, 5, 0.1, np.uint8)
    pf, cf = pkg.YUVFrame(prev), pkg.YUVFrame(curr)
    mask, changed, _ = vfc._calculate_frame_diff(pf, cf, threshold=0.0)
    rec = vfc._apply_frame_diff(pf, mask, changed)
    assert np.array_equal(rec.data, curr) and np.array_equal(rec.yuv_info["u_plane"], curr[:, :, 1])
    assert np.array_equal(pf.data, prev)                                  # the base is not modified


def test_encode_host_chunked_matches_resident(pkg, co):
    """The end-to-end call (host frames in, packed outputs out, chunked H2D overlapped with the kernels) gives the same
    bytes as the device-resident encode, across chunk boundaries."""
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    frames = synth_stream(120, 160, 11, 91, [0.05, 0.2, 0.0, 0.4, 0.01])
    st = pkg.FrameStream(120, 160, 3, np.uint8, max_frames=11)
    st.upload(frames)
    ref = st.encode_consecutive(11, 3.0)
    want = [st.fetch(t, want_mask=False)[:2] for t in range(10)]
    slot_b = (max(r.l for r in ref) + 7) // 8 + 16
    slot_w = (max(r.wlen for r in ref) + 7) // 8 + 16
    for chunk in (2, 3, 32):
        pkg._cabi.check(L.rbf_set_option(ctx, b"host_chunk_frames", chunk), ctx)
        ob = np.zeros((10, slot_b), np.uint8); ow = np.zeros((10, slot_w), np.uint8)
        res = st.encode_host(frames, 3.0, bitmap_slot=slot_b, witness_slot=slot_w, out_bitmaps=ob, out_witness=ow)
        for t in range(10):
            assert (res[t].raw, res[t].l, res[t].wlen, res[t].ones, res[t].k) == (ref[t].raw, ref[t].l, ref[t].wlen, ref[t].ones, ref[t].k)
            if not res[t].raw:
                assert np.array_equal(ob[t, : len(want[t][0])], want[t][0]) and np.array_equal(ow[t, : len(want[t][1])], want[t][1])
        assert not st.decode_verify().any()
    L.rbf_set_option(ctx, b"host_chunk_frames", 32)
    st.close()


def test_compress_empty_and_constant_inputs(pkg):
    comp = pkg.BloomFilterCompressor()
    empty = np.zeros(0, dtype=np.uint8)
    bitmap, witness, p, n, ratio = comp.compress(empty)          # reference: 0/0 -> nan -> raw passthrough
    assert bitmap is empty and witness == [] and np.isnan(p) and n == 0 and ratio == 1.0
    ones = np.ones(777, dtype=np.uint8)
    bitmap, witness, p, n, ratio = comp.compress(ones)           # p = 1 >= P*  (ivc:215-218)
    assert bitmap is ones and witness == [] and p == 1.0 and ratio == 1.0
    with pytest.raises(ValueError):
        comp.compress(np.full(10, 2, dtype=np.uint8))            # not a 0/1 vector


# ------------------------------------------------------------------ SURVEY 8(f) N3: adaptive threshold (ivc:727-766)
def test_adaptive_threshold_against_golden(pkg):
    import hashlib
    g = golden_json("adaptive_kat.json")
    vfc = pkg.VideoFrameCompressor(use_direct_yuv=True)
    for rec in g["cases"]:
        dt = np.dtype(rec["dtype"]).type
        h, w, noise_amp = rec["h"], rec["w"], rec["noise_amp"]
        rng = np.random.default_rng(rec["seed"])
        hi = 256 if dt == np.uint8 else 65536
        yy, xx = np.mgrid[0:h, 0:w]
        base = ((yy * 5 + xx * 3) * (hi // 512) % (hi - 2 * noise_amp - 1)).astype(np.int64)
        if rec["name"] in ("u8_tiny", "u8_mid"):
            base = ((yy + xx) // 4 + 20).astype(np.int64)
        prev = np.stack([base + rng.integers(0, noise_amp + 1, (h, w)) for _ in range(3)], axis=-1).astype(dt)
        curr = prev.copy()
        ch = rng.random((h, w)) < rec["p_change"]
        curr[ch] = (curr[ch].astype(np.int64) + rec["delta"]) % hi
        y = curr[:, :, 0].copy()
        smoothed = np.empty_like(y)
        pkg._cabi.check(pkg._cabi.lib().rbf_median_blur5(pkg._cabi.ctx(), pkg._cabi.ptr(y), h, w, y.dtype.itemsize, pkg._cabi.ptr(smoothed)), pkg._cabi.ctx())
        assert sha(smoothed) == rec["median_sha256"], rec["name"]          # == cv2.medianBlur(y, 5)
        nl = vfc._estimate_noise_level(y)
        assert type(nl).__name__ == rec["noise_level_type"] and float(nl).hex() == rec["noise_level"], rec["name"]
        assert float(vfc._adaptive_diff_threshold(y)).hex() == rec["threshold"]
        mask, changed, dens = vfc._calculate_frame_diff(pkg.YUVFrame(prev), pkg.YUVFrame(curr), threshold=None)
        assert int(mask.sum()) == rec["ones"] and sha(np.packbits(mask.reshape(-1))) == rec["mask_sha256"], rec["name"]


# ------------------------------------------------------------------ exchange over peer memory (single rank here; N > 1: test_two_ranks_p2p_equals_nccl, bench.py)
def test_peer_gather_single_rank(pkg):
    from new_bloom_filter_repo_b200 import distributed as rdist
    cabi = pkg._cabi
    st = pkg.FrameStream(270, 480, 3, np.uint8, max_frames=5)
    st.upload(synth_stream(270, 480, 5, 41, [0.05, 0.1]))
    res = st.encode_consecutive(5, 3.0)
    slot = (max((r.l + 7) // 8 for r in res) + 15) // 16 * 16 + 64
    pg = rdist.PeerGather(None, 4, slot)
    try:
        want1 = [st.fetch(t, want_mask=False)[0] for t in range(4)]
        pg.exchange(st)
        st.upload(synth_stream(270, 480, 5, 43, [0.1, 0.05]))      # the push overlaps this encode and must not see it
        st.encode_consecutive(5, 3.0)
        got1 = pg.result()
        assert got1.shape == (1, 4, slot)
        for t in range(4):
            assert np.array_equal(got1[0, t, : len(want1[t])], want1[t]) and not got1[0, t, len(want1[t]):].any()
        want2 = [st.fetch(t, want_mask=False)[0] for t in range(4)]
        pg.exchange(st)
        got2 = pg.result()                                       # the other half of the receive buffer
        for t in range(4):
            assert np.array_equal(got2[0, t, : len(want2[t])], want2[t])
        full = pg.recv.to_host().reshape(2, 1, 4, slot)
        for t in range(4):                                       # exchange 1 is still intact in half 1
            assert np.array_equal(full[1, 0, t, : len(want1[t])], want1[t])
    finally:
        pg.close()
    st.close()


# ------------------------------------------------------------------ round 2: per-stream options, pipelined encode, batched fetch
def test_pipelined_ranges_match_serial_and_oracle(pkg, co):
    """rbf_stream_encode pipelines K1/K2 over ranges of pairs on two streams: same bytes as the serial form (encode_ranges=1)
    and as the C oracle, including raw-passthrough pairs inside the ranges."""
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    frames = synth_stream(135, 240, 70, 17, [0.05, 0.01, 0.15, 0.0, 0.30, 0.40, 0.02])
    outs = {}
    for ranges in (1, 4, 8):
        pkg._cabi.check(L.rbf_set_option(ctx, b"encode_ranges", ranges), ctx)
        try:
            st = pkg.FrameStream(135, 240, 3, np.uint8, max_frames=70)
            st.upload(frames)
            res = st.encode_consecutive(70, 3.0)
            assert not st.decode_verify().any()
            outs[ranges] = [(r.ones, r.l, r.wlen, r.k, r.raw) + tuple(x.tobytes() for x in st.fetch(t)) for t, r in enumerate(res)]
            ms = st.stage_ms()
            assert ms["k3_query"] > 0 and ms["encode_total"] >= ms["k3_query"]
            st.close()
        finally:
            L.rbf_set_option(ctx, b"encode_ranges", 1)
    assert outs[1] == outs[4] == outs[8]
    assert any(o[4] for o in outs[4]) and not all(o[4] for o in outs[4])
    for t in (0, 3, 33, 68):
        m, ones = co.frame_diff_mask(frames[t], frames[t + 1], 3.0)
        ob, ow, op, on, oratio, ok, ol = co.compress(m.reshape(-1))
        o = outs[4][t]
        assert o[0] == ones and (o[4] or (o[1] == ol and o[5] == np.packbits(ob).tobytes() and o[6] == np.packbits(ow).tobytes()))


def test_stream_reuse_large_then_small_filters(pkg, co):
    """The per-slot clear only covers the high-water mark of what may hold set bits: a stream that coded big filters and then
    small ones (and the other way round) must still match the oracle, and the slot tails handed to the all-gather stay zero."""
    st = pkg.FrameStream(270, 480, 3, np.uint8, max_frames=4)
    for seq in ([0.30, 0.25, 0.2], [0.01, 0.02, 0.005], [0.2, 0.01, 0.1]):
        frames = synth_stream(270, 480, 4, 23, seq)
        st.upload(frames)
        res = st.encode_consecutive(4, 3.0)
        bms, wts, _ = st.fetch_batch(0, 3)
        for t, r in enumerate(res):
            m, ones = co.frame_diff_mask(frames[t], frames[t + 1], 3.0)
            ob, ow, op, on, oratio, ok, ol = co.compress(m.reshape(-1))
            assert (r.l, r.wlen, r.ones) == (ol, len(ow), ones)
            nb, nw = (ol + 7) // 8, (len(ow) + 7) // 8
            assert np.array_equal(bms[t, :nb], np.packbits(ob)) and not bms[t, nb:].any()
            assert np.array_equal(wts[t, :nw], np.packbits(ow)) and not wts[t, nw:].any()
            bm, wt, _ = st.fetch(t, want_mask=False)
            assert np.array_equal(bm, bms[t, :nb]) and np.array_equal(wt, wts[t, :nw])
        assert not st.decode_verify().any()
    st.close()


def test_gray_mode_against_golden(pkg):
    """BGR->gray branch of _calculate_frame_diff (ivc:792-795): K1 gray mode against fixtures from the real reference + cv2."""
    from tests.util import gray_pair
    g = golden_json("gray_kat.json")
    vfc = pkg.VideoFrameCompressor(use_direct_yuv=False)
    for rec in g["cases"]:
        prev, curr = gray_pair(rec)
        if rec["threshold"] is None:
            assert float(vfc._adaptive_diff_threshold(vfc._bgr2gray(curr))).hex() == rec["adaptive_threshold"]
        mask, changed, dens = vfc._calculate_frame_diff(prev, curr, threshold=rec["threshold"])
        assert int(mask.sum()) == rec["ones"], rec["name"]
        assert sha(np.packbits(mask.reshape(-1))) == rec["mask_sha256"], rec["name"]
        assert float(dens).hex() == rec["density"]
        assert changed.dtype.name == rec["changed_dtype"] and len(changed) == rec["changed_len"] and sha(changed) == rec["changed_sha256"]
    with pytest.raises(NotImplementedError):
        vfc._calculate_frame_diff(np.zeros((8, 8, 4), np.uint8), np.zeros((8, 8, 4), np.uint8), 3.0)


def test_gray_mode_large_frame_vs_oracle(pkg):
    from oracle import rbf_oracle as po
    for dt in (np.uint8, np.uint16):
        prev, curr = synth_pair(1080, 1920, 88, 0.05, dt)
        st = pkg.FrameStream(1080, 1920, 3, dt, max_frames=2, max_pairs=1, k1_only=True, gray_mode=True)
        st.upload(np.stack([prev, curr]))
        r = st.encode([0], [1], 7.0)[0]
        om = po.frame_diff_mask(prev, curr, 7.0, gray=True)
        assert r.ones == int(om.sum()) and np.array_equal(st.fetch(0)[2].reshape(1080, 1920), om)
        st.close()


def test_two_compressors_keep_their_own_options(pkg, co):
    """Options are per-stream state: a lossless GOP stream (mask_mode 1), a reference-mode stream and k1_only / gray streams
    used alternately give the same results as when used alone (VERDICT r01 weak #8: no process-global switches)."""
    frames = synth_stream(96, 128, 3, 51, [0.05])
    frames[2, 5, 5, 2] ^= 1                                  # chroma-only change: visible to mask_mode 1 only
    a = pkg.FrameStream(96, 128, 3, np.uint8, max_frames=3, mask_mode=1)
    b = pkg.FrameStream(96, 128, 3, np.uint8, max_frames=3, mask_mode=0)
    k = pkg.FrameStream(96, 128, 3, np.uint8, max_frames=3, k1_only=True)
    for s_ in (a, b, k):
        s_.upload(frames)
    ra1, rb1, rk1 = a.encode_consecutive(3, 3.0), b.encode_consecutive(3, 3.0), k.encode_consecutive(3, 3.0)
    rb2, rk2, ra2 = b.encode_consecutive(3, 3.0), k.encode_consecutive(3, 3.0), a.encode_consecutive(3, 3.0)
    assert [(r.ones, r.l, r.wlen) for r in ra1] == [(r.ones, r.l, r.wlen) for r in ra2]
    assert [(r.ones, r.l, r.wlen) for r in rb1] == [(r.ones, r.l, r.wlen) for r in rb2]
    assert ra1[1].ones == rb1[1].ones + 1 and ra1[1].resid == 0 and rb1[1].resid == 1
    assert all(r.wlen == 0 for r in rk1 + rk2) and [r.ones for r in rk1] == [r.ones for r in rb1]
    m, ones = co.frame_diff_mask(frames[1], frames[2], 3.0)
    assert rb1[1].ones == ones
    for s_ in (a, b, k):
        s_.close()


def test_index_filter_items_outside_uint32_follow_str_semantics(pkg, co):
    """ivc.RationalBloomFilter hashes str(item) (ivc:77-78): negative and >= 2**32 items must do the same, and the bit_array
    snapshot is read-only so that in-place writes cannot be silently lost."""
    items = [-5, -1, 2 ** 32, 2 ** 32 + 7, 2 ** 40 + 123, 2 ** 70 + 1, 17]
    f = pkg.IndexRationalBloomFilter(5000, 2.6)
    f.add_indices(items)
    bits = np.zeros(5000, dtype=np.uint8)
    co.filter_add_strings(bits, 2.6, pkg._cabi.IVC_SEEDS, [str(i) for i in items])
    assert np.array_equal(f.bit_array, bits)
    assert f.check_indices(items).all() and f.check_index(-5) and f.check_index(2 ** 70 + 1)
    probes = [-7, 2 ** 33, 99, 2 ** 64 + 3]
    assert np.array_equal(f.check_indices(probes), co.filter_check_strings(bits, 2.6, pkg._cabi.IVC_SEEDS, [str(i) for i in probes]).astype(bool))
    with pytest.raises(ValueError):
        f.bit_array[3] = 1
    g = pkg.IndexRationalBloomFilter(5000, 2.6)
    g.bit_array = bits
    assert np.array_equal(g.bit_array, bits)
    # every other item type, as an array of its own: each element hashes as str(element)
    typed = [np.array([2 ** 32, 2 ** 33 + 5, 2 ** 40 + 9, 2 ** 64 - 1], dtype=np.uint64),
             np.array([0, 5, 123456789, 2 ** 31, 2 ** 32 - 1], dtype=np.int64),          # no negatives: the index kernels
             np.array([-3, 0, 42, -2 ** 40, 2 ** 40], dtype=np.int64),
             np.array([5.0, -0.5, 1e20, 2.5e-7, 3.25]),
             ["5", "abc", "", "-0"],
             np.array([True, False]),
             np.array([7, "x", 2.5, -1, 2 ** 70, True, np.uint64(2 ** 63), "7"], dtype=object)]
    for arr in typed:
        names = [str(x) for x in arr]
        h =pkg.IndexRationalBloomFilter(5000, 2.6)
        h.add_indices(arr)
        want = np.zeros(5000, dtype=np.uint8)
        co.filter_add_strings(want, 2.6, pkg._cabi.IVC_SEEDS, names)
        assert np.array_equal(h.bit_array, want), names
        assert h.check_indices(arr).all() and h.check_index(arr[0])
        probe = np.concatenate([np.asarray(arr, dtype=object), np.array([6, "6", 6.0, False, -6, 2 ** 32 + 6], dtype=object)])
        assert np.array_equal(h.check_indices(probe),
                              co.filter_check_strings(want, 2.6, pkg._cabi.IVC_SEEDS, [str(x) for x in probe]).astype(bool)), names
    assert [str(x) for x in typed[5]] == ["True", "False"] and [str(x) for x in typed[3]][0] == "5.0"
    # "5" (string kernel) sets the bits of 5 (index kernel); 5.0 those of "5.0", a numpy bool those of "True"
    for a, b in ((["5"], [5]), (np.array(["5"]), np.array([5], dtype=np.uint32)), (np.array([5.0]), ["5.0"]),
                 (np.array([True]), ["True"])):
        ha, hb = pkg.IndexRationalBloomFilter(5000, 2.6), pkg.IndexRationalBloomFilter(5000, 2.6)
        ha.add_indices(a)
        hb.add_indices(b)
        assert np.array_equal(ha.bit_array, hb.bit_array) and ha.bit_array.any(), (a, b)


def test_inter_payloads_match_oracle_bytes_and_thread_count(pkg, co, tmp_path):
    """The batched GOP path (one fetch per group, zlib in a thread pool) writes the same bytes whatever the thread count, and
    each coded inter payload equals header + C-oracle bitmap/witness + zlib(values)."""
    import struct
    import zlib
    from new_bloom_filter_repo_b200 import improved_video_compressor as ivcmod
    frames = [f for f in synth_stream(120, 160, 9, 61, [0.05, 0.0, 0.2, 0.4])]
    payloads = {}
    for nt in (1, 4):
        comp = pkg.ImprovedVideoCompressor(keyframe_interval=4, num_threads=nt, batch_size=3)
        comp.inter_frame_mode = "reference"
        comp.inter_frame_threshold = 3.0
        comp.compress_video(list(frames), input_color_space="YUV")
        payloads[nt] = list(comp._last_compressed_frames)
        dec = comp.decompress_video(compressed_frames=payloads[nt])
        assert comp.verify_lossless(frames, dec)["lossless"]
    assert payloads[1] == payloads[4]
    checked = raw_seen = 0
    for i, pl in enumerate(payloads[4]):
        if not pl.startswith(ivcmod._INTER_TAG):
            continue
        prev, curr = frames[i - 1], frames[i]
        m, ones = co.frame_diff_mask(prev, curr, 3.0)
        ob, ow, op, on, oratio, ok, ol = co.compress(m.reshape(-1))
        vals = curr[m.astype(bool)].reshape(-1)
        hdr = ivcmod._INTER_TAG + struct.pack("<IIIBB", 120, 160, 1, 3, 1 if ok == 0 else 0)
        body = struct.pack("<dIIQ", ok, ol, len(ow), ones)
        if ok == 0:
            rz = zlib.compress(np.packbits(m.reshape(-1)).tobytes(), 9)
            body += struct.pack("<I", len(rz)) + rz + struct.pack("<I", 0)
            raw_seen += 1
        else:
            bb, wb = np.packbits(ob).tobytes(), np.packbits(ow).tobytes()
            body += struct.pack("<I", len(bb)) + bb + struct.pack("<I", len(wb)) + wb
        vz = zlib.compress(vals.tobytes(), 9)
        body += struct.pack("<II", len(vz), vals.size) + vz
        assert pl == hdr + body, i
        checked += 1
    assert checked >= 4 and raw_seen >= 1
    # a static scene: the raw-passthrough mask is stored compressed (ADVICE r01), far below n/8 bytes
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=30)
    comp.compress_video([frames[0], frames[0].copy(), frames[0].copy()], input_color_space="YUV")
    assert all(len(p) < 200 for p in comp._last_compressed_frames[1:])


def test_inter_payload_v1_still_decodes_and_corruption_raises(pkg):
    import struct
    import zlib
    from new_bloom_filter_repo_b200 import improved_video_compressor as ivcmod
    frames = [f for f in synth_stream(64, 64, 3, 71, [0.4, 0.05])]
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=30)
    comp.compress_video(list(frames), input_color_space="YUV")
    pls = list(comp._last_compressed_frames)
    assert pls[1].startswith(ivcmod._INTER_TAG)
    # rebuild frame 1 (raw passthrough at p = 0.4) in the round-1 layout: plain packbits mask
    pos = len(ivcmod._INTER_TAG)
    h, w, isz, ch, raw = struct.unpack_from("<IIIBB", pls[1], pos)
    assert raw == 1
    p2 = pos + struct.calcsize("<IIIBB") + struct.calcsize("<dIIQ")
    (bl,) = struct.unpack_from("<I", pls[1], p2)
    rawbits = zlib.decompress(pls[1][p2 + 4:p2 + 4 + bl])
    v1 = ivcmod._INTER_TAG_V1 + pls[1][pos:p2] + struct.pack("<I", len(rawbits)) + rawbits + pls[1][p2 + 4 + bl:]
    dec = comp.decompress_video(compressed_frames=[pls[0], v1, pls[2]])
    assert comp.verify_lossless(frames, dec)["lossless"]
    # a payload whose announced pixel count does not match its mask must raise, not return a wrong frame (ADVICE r01)
    bad = bytearray(pls[2])
    off = len(ivcmod._INTER_TAG) + struct.calcsize("<IIIBB") + struct.calcsize("<dII")
    (ones,) = struct.unpack_from("<Q", bad, off)
    struct.pack_into("<Q", bad, off, ones + 1)
    with pytest.raises(ValueError):
        comp.decompress_video(compressed_frames=[pls[0], pls[1], bytes(bad)])
    with pytest.raises(ValueError):
        comp.decompress_video(compressed_frames=[pls[1]])


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16])
def test_single_channel_frames_mask_gather_apply(pkg, dtype):
    """Grayscale branch of _calculate_frame_diff / _apply_frame_diff (ivc:796-798, ivc:843, ivc:897-905): 1 and 2 bytes per pixel."""
    from oracle import rbf_oracle as po
    rng = np.random.default_rng(91)
    hi = 256 if dtype == np.uint8 else 65536
    prev = rng.integers(0, hi, (211, 333)).astype(dtype)
    curr = prev.copy()
    ch = rng.random(prev.shape) < 0.07
    curr[ch] = (curr[ch].astype(np.int64) + hi // 4) % hi
    vfc = pkg.VideoFrameCompressor()
    mask, changed, dens = vfc._calculate_frame_diff(prev, curr, threshold=3.0)
    om = po.frame_diff_mask(prev, curr, 3.0)
    assert np.array_equal(mask, om) and changed.dtype == dtype
    assert np.array_equal(changed, curr[np.where(om == 1)])
    assert np.array_equal(vfc._apply_frame_diff(prev, mask, changed), curr)


def test_k2_beside_k3_matches_serial(pkg):
    """kq_ranges > 1 runs K2 of range q+1 on a second stream beside K3 of range q (K3 with fewer warps / less shared memory so that
    a K2 CTA fits next to it): same bytes as the serial encode, round trip intact."""
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    frames = synth_stream(540, 960, 40, 19, [0.05, 0.02, 0.12, 0.0, 0.30, 0.40])
    outs = {}
    for name, opts in (("serial", {"kq_ranges": 1, "query_warps": 0, "query_smem_bytes": 0}),
                       ("beside", {"kq_ranges": 4, "query_warps": 24, "query_smem_bytes": 222000}),
                       ("beside8", {"kq_ranges": 8, "query_warps": 20, "query_smem_bytes": 200000})):
        for k, v in opts.items():
            pkg._cabi.check(L.rbf_set_option(ctx, k.encode(), v), ctx)
        try:
            st = pkg.FrameStream(540, 960, 3, np.uint8, max_frames=40)
            st.upload(frames)
            for _ in range(2):                                  # twice: the second call sees the first one's leftovers
                res = st.encode_consecutive(40, 3.0)
            assert not st.decode_verify().any()
            bms, wts, _ = st.fetch_batch(0, 39)
            outs[name] = [(r.ones, r.l, r.wlen, r.raw, bms[t].tobytes(), wts[t].tobytes()) for t, r in enumerate(res)]
            st.close()
        finally:
            for k, v in (("kq_ranges", 1), ("query_warps", 0), ("query_smem_bytes", 0)):
                L.rbf_set_option(ctx, k.encode(), v)
    assert outs["serial"] == outs["beside"] == outs["beside8"]
    assert any(o[3] for o in outs["serial"]) and not all(o[3] for o in outs["serial"])


def test_two_ranks_p2p_equals_nccl(pkg, tmp_path):
    """One stream block-partitioned over 2 GPUs (ShardedStreamEncoder): the NCCL all-gather and the peer-memory push leave the same
    bytes on both ranks, equal to a single-GPU encode of the whole stream.  Skipped on a 1-GPU box (bench.py --gpus N verifies the
    same thing at N = 2 / 4 / 8 after its timed region: `gather_verified`, `strong_matches_single_gpu`)."""
    import json
    import socket
    import subprocess
    import sys
    try:
        ngpu = int(subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout.count("GPU "))
    except Exception:
        ngpu = 1
    if ngpu < 2:
        pytest.skip("needs 2 GPUs")
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    root = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(root, "tests", "_rank_worker_gpu.py"), str(tmp_path)]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    outs = [json.load(open(tmp_path / ("rank%d.json" % r))) for r in range(2)]
    assert outs[0]["nccl"]["sha"] == outs[1]["nccl"]["sha"] == outs[0]["p2p"]["sha"] == outs[1]["p2p"]["sha"] == outs[0]["single_gpu_sha"]
    assert outs[0]["p2p"]["l"] == outs[0]["single_gpu_l"] and outs[0]["p2p"]["used"] == "p2p"
