"""Adaptive value coding of inter frames (value_coding="adaptive", 'RBF3' payloads): the value stream of each inter frame holds either
the current samples at the changed pixels or their residuals (curr - prev) mod 2^bits per sample, whichever zlib stream is shorter.
The device side -- the residual gather (value_mode 1 of rbf_stream_gather_changed / rbf_stream_zlib_changed) and the residual apply
of K4c (rbf_stream_apply_chain with value modes) -- is compared with the numpy forms below, and decompress_video with a frame-by-frame route
built from the C oracle's mask decode and these numpy forms."""
import hashlib
import struct
import zlib

import numpy as np
import pytest

from tests.util import synth_stream

gpu = pytest.mark.gpu


# ------------------------------------------------------------------ numpy oracle of the residual coding
def np_gather(prev, curr, mask, residual):
    """Values of the set pixels of `mask` (H x W) in row-major, channel-minor order: curr's samples, or (curr - prev) mod 2^bits."""
    n = mask.size
    m = mask.reshape(-1).astype(bool)
    c = curr.reshape(n, -1)[m]
    return ((c - prev.reshape(n, -1)[m]) if residual else c).reshape(-1)


def np_apply(prev, mask, values, residual):
    """The next frame: the set pixels of `mask` replaced by `values`, or `values` added to them per sample mod 2^bits."""
    out = prev.copy()
    flat = out.reshape(mask.size, -1)
    m = mask.reshape(-1).astype(bool)
    v = np.asarray(values, dtype=prev.dtype).reshape(-1, flat.shape[1])
    flat[m] = (flat[m] + v) if residual else v
    return out


# ------------------------------------------------------------------ fixtures and helpers
@pytest.fixture(scope="module")
def pkg():
    import new_bloom_filter_repo_b200 as p
    assert p._cabi.device_info()["cc"] == (9, 0)
    return p


@pytest.fixture(scope="module")
def co():
    from oracle import c_oracle
    c_oracle.build()
    return c_oracle


def _ivc():
    from new_bloom_filter_repo_b200 import improved_video_compressor as ivcmod
    return ivcmod


def _independent_decode(co, payloads):
    """Frame by frame: keyframes with the CPU keyframe codec; inter frames with the C oracle's mask decode and np_apply on the
    previously decoded frame."""
    from new_bloom_filter_repo_b200.fixed_video_compressor import FixedVideoCompressor
    ivcmod = _ivc()
    out = []
    for c in payloads:
        if not c.startswith(ivcmod._INTER_TAGS):
            f = FixedVideoCompressor(verbose=False).decompress_frame(c)
            out.append(np.asarray(f.data if hasattr(f, "yuv_info") else f))
            continue
        p = ivcmod.ImprovedVideoCompressor._parse_inter(c)
        n = p.h * p.w
        vals = np.frombuffer(zlib.decompress(p.vz), dtype=np.uint8 if p.isz == 1 else np.uint16)[:p.vcount]
        if p.raw:
            bits = bytes(p.mask_bytes) if p.v1 else zlib.decompress(p.mask_bytes)
            mask = np.unpackbits(np.frombuffer(bits, dtype=np.uint8))[:n]
        else:
            bm = np.unpackbits(np.frombuffer(p.mask_bytes, dtype=np.uint8))[:p.l]
            wt = np.unpackbits(np.frombuffer(p.witness_bytes, dtype=np.uint8))[:p.wlen]
            mask = co.decompress(bm, wt, n, p.k)
        out.append(np_apply(out[-1], mask.reshape(p.h, p.w), vals, p.vmode == 1))
    return out


def _frames(h, w, ch, dtype, nfr, seed, p_seq):
    f = synth_stream(h, w, nfr, seed, p_seq, dtype)
    if ch == 1:
        f = np.ascontiguousarray(f[..., 0])
    return [x for x in f]


def _compress(pkg, frames, ki, bs, coder="zlib", yuv=False, coding="adaptive"):
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=ki, batch_size=bs, use_direct_yuv=yuv)
    comp.entropy_coder = coder
    comp.value_coding = coding
    comp.compress_video(list(frames), input_color_space="YUV" if yuv else "BGR")
    return comp, list(comp._last_compressed_frames)


def _vmodes(payloads):
    ivcmod = _ivc()
    return [ivcmod.ImprovedVideoCompressor._parse_inter(p).vmode if p.startswith(ivcmod._INTER_TAGS) else None for p in payloads]


def _check_round_trip(co, comp, frames, payloads, yuv):
    dec = comp.decompress_video(compressed_frames=payloads)
    ref = _independent_decode(co, payloads)
    assert len(dec) == len(frames) == len(ref)
    for i, (d, r, f) in enumerate(zip(dec, ref, frames)):
        dd = d.data if hasattr(d, "yuv_info") else d
        assert hasattr(d, "yuv_info") == yuv, i
        assert dd.dtype == r.dtype and dd.shape == r.shape, i
        assert np.array_equal(dd, r), i
        assert np.array_equal(dd, np.asarray(f.data if hasattr(f, "yuv_info") else f)), i
    return dec


def _raw_slots(masks, n):
    nb = (n + 7) // 8
    bms = np.zeros((len(masks), (nb + 15) // 16 * 16), dtype=np.uint8)
    for i, m in enumerate(masks):
        bms[i, :nb] = np.packbits(m)
    return bms


# ------------------------------------------------------------------ CPU: the RBF3 layout
class _R:
    def __init__(self, raw, k, l, wlen, ones):
        self.raw, self.k, self.l, self.wlen, self.ones = raw, k, l, wlen, ones


def _layout(raw, vmode):
    I = _ivc().ImprovedVideoCompressor
    rng = np.random.default_rng(11)
    bm, wt = rng.integers(0, 256, 300).astype(np.uint8), rng.integers(0, 256, 300).astype(np.uint8)
    r = _R(raw, 0.0 if raw else 1.4142135623730951, 0 if raw else 999, 0 if raw else 333, 41)
    rz = rng.integers(0, 256, 50).astype(np.uint8).tobytes() if raw else None
    return I._inter_layout((17, 29), 1, 3, r, bm, wt, rz, b"value-or-residual-stream", 123, vmode), r, bm, wt, rz


@pytest.mark.parametrize("vmode", [0, 1])
@pytest.mark.parametrize("raw", [False, True])
def test_rbf3_layout_round_trips(raw, vmode):
    ivcmod = _ivc()
    pl, r, bm, wt, rz = _layout(raw, vmode)
    assert pl.startswith(ivcmod._INTER_TAG_V3)
    assert pl[len(ivcmod._INTER_TAG_V3) + struct.calcsize("<IIIBB")] == vmode          # right after the raw flag
    p = ivcmod.ImprovedVideoCompressor._parse_inter(pl)
    assert not p.v1 and p.vmode == vmode
    assert (p.h, p.w, p.isz, p.ch, bool(p.raw)) == (17, 29, 1, 3, raw)
    assert (p.k, p.l, p.wlen, p.ones, p.vcount) == (r.k, r.l, r.wlen, 41, 123)
    assert bytes(p.vz) == b"value-or-residual-stream"
    if raw:
        assert bytes(p.mask_bytes) == rz and bytes(p.witness_bytes) == b""
    else:
        assert bytes(p.mask_bytes) == bm[:(999 + 7) // 8].tobytes() and bytes(p.witness_bytes) == wt[:(333 + 7) // 8].tobytes()
    # without a vmode the layout is RBF2, one byte shorter, read back as plain values
    p2 = _ivc().ImprovedVideoCompressor._inter_layout((17, 29), 1, 3, r, bm, wt, rz, b"value-or-residual-stream", 123)
    assert p2.startswith(ivcmod._INTER_TAG) and len(p2) == len(pl) - 1
    assert ivcmod.ImprovedVideoCompressor._parse_inter(p2).vmode == 0


@pytest.mark.parametrize("bad", [2, 7, 255])
def test_rbf3_bad_vmode_raises(bad):
    ivcmod = _ivc()
    pl = bytearray(_layout(False, 1)[0])
    pl[len(ivcmod._INTER_TAG_V3) + struct.calcsize("<IIIBB")] = bad
    with pytest.raises(ValueError, match="value coding"):
        ivcmod.ImprovedVideoCompressor._parse_inter(bytes(pl))


# ------------------------------------------------------------------ residual gather (value_mode 1)
def _four_frames(h, w, ch, dtype, seed):
    """f0 random; f1 = f0 (empty mask); f2 = f1 + 1 on every sample (all-ones mask, wrapping at the top); f3 = f2 with 30 % of the
    pixels changed at random."""
    rng = np.random.default_rng(seed)
    hi = 256 if dtype == np.uint8 else 65536
    shape = (h, w, ch) if ch > 1 else (h, w)
    f0 = rng.integers(0, hi, shape).astype(dtype)
    f0.reshape(-1)[:3] = hi - 1
    f2 = f0 + dtype(1)
    f3 = f2.copy()
    sel = rng.random((h, w)) < 0.3
    f3[sel] = rng.integers(0, hi, f3[sel].shape).astype(dtype)
    return [f0, f0.copy(), f2, f3]


@gpu
@pytest.mark.parametrize("h,w,ch,dtype", [(37, 53, 1, np.uint8), (37, 53, 3, np.uint8), (37, 53, 1, np.uint16), (37, 53, 3, np.uint16),
                                          (2160, 3840, 3, np.uint8)])
def test_residual_gather_matches_oracle(pkg, h, w, ch, dtype):
    fr = _four_frames(h, w, ch, dtype, h + w + ch)
    st = pkg.FrameStream(h, w, ch, dtype, max_frames=4, max_pairs=3, k1_only=True, mask_mode=1)
    try:
        st.upload(np.stack(fr))
        st.encode([0, 1, 2], [1, 2, 3], 0.0)
        masks = [st.fetch(j)[2].reshape(h, w) for j in range(3)]
        for j in range(3):
            a, b = fr[j], fr[j + 1]
            assert np.array_equal(masks[j], (a != b).reshape(h, w, -1).any(-1)), j
        assert not masks[0].any() and masks[1].all()
        plain = st.gather_changed()
        st.set_option("value_mode", 1)
        resid = st.gather_changed()
        zs = st.zlib_changed()
        st.set_option("value_mode", 0)
        assert all(np.array_equal(x, y) for x, y in zip(st.gather_changed(), plain))        # the option switches back
        for j in range(3):
            assert plain[j].dtype == resid[j].dtype == np.dtype(dtype)
            assert np.array_equal(plain[j], np_gather(fr[j], fr[j + 1], masks[j], False)), j
            assert np.array_equal(resid[j], np_gather(fr[j], fr[j + 1], masks[j], True)), j
            assert zlib.decompress(zs[j]) == resid[j].tobytes(), j
        assert resid[0].size == 0 and (resid[1] == 1).all()
    finally:
        st.close()


@gpu
def test_value_mode_is_checked_before_any_launch(pkg):
    import ctypes as C
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    fr = _four_frames(16, 24, 3, np.uint8, 3)
    st = pkg.FrameStream(16, 24, 3, np.uint8, max_frames=4, max_pairs=3, k1_only=True, mask_mode=1)
    try:
        st.upload(np.stack(fr))
        st.encode([0, 1, 2], [1, 2, 3], 0.0)
        L.rbf_reset_counters(ctx)
        for bad in (2, -1, 256):
            assert L.rbf_stream_set_option(st._h, b"value_mode", bad) == -1            # RBF_ERR_INVALID
        # the stream only holds 1 or 3 channels of 1- or 2-byte samples: other (C, S) never get a stream to set value_mode on
        h = C.c_void_p()
        for c_, s_ in ((2, 1), (4, 1), (3, 4), (2, 2)):
            assert L.rbf_stream_create(ctx, 16, 24, c_, s_, 4, 3, C.byref(h)) == -1, (c_, s_)
        assert L.rbf_get_counter(ctx, b"kernel_launches") == 0
        assert L.rbf_get_counter(ctx, b"h2d_bytes") == 0 and L.rbf_get_counter(ctx, b"d2h_bytes") == 0
        plain = st.gather_changed()                                                     # the failed calls left value_mode at 0
        assert all(np.array_equal(plain[j], np_gather(fr[j], fr[j + 1], st.fetch(j)[2], False)) for j in range(3))
    finally:
        st.close()


# ------------------------------------------------------------------ residual apply in K4c (apply_chain with per-pair flags)
@gpu
@pytest.mark.parametrize("h,w,ch,dtype", [(37, 53, 1, np.uint8), (37, 53, 3, np.uint8), (45, 91, 1, np.uint16), (67, 129, 3, np.uint16),
                                          (2160, 3840, 3, np.uint8)])
def test_apply_chain_mixed_flags_matches_oracle(pkg, h, w, ch, dtype):
    rng = np.random.default_rng(h * w + ch)
    n = h * w
    hi = 256 if dtype == np.uint8 else 65536
    shape = (h, w, ch) if ch > 1 else (h, w)
    masks = [np.zeros(n, np.uint8), np.ones(n, np.uint8), (rng.random(n) < 0.3).astype(np.uint8),
             (rng.random(n) < 0.01).astype(np.uint8)]
    flags = [1, 1, 0, 1]
    st = pkg.FrameStream(h, w, ch, dtype, max_frames=5, max_pairs=4, k1_only=True)
    try:
        cnt = len(masks)
        consumed, ones = st.decode_masks(_raw_slots(masks, n), np.zeros((cnt, 0), np.uint8), [0] * cnt, [0] * cnt, [0.0] * cnt,
                                         [1] * cnt)
        assert list(ones) == [int(m.sum()) for m in masks]
        base = rng.integers(0, hi, shape).astype(dtype)
        base.reshape(-1)[:5] = hi - 1                        # residuals that wrap past the top
        vals = [rng.integers(0, hi, int(m.sum()) * ch).astype(dtype) for m in masks]
        exp, cur = [], base
        for m, v, f in zip(masks, vals, flags):
            cur = np_apply(cur, m.reshape(h, w), v, f)
            exp.append(cur)
        # base in slot 3: the chain writes slots 4, 0, 1, 2 (slots wrap)
        st.upload(base, first=3)
        applied = st.apply_chain(3, vals, modes=flags)
        assert list(applied) == list(ones)
        got = st.download_batch(4, cnt)
        for t in range(cnt):
            assert np.array_equal(got[t], exp[t]), t
        assert np.array_equal(st.download(3), base)
        # all pairs plain through the same entry point equals apply_chain without flags
        st.upload(base, first=0)
        a0 = st.apply_chain(0, vals, modes=[0] * cnt)
        g0 = st.download_batch(1, cnt)
        st.upload(base, first=0)
        a1 = st.apply_chain(0, vals)
        assert list(a0) == list(a1) and np.array_equal(g0, st.download_batch(1, cnt))
        # one value too few at residual pair 2: pairs 0 and 1 are applied, frames of pairs 2 and 3 are not written
        mixed = [0, 1, 1, 0]
        exp2, cur = [], base
        for m, v, f in zip(masks, vals, mixed):
            cur = np_apply(cur, m.reshape(h, w), v, f)
            exp2.append(cur)
        sentinel = np.full((2,) + shape, 7, dtype=dtype)
        st.upload(base, first=0)
        st.upload(sentinel, first=3)
        short = vals[:2] + [vals[2][:-ch]] + vals[3:]
        applied = st.apply_chain(0, short, modes=mixed)
        assert list(applied) == [ones[0], ones[1], 0, 0]
        got = st.download_batch(1, 4)
        assert np.array_equal(got[0], exp2[0]) and np.array_equal(got[1], exp2[1])
        assert (got[2] == 7).all() and (got[3] == 7).all()
        with pytest.raises(pkg._cabi.RbfError):
            st.apply_chain(0, vals, modes=[0, 2, 0, 0])
        with pytest.raises(ValueError):
            st.apply_chain(0, vals, modes=[0, 1])
    finally:
        st.close()


# ------------------------------------------------------------------ compress_video(value_coding="adaptive") round trips
P_MIX = [0.05, 0.0, 0.4, 0.01]           # coded, unchanged (raw, empty mask), dense (raw), sparse coded


@gpu
@pytest.mark.parametrize("h,w,ch,dtype,yuv,nfr,ki,bs,coder", [
    (37, 53, 3, np.uint8, True, 12, 30, 4, "zlib"),        # YUV444: one run of 11 in groups of 4, 4, 3
    (64, 64, 3, np.uint8, False, 12, 6, 5, "gpu"),         # BGR: runs of 5 = exactly one group each
    (37, 53, 1, np.uint8, False, 7, 30, 1, "zlib"),        # groups of one
    (64, 64, 1, np.uint16, False, 11, 5, 3, "gpu"),
    (37, 53, 3, np.uint16, False, 10, 30, 7, "zlib"),
    (1080, 1920, 3, np.uint8, True, 6, 30, 3, "gpu"),
])
def test_adaptive_round_trip(pkg, co, h, w, ch, dtype, yuv, nfr, ki, bs, coder):
    frames = _frames(h, w, ch, dtype, nfr, 5, P_MIX)
    if yuv:
        frames = [pkg.YUVFrame(f) for f in frames]
    comp, payloads = _compress(pkg, frames, ki, bs, coder, yuv)
    ivcmod = _ivc()
    assert sum(p.startswith(ivcmod._INTER_TAG_V3) for p in payloads) == nfr - (nfr + ki - 1) // ki
    assert not any(p.startswith(ivcmod._INTER_TAG) for p in payloads)
    _check_round_trip(co, comp, frames, payloads, yuv)


@gpu
@pytest.mark.parametrize("coder", ["zlib", "gpu"])
def test_adaptive_reference_mode_keyframe_fallbacks(pkg, co, coder):
    f = synth_stream(96, 80, 11, 13, [0.05, 0.02])
    y, x = np.argwhere((f[3, ..., 0] == f[2, ..., 0]) & (f[7, ..., 0] == f[6, ..., 0]))[0]
    f[3:, y, x, 2] ^= 1                                    # chroma-only changes: frames 3 and 7 become keyframes inside the run
    f[7:, y, x, 2] ^= 1
    frames = [pkg.YUVFrame(a) for a in f]
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=30, batch_size=3)
    comp.inter_frame_mode = "reference"
    comp.inter_frame_threshold = 3.0
    comp.entropy_coder = coder
    comp.value_coding = "adaptive"
    stats = comp.compress_video(list(frames), input_color_space="YUV")
    pls = list(comp._last_compressed_frames)
    vm = _vmodes(pls)
    assert stats["keyframes"] == 3 and vm[0] is None and vm[3] is None and vm[7] is None
    assert 1 in vm
    _check_round_trip(co, comp, frames, pls, True)


def _texture(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3)).astype(np.uint8)


def _gradient(h, w):
    yy, xx = np.mgrid[0:h, 0:w]
    g = ((yy + 2 * xx) // 3) % 256
    return np.stack([g, (g + 40) % 256, (255 - g)], -1).astype(np.uint8)


@gpu
@pytest.mark.parametrize("coder", ["zlib", "gpu"])
def test_choice_is_pinned_by_content(pkg, co, coder):
    """Random texture -> the same + 1 on every sample: the residuals are all ones, the values incompressible -> residuals.
    -> a cut to a smooth gradient: the values compress, the residuals are noise -> plain.  Then the gradient + 1 (residuals) and a
    cut to one flat colour (plain).  All in one group."""
    h, w = 120, 160
    t = _texture(h, w, 1)
    g = _gradient(h, w)
    frames = [t, t + np.uint8(1), g, g + np.uint8(1), np.full((h, w, 3), 77, np.uint8)]
    comp, pls = _compress(pkg, frames, 30, 8, coder)
    assert _vmodes(pls) == [None, 1, 0, 1, 0]
    _check_round_trip(co, comp, frames, pls, False)


@gpu
@pytest.mark.parametrize("coder", ["zlib", "gpu"])
def test_adaptive_payload_is_never_longer_than_plain(pkg, coder):
    frames = _frames(64, 96, 3, np.uint8, 9, 17, P_MIX)
    _, plain = _compress(pkg, frames, 30, 4, coder, coding="plain")
    _, adapt = _compress(pkg, frames, 30, 4, coder)
    vm = _vmodes(adapt)
    assert 0 in vm and 1 in vm
    ivcmod = _ivc()
    hdr = len(ivcmod._INTER_TAG) + struct.calcsize("<IIIBB")
    for i, (a, b) in enumerate(zip(plain, adapt)):
        if i == 0:
            assert a == b                                  # keyframes are the reference's bytes
        elif vm[i] == 0:                                   # the plain payload with the RBF3 tag and a vmode byte of 0
            assert b == ivcmod._INTER_TAG_V3 + a[len(ivcmod._INTER_TAG):hdr] + b"\x00" + a[hdr:], i
        else:                                              # residuals are kept only when strictly shorter
            assert len(b) <= len(a), i


@gpu
def test_value_coding_is_validated(pkg):
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=30)
    assert comp.value_coding == "plain"
    comp.value_coding = "residual"
    with pytest.raises(ValueError, match="value_coding"):
        comp.compress_video(_frames(16, 16, 3, np.uint8, 2, 1, [0.1]))


# ------------------------------------------------------------------ the default writes exactly the parent's bytes
def _stream_sha(pkg, coder):
    frames = _frames(96, 128, 3, np.uint8, 12, 21, P_MIX)
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=30, batch_size=4)
    comp.entropy_coder = coder
    comp.compress_video(list(frames))
    pls = list(comp._last_compressed_frames)
    hs = hashlib.sha256()
    for p in pls:
        hs.update(struct.pack("<I", len(p)) + p)
    return hs.hexdigest(), pls


# sha256 of the length-prefixed payloads of _stream_sha's stream, written by the commit before value_coding existed
PLAIN_SHA = {
    "zlib": "f6f4e929f1e4fa2fc419927dac33a1f5a7ecdf859471a0dd5c3a841a73a360a4",
    "gpu": "5e1b0f787e12ef175d3aac062ca920a53078bb296e66ae84e89f56ba0cce880e",
}


@gpu
@pytest.mark.parametrize("coder", ["zlib", "gpu"])
def test_default_writes_the_previous_bytes(pkg, coder):
    digest, pls = _stream_sha(pkg, coder)
    assert not any(p.startswith(_ivc()._INTER_TAG_V3) for p in pls)
    assert digest == PLAIN_SHA[coder]


# ------------------------------------------------------------------ a group costs the same with adaptive payloads
@gpu
def test_counters_per_group_match_plain(pkg):
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    frames = _frames(120, 160, 3, np.uint8, 30, 37, [0.05, 0.02, 0.08])
    counts = {}
    for coding in ("plain", "adaptive"):
        comp, pls = _compress(pkg, frames, 30, 10, coding=coding)
        if coding == "adaptive":
            assert 1 in _vmodes(pls)
        L.rbf_reset_counters(ctx)
        dec = comp.decompress_video(compressed_frames=pls)
        assert np.array_equal(np.asarray(dec[-1]), frames[-1])
        counts[coding] = tuple(L.rbf_get_counter(ctx, k) for k in (b"kernel_launches", b"h2d_bytes", b"d2h_bytes"))
    assert counts["plain"] == counts["adaptive"], counts
