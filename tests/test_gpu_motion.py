"""Motion-compensated value coding of inter frames (value_coding="motion", 'RBF4' payloads).  Each inter frame stores the changed samples,
their residuals against the co-located previous pixel, or their residuals against the previous frame shifted per 16 x 16 block by the
vector a full +-16 px SAD search found, whichever costs least.  The device side -- the search (FrameStream.motion_search), the motion
residual gather (motion_values 1) and the motion-compensated apply (apply_chain(motion=...)) -- is compared with the numpy model below,
and decompress_video with a frame-by-frame route built from the C oracle's mask decode and that model."""
import struct
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
from numpy.lib.stride_tricks import sliding_window_view

from tests.util import synth_stream

gpu = pytest.mark.gpu
B, R = 16, 16


# ------------------------------------------------------------------ numpy model of search, prediction, gather and apply
def np_block_vector(prev, curr, by, bx):
    """(dx, dy) of block (by, bx): the minimum of (SAD, |dx| + |dy|, dy, dx) over the 33 x 33 candidates, the SAD taken over the block's
    in-frame pixels and every sample of |curr - prev(clamp(y + dy), clamp(x + dx))|."""
    H, W = curr.shape[:2]
    p = prev.reshape(H, W, -1).astype(np.int64)
    c = curr.reshape(H, W, -1).astype(np.int64)
    y0, x0 = B * by, B * bx
    bh, bw = min(B, H - y0), min(B, W - x0)
    ys = np.clip(np.arange(y0 - R, y0 + B + R), 0, H - 1)
    xs = np.clip(np.arange(x0 - R, x0 + B + R), 0, W - 1)
    win = p[ys][:, xs]                                                     # window(wy, wx) = prev(clamp(y0 - 16 + wy), clamp(x0 - 16 + wx))
    v = sliding_window_view(win, (bh, bw), axis=(0, 1))[:2 * R + 1, :2 * R + 1]   # [dy + 16, dx + 16, C, bh, bw]
    sad = np.abs(v - c[y0:y0 + bh, x0:x0 + bw].transpose(2, 0, 1)[None, None]).sum((2, 3, 4))
    dy, dx = np.mgrid[-R:R + 1, -R:R + 1]
    best = np.lexsort((dx.ravel(), dy.ravel(), (np.abs(dx) + np.abs(dy)).ravel(), sad.ravel()))[0]
    return int(dx.ravel()[best]), int(dy.ravel()[best])


def np_motion_search(prev, curr, blocks=None):
    """int8 [by, bx, 2] field of a pair; `blocks` (a list of (by, bx)) limits the model to those blocks (the rest stay 0)."""
    H, W = curr.shape[:2]
    nby, nbx = -(-H // B), -(-W // B)
    out = np.zeros((nby, nbx, 2), np.int8)
    for by, bx in (blocks if blocks is not None else [(i, j) for i in range(nby) for j in range(nbx)]):
        out[by, bx] = np_block_vector(prev, curr, by, bx)
    return out


def np_predict(prev, field):
    H, W = prev.shape[:2]
    yy, xx = np.mgrid[0:H, 0:W]
    f = np.asarray(field, np.int64).reshape(-(-H // B), -(-W // B), 2)
    dx, dy = f[yy // B, xx // B, 0], f[yy // B, xx // B, 1]
    return prev[np.clip(yy + dy, 0, H - 1), np.clip(xx + dx, 0, W - 1)]


def np_motion_gather(prev, curr, mask, field):
    """(curr - pred) mod 2^bits at the set pixels of `mask`, pixel-major, channel-minor."""
    n = mask.size
    m = mask.reshape(-1).astype(bool)
    return (curr.reshape(n, -1)[m] - np_predict(prev, field).reshape(n, -1)[m]).reshape(-1)


def np_motion_apply(prev, mask, values, field):
    """The next frame: prev where the mask is clear, pred + value per sample (mod 2^bits) where it is set."""
    out = prev.copy()
    flat = out.reshape(mask.size, -1)
    m = mask.reshape(-1).astype(bool)
    v = np.asarray(values, dtype=prev.dtype).reshape(-1, flat.shape[1])
    flat[m] = np_predict(prev, field).reshape(mask.size, -1)[m] + v
    return out


def np_apply(prev, mask, values, residual):
    out = prev.copy()
    flat = out.reshape(mask.size, -1)
    m = mask.reshape(-1).astype(bool)
    v = np.asarray(values, dtype=prev.dtype).reshape(-1, flat.shape[1])
    flat[m] = (flat[m] + v) if residual else v
    return out


def _texture(h, w, ch, dtype, seed):
    hi = 256 if dtype == np.uint8 else 65536
    shape = (h, w, ch) if ch > 1 else (h, w)
    return np.random.default_rng(seed).integers(0, hi, shape).astype(dtype)


def _shifted(big, h, w, sx, sy, pad=20):
    """The (h, w) view of `big` whose content has moved by (sx, sy) against the view at (pad, pad): curr(y, x) = base(y - sy, x - sx)."""
    return np.ascontiguousarray(big[pad - sy:pad - sy + h, pad - sx:pad - sx + w])


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
    """Frame by frame: keyframes with the CPU keyframe codec; inter frames with the C oracle's mask decode and the numpy apply of their
    vmode on the previously decoded frame."""
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
        mask = mask.reshape(p.h, p.w)
        if p.vmode == 2:
            out.append(np_motion_apply(out[-1], mask, vals, np.frombuffer(zlib.decompress(p.fz), np.int8)))
        else:
            out.append(np_apply(out[-1], mask, vals, p.vmode == 1))
    return out


def _compress(pkg, frames, ki, bs, coder="zlib", yuv=False, coding="motion", mode="lossless"):
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=ki, batch_size=bs, use_direct_yuv=yuv)
    comp.entropy_coder = coder
    comp.value_coding = coding
    if mode != "lossless":
        comp.inter_frame_mode = mode
        comp.inter_frame_threshold = 3.0
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


# ------------------------------------------------------------------ CPU: the model itself
def test_model_finds_a_known_shift_and_prefers_zero_on_flat_content():
    big = _texture(80, 96, 3, np.uint8, 1)
    prev = _shifted(big, 40, 56, 0, 0)
    curr = _shifted(big, 40, 56, 3, -2)                    # content moved 3 right, 2 up: pred = prev(y - 2 .. ) -> (dx, dy) = (-3, 2)
    f = np_motion_search(prev, curr)
    assert (f[0, 0] == (-3, 2)).all() and (f[1, 1] == (-3, 2)).all()
    assert np.array_equal(np_predict(prev, f)[8:30, 8:40], curr[8:30, 8:40])
    flat = np.full((40, 56, 3), 9, np.uint8)
    assert not np_motion_search(flat, flat).any()
    assert not np_motion_search(flat, flat + np.uint8(5)).any()   # every candidate ties: (0, 0)
    g = np.tile(np.arange(56, dtype=np.uint8)[None, :, None], (40, 1, 3))
    assert (np_motion_search(g, g)[..., 1] == 0).all()       # vertical ties go to dy = 0 as well


# ------------------------------------------------------------------ CPU: the RBF4 layout
class _R:
    def __init__(self, raw, k, l, wlen, ones):
        self.raw, self.k, self.l, self.wlen, self.ones = raw, k, l, wlen, ones


FZ = zlib.compress(np.array([1, -2, 16, -16, 0, 0], np.int8).tobytes())


def _layout(raw, vmode, v4=True):
    I = _ivc().ImprovedVideoCompressor
    rng = np.random.default_rng(11)
    bm, wt = rng.integers(0, 256, 300).astype(np.uint8), rng.integers(0, 256, 300).astype(np.uint8)
    r = _R(raw, 0.0 if raw else 1.4142135623730951, 0 if raw else 999, 0 if raw else 333, 41)
    rz = rng.integers(0, 256, 50).astype(np.uint8).tobytes() if raw else None
    return I._inter_layout((17, 29), 1, 3, r, bm, wt, rz, b"value-or-residual-stream", 123, vmode, FZ if vmode == 2 else None, v4), r, bm, wt, rz


@pytest.mark.parametrize("vmode", [0, 1, 2])
@pytest.mark.parametrize("raw", [False, True])
def test_rbf4_layout_round_trips(raw, vmode):
    ivcmod = _ivc()
    pl, r, bm, wt, rz = _layout(raw, vmode)
    hdr = len(ivcmod._INTER_TAG_V4) + struct.calcsize("<IIIBB")
    assert pl.startswith(ivcmod._INTER_TAG_V4) and pl[hdr] == vmode
    p = ivcmod.ImprovedVideoCompressor._parse_inter(pl)
    assert not p.v1 and p.vmode == vmode
    assert (p.h, p.w, p.isz, p.ch, bool(p.raw)) == (17, 29, 1, 3, raw)
    assert (p.k, p.l, p.wlen, p.ones, p.vcount) == (r.k, r.l, r.wlen, 41, 123)
    assert bytes(p.vz) == b"value-or-residual-stream"
    if vmode == 2:
        assert pl[hdr + 1:hdr + 5] == struct.pack("<I", len(FZ)) and bytes(p.fz) == FZ
    else:
        assert p.fz is None
    if raw:
        assert bytes(p.mask_bytes) == rz and bytes(p.witness_bytes) == b""
    else:
        assert bytes(p.mask_bytes) == bm[:(999 + 7) // 8].tobytes() and bytes(p.witness_bytes) == wt[:(333 + 7) // 8].tobytes()


@pytest.mark.parametrize("vmode", [0, 1])
@pytest.mark.parametrize("raw", [False, True])
def test_rbf4_equals_rbf3_apart_from_the_tag(raw, vmode):
    ivcmod = _ivc()
    v4, v3 = _layout(raw, vmode)[0], _layout(raw, vmode, v4=False)[0]
    assert v3.startswith(ivcmod._INTER_TAG_V3) and v4 == ivcmod._INTER_TAG_V4 + v3[len(ivcmod._INTER_TAG_V3):]


def test_vmode_2_needs_rbf4_and_a_field():
    I = _ivc().ImprovedVideoCompressor
    r = _R(True, 0.0, 0, 0, 1)
    for v4, fz in ((False, FZ), (True, None)):
        with pytest.raises(ValueError):
            I._inter_layout((17, 29), 1, 3, r, None, None, b"", b"", 3, 2, fz, v4)


@pytest.mark.parametrize("bad", [3, 7, 255])
def test_rbf4_bad_vmode_raises(bad):
    ivcmod = _ivc()
    pl = bytearray(_layout(False, 1)[0])
    pl[len(ivcmod._INTER_TAG_V4) + struct.calcsize("<IIIBB")] = bad
    with pytest.raises(ValueError, match="value coding"):
        ivcmod.ImprovedVideoCompressor._parse_inter(bytes(pl))


def test_rbf3_still_rejects_vmode_2():
    ivcmod = _ivc()
    pl = _layout(False, 2)[0]
    with pytest.raises(ValueError, match="value coding"):
        ivcmod.ImprovedVideoCompressor._parse_inter(ivcmod._INTER_TAG_V3 + pl[len(ivcmod._INTER_TAG_V4):])


def _motion_payload(h, w, field_bytes, ch=1):
    """A raw-mask RBF4 payload of an (h, w) 8-bit frame with every pixel set to value 0 in vmode 2, and the given field bytes."""
    I = _ivc().ImprovedVideoCompressor
    n = h * w
    r = _R(True, 0.0, 0, 0, n)
    rz = zlib.compress(np.packbits(np.ones(n, np.uint8)).tobytes())
    vz = zlib.compress(bytes(n * ch))
    return I._inter_layout((h, w), 1, ch, r, None, None, rz, vz, n * ch, 2, zlib.compress(field_bytes), True)


def _check(payload, prev):
    ivcmod = _ivc()
    I = ivcmod.ImprovedVideoCompressor
    comp = object.__new__(I)                               # _start_inter / _check_inter need no device
    with ThreadPoolExecutor(2) as pool:
        job = I._start_inter(comp, payload, pool)
        I._check_inter(job, prev)
    return job


def test_bad_fields_raise_value_error():
    h, w = 20, 40                                          # 2 x 3 blocks: 12 field bytes
    prev = np.zeros((h, w), np.uint8)
    good = np.array([1, -1, 16, -16, 0, 0, -16, 16, 5, 5, 0, 1], np.int8)
    job = _check(_motion_payload(h, w, good.tobytes()), prev)
    assert np.array_equal(job.field_arr, good)
    for bad in (good[:-2], np.concatenate([good, good[:2]]), np.zeros(0, np.int8)):
        with pytest.raises(ValueError, match="motion field"):
            _check(_motion_payload(h, w, bad.tobytes()), prev)
    for v in (17, -17, 127, -128):
        b = good.copy()
        b[7] = v
        with pytest.raises(ValueError, match=r"\[-16, 16\]"):
            _check(_motion_payload(h, w, b.tobytes()), prev)
    pl = bytearray(_motion_payload(h, w, good.tobytes()))
    at = len(_ivc()._INTER_TAG_V4) + struct.calcsize("<IIIBB") + 1
    pl[at:at + 4] = struct.pack("<I", 1 << 30)              # a field length past the end of the payload
    with pytest.raises(ValueError, match="motion field"):
        _check(bytes(pl), prev)


# ------------------------------------------------------------------ GPU: motion_search against the model
SHIFTS = [(0, 0), (1, 1), (-1, -1), (1, -1), (-1, 1), (16, -16), (-16, 16), (17, 0)]


@gpu
@pytest.mark.parametrize("ch,dtype", [(1, np.uint8), (3, np.uint8), (1, np.uint16), (3, np.uint16)])
@pytest.mark.parametrize("h,w", [(1, 40), (5, 5), (15, 17), (16, 16), (17, 33), (37, 53), (64, 96)])
def test_motion_search_matches_model(pkg, h, w, ch, dtype):
    big = _texture(h + 40, w + 40, ch, dtype, h * w + ch)
    base = _shifted(big, h, w, 0, 0)
    frames = [base] + [_shifted(big, h, w, sx, sy) for sx, sy in SHIFTS]
    hi = 255 if dtype == np.uint8 else 65535
    frames += [np.full_like(base, hi // 3), np.full_like(base, hi // 2)]   # flat -> flat: every candidate ties
    npairs = len(SHIFTS) + 1
    st = pkg.FrameStream(h, w, ch, dtype, max_frames=len(frames), max_pairs=npairs, k1_only=True, mask_mode=1)
    try:
        st.upload(np.stack(frames))
        st.encode([0] * len(SHIFTS) + [len(frames) - 2], list(range(1, len(SHIFTS) + 1)) + [len(frames) - 1], 0.0)
        got = st.motion_search()
        assert got.shape == (npairs, -(-h // 16), -(-w // 16), 2) and got.dtype == np.int8
        prevs = [base] * len(SHIFTS) + [frames[-2]]
        for j, (p, c) in enumerate(zip(prevs, frames[1:len(SHIFTS) + 1] + [frames[-1]])):
            assert np.array_equal(got[j], np_motion_search(p, c)), (j, SHIFTS[j] if j < len(SHIFTS) else "flat")
        assert not got[-1].any()
        if h >= 48 and w >= 48:                           # an interior block sees the true vector (not (17, 0): out of range)
            for j, (sx, sy) in enumerate(SHIFTS[:-1]):
                assert tuple(got[j, 1, 1]) == (-sx, -sy), j
    finally:
        st.close()


@gpu
def test_motion_search_4k_edges_and_sampled_interior(pkg):
    h, w = 2160, 3840
    rng = np.random.default_rng(4)
    big = np.clip(_texture(h + 40, w + 40, 3, np.uint8, 9).astype(np.int16) // 2 + 64, 0, 255).astype(np.uint8)
    prev = _shifted(big, h, w, 0, 0)
    curr = _shifted(big, h, w, 3, -2)
    noise = rng.integers(-2, 3, curr.shape)
    curr = np.clip(curr.astype(np.int16) + noise, 0, 255).astype(np.uint8)
    st = pkg.FrameStream(h, w, 3, np.uint8, max_frames=2, max_pairs=1, k1_only=True, mask_mode=1)
    try:
        st.upload(np.stack([prev, curr]))
        st.encode([0], [1], 0.0)
        got = st.motion_search()[0]
    finally:
        st.close()
    nby, nbx = got.shape[:2]
    edge = {(y, x) for y in range(nby) for x in (0, nbx - 1)} | {(y, x) for y in (0, nby - 1) for x in range(nbx)}
    interior = [(int(y), int(x)) for y, x in zip(rng.integers(1, nby - 1, 200), rng.integers(1, nbx - 1, 200))]
    blocks = sorted(edge | set(interior))
    ref = np_motion_search(prev, curr, blocks)
    for b in blocks:
        assert tuple(got[b]) == tuple(ref[b]), b
    assert all(tuple(got[b]) == (-3, 2) for b in interior)


# ------------------------------------------------------------------ GPU: the motion_values gather
@gpu
@pytest.mark.parametrize("h,w,ch,dtype", [(37, 53, 1, np.uint8), (37, 53, 3, np.uint8), (45, 91, 1, np.uint16), (37, 53, 3, np.uint16),
                                          (1080, 1920, 3, np.uint8)])
def test_motion_gather_matches_model(pkg, h, w, ch, dtype):
    big = _texture(h + 40, w + 40, ch, dtype, 3 * h + w)
    f0 = _shifted(big, h, w, 0, 0)
    f1 = _shifted(big, h, w, 2, 1)
    f2 = f1.copy()
    sel = np.random.default_rng(5).random((h, w)) < 0.2
    f2[sel] = _texture(h, w, ch, dtype, 6)[sel]
    fr = [f0, f1, f2, f2.copy()]                           # the last pair has an empty mask
    st = pkg.FrameStream(h, w, ch, dtype, max_frames=4, max_pairs=3, k1_only=True, mask_mode=1)
    RbfError = pkg._cabi.RbfError
    try:
        st.upload(np.stack(fr))
        st.encode([0, 1, 2], [1, 2, 3], 0.0)
        masks = [st.fetch(j)[2].reshape(h, w) for j in range(3)]
        with pytest.raises(RbfError):                     # no search since the encode
            st.set_option("motion_values", 1)
        fields = st.motion_search()
        plain = st.gather_changed()
        st.set_option("value_mode", 1)
        with pytest.raises(RbfError):                     # value_mode 1 and motion_values 1 exclude each other
            st.set_option("motion_values", 1)
        st.set_option("value_mode", 0)
        st.set_option("motion_values", 1)
        with pytest.raises(RbfError):
            st.set_option("value_mode", 1)
        for bad in (2, -1):
            with pytest.raises(RbfError):
                st.set_option("motion_values", bad)
        got = st.gather_changed()
        zs = st.zlib_changed()
        st.set_option("motion_values", 0)
        assert all(np.array_equal(x, y) for x, y in zip(st.gather_changed(), plain))        # the option switches back
        for j in range(3):
            exp = np_motion_gather(fr[j], fr[j + 1], masks[j], fields[j])
            assert got[j].dtype == np.dtype(dtype) and np.array_equal(got[j], exp), j
            assert zlib.decompress(zs[j]) == exp.tobytes(), j
        assert got[2].size == 0
        assert (got[0] == 0).mean() > 0.8                  # the pan: zero except where the clamped edge or a search miss leaves a residual
        # a search over fewer pairs than are gathered, and a new encode, both leave the gathers without fields
        st.motion_search(1)
        st.set_option("motion_values", 1)
        with pytest.raises(RbfError):
            st.gather_changed(2)
        assert np.array_equal(st.gather_changed(1)[0], got[0])
        st.encode([0, 1, 2], [1, 2, 3], 0.0)
        with pytest.raises(RbfError):
            st.gather_changed()
        st.set_option("motion_values", 0)
    finally:
        st.close()


# ------------------------------------------------------------------ GPU: apply_chain with motion pairs
MODES = [0, 1, 2, 2, 0, 2]


@gpu
@pytest.mark.parametrize("h,w,ch,dtype", [(37, 53, 1, np.uint8), (37, 53, 3, np.uint8), (45, 91, 1, np.uint16), (67, 129, 3, np.uint16),
                                          (1080, 1920, 3, np.uint8)])
def test_apply_chain_motion_matches_model(pkg, h, w, ch, dtype):
    rng = np.random.default_rng(h * w + ch)
    n, cnt = h * w, len(MODES)
    hi = 256 if dtype == np.uint8 else 65536
    shape = (h, w, ch) if ch > 1 else (h, w)
    masks = [np.zeros(n, np.uint8), (rng.random(n) < 0.3).astype(np.uint8), np.ones(n, np.uint8), (rng.random(n) < 0.5).astype(np.uint8),
             (rng.random(n) < 0.2).astype(np.uint8), (rng.random(n) < 0.05).astype(np.uint8)]
    nb = (-(-h // 16), -(-w // 16), 2)
    fields = [rng.integers(-16, 17, nb).astype(np.int8) if m == 2 else None for m in MODES]
    fields[2][0, 0] = (16, -16)
    vals = [rng.integers(0, hi, int(m.sum()) * ch).astype(dtype) for m in masks]
    base = rng.integers(0, hi, shape).astype(dtype)
    base.reshape(-1)[:5] = hi - 1                          # sums that wrap past the top

    def model(modes, flds):
        out, cur = [], base
        for t in range(cnt):
            m = masks[t].reshape(h, w)
            cur = np_motion_apply(cur, m, vals[t], flds[t]) if modes[t] == 2 else np_apply(cur, m, vals[t], modes[t] == 1)
            out.append(cur)
        return out

    mf = 8
    st = pkg.FrameStream(h, w, ch, dtype, max_frames=mf, max_pairs=cnt, k1_only=True)
    RbfError = pkg._cabi.RbfError
    try:
        consumed, ones = st.decode_masks(_raw_slots(masks, n), np.zeros((cnt, 0), np.uint8), [0] * cnt, [0] * cnt, [0.0] * cnt, [1] * cnt)
        assert list(ones) == [int(m.sum()) for m in masks]
        exp = model(MODES, fields)
        st.upload(base, first=5)                           # the chain writes slots 6, 7, 0, 1, 2, 3
        applied = st.apply_chain(5, vals, modes=MODES, motion=fields)
        assert list(applied) == list(ones)
        got = st.download_batch(6, cnt)
        for t in range(cnt):
            assert np.array_equal(got[t], exp[t]), t
        assert np.array_equal(st.download(5), base)
        # one value too few at motion pair 3, then at plain pair 4: nothing from that pair on is written (sentinels stay)
        for bad in (3, 4):
            short = [v[:-ch] if t == bad else v for t, v in enumerate(vals)]
            st.upload(base, first=0)
            st.upload(np.full((mf - 1,) + shape, 7, dtype=dtype), first=1)
            applied = st.apply_chain(0, short, modes=MODES, motion=fields)
            assert list(applied) == list(ones[:bad]) + [0] * (cnt - bad), bad
            got = st.download_batch(1, cnt)
            for t in range(cnt):
                if t < bad:
                    assert np.array_equal(got[t], exp[t]), (bad, t)
                else:
                    assert (got[t] == 7).all(), (bad, t)
        # all motion, and no motion pair through the same entry point
        st.upload(base, first=0)
        assert list(st.apply_chain(0, vals, modes=[2] * cnt, motion=[fields[2]] * cnt)) == list(ones)
        exp_all = model([2] * cnt, [fields[2]] * cnt)
        got = st.download_batch(1, cnt)
        assert all(np.array_equal(got[t], exp_all[t]) for t in range(cnt))
        st.upload(base, first=0)
        assert list(st.apply_chain(0, vals, modes=[0, 1, 0, 1, 0, 0], motion=fields)) == list(ones)   # fields unused: no motion pair
        exp_none = model([0, 1, 0, 1, 0, 0], fields)
        got = st.download_batch(1, cnt)
        assert all(np.array_equal(got[t], exp_none[t]) for t in range(cnt))
        # no modes: every pair plain, and fields passed anyway are not read
        L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
        buf = np.concatenate([v.view(np.uint8) for v in vals])
        offs = np.concatenate([[0], np.cumsum([v.nbytes for v in vals])]).astype(np.uint64)
        out = np.zeros(cnt, np.uint64)
        ptr = pkg._cabi.ptr
        fl = np.full((cnt,) + nb, 100, np.int8)
        st.upload(base, first=0)
        assert L.rbf_stream_apply_chain(st._h, 0, cnt, ptr(buf), ptr(offs), None, ptr(fl), ptr(out)) == 0
        assert list(out) == list(ones)
        exp_plain = model([0] * cnt, fields)
        got = st.download_batch(1, cnt)
        assert all(np.array_equal(got[t], exp_plain[t]) for t in range(cnt))
        # errors, checked before any launch
        L.rbf_reset_counters(ctx)
        with pytest.raises(ValueError):                    # a motion pair without a field
            st.apply_chain(0, vals, modes=MODES, motion=fields[:3] + [None] + fields[4:])
        with pytest.raises(RbfError):                      # without `motion` the motion pairs reach C without fields
            st.apply_chain(0, vals, modes=MODES)
        with pytest.raises(RbfError):
            st.apply_chain(0, vals, modes=[0, 1, 3, 0, 0, 0], motion=fields)
        fl = np.zeros((cnt,) + nb, np.int8)
        flags = np.array([0, 1, 2, 0, 0, 0], np.uint8)
        assert L.rbf_stream_apply_chain(st._h, 0, cnt, ptr(buf), ptr(offs), ptr(flags), None, ptr(out)) == -1   # mode 2, no fields
        flags[2] = 3
        assert L.rbf_stream_apply_chain(st._h, 0, cnt, ptr(buf), ptr(offs), ptr(flags), ptr(fl), ptr(out)) == -1    # a mode of 3
        for v in (17, -17, -128):
            bad_f = [None if f is None else f.copy() for f in fields]
            bad_f[5][-1, -1, 1] = v
            with pytest.raises(RbfError):
                st.apply_chain(0, vals, modes=MODES, motion=bad_f)
        assert L.rbf_get_counter(ctx, b"kernel_launches") == 0 and L.rbf_get_counter(ctx, b"h2d_bytes") == 0
    finally:
        st.close()


# ------------------------------------------------------------------ compress_video(value_coding="motion") round trips
def _pan_frames(h, w, ch, dtype, nfr, seed, noise=0):
    """A textured pan of 3 px right and 2 px up per frame (frame t+1 (y, x) = frame t (y + 2, x - 3)), optional +-noise."""
    big = _texture(h + 2 * nfr, w + 3 * nfr, ch, dtype, seed)
    rng = np.random.default_rng(seed + 1)
    out = []
    for t in range(nfr):
        f = big[2 * t:2 * t + h, 3 * (nfr - t):3 * (nfr - t) + w]
        if noise:
            hi = 255 if dtype == np.uint8 else 65535
            f = np.clip(f.astype(np.int64) + rng.integers(-noise, noise + 1, f.shape), 0, hi).astype(dtype)
        out.append(np.ascontiguousarray(f))
    return out


def _mixed_frames(h, w, ch, dtype, nfr, seed):
    """A pan for the first half, then synth_stream changes (coded, unchanged, dense, sparse)."""
    pan = _pan_frames(h, w, ch, dtype, nfr // 2 + 1, seed)
    s = synth_stream(h, w, nfr - len(pan) + 1, seed, [0.05, 0.0, 0.4, 0.01], dtype)
    s = [np.ascontiguousarray(x[..., 0]) if ch == 1 else x for x in s]
    d = [((x.astype(np.int64) - s[0] + pan[-1]) % (256 if dtype == np.uint8 else 65536)).astype(dtype) for x in s[1:]]
    return pan + d


@gpu
@pytest.mark.parametrize("h,w,ch,dtype,yuv,nfr,ki,bs,coder,mode", [
    (37, 53, 3, np.uint8, True, 12, 30, 4, "zlib", "lossless"),     # YUV444: one run of 11 in groups of 4, 4, 3
    (64, 64, 3, np.uint8, False, 12, 6, 5, "gpu", "lossless"),      # BGR: runs of 5 = exactly one group each
    (37, 53, 1, np.uint8, False, 7, 30, 1, "zlib", "lossless"),     # groups of one
    (64, 64, 1, np.uint16, False, 11, 5, 3, "gpu", "lossless"),
    (37, 53, 3, np.uint16, False, 10, 30, 7, "zlib", "lossless"),
    (48, 80, 3, np.uint8, True, 9, 30, 4, "zlib", "reference"),
    (48, 80, 3, np.uint8, True, 9, 30, 4, "gpu", "reference"),
    (1080, 1920, 3, np.uint8, True, 6, 30, 3, "gpu", "lossless"),
    (1080, 1920, 3, np.uint8, True, 5, 30, 4, "zlib", "lossless"),
])
def test_motion_round_trip(pkg, co, h, w, ch, dtype, yuv, nfr, ki, bs, coder, mode):
    frames = _mixed_frames(h, w, ch, dtype, nfr, 5)
    if mode == "reference":                                # every change is a multiple of 8 on all channels alike, so above the
        frames = _pan_frames(h, w, 1, np.uint8, nfr, 7)    # threshold on Y: no unflagged pixel changes and every frame stays inter
        frames = [np.ascontiguousarray(np.repeat((f // 8 * 8)[..., None], 3, -1)) for f in frames]
    if yuv:
        frames = [pkg.YUVFrame(f) for f in frames]
    comp, payloads = _compress(pkg, frames, ki, bs, coder, yuv, mode=mode)
    ivcmod = _ivc()
    vm = _vmodes(payloads)
    inter = [p for p in payloads if p.startswith(ivcmod._INTER_TAGS)]
    assert inter and all(p.startswith(ivcmod._INTER_TAG_V4) for p in inter)
    if mode == "lossless":
        assert len(inter) == nfr - (nfr + ki - 1) // ki
    if h * w * ch > 3000:
        assert 2 in vm
    _check_round_trip(co, comp, frames, payloads, yuv)


def _gradient(h, w):
    yy, xx = np.mgrid[0:h, 0:w]
    g = ((yy + 2 * xx) // 3) % 256
    return np.stack([g, (g + 40) % 256, (255 - g)], -1).astype(np.uint8)


@gpu
@pytest.mark.parametrize("coder", ["zlib", "gpu"])
def test_choice_is_pinned_by_content(pkg, co, coder):
    """Random texture -> panned 3 right, 2 up: motion residuals are zero but at the entering edges -> 2.  -> the same + 1 on every
    sample: co-located residuals are all ones, the motion ones equal them plus a field to store -> 1.  -> a cut to a smooth gradient:
    the values compress, both residuals are noise -> 0."""
    h, w = 120, 160
    p0, p1 = _pan_frames(h, w, 3, np.uint8, 2, 1)
    frames = [p0, p1, p1 + np.uint8(1), _gradient(h, w)]
    comp, pls = _compress(pkg, frames, 30, 8, coder)
    assert _vmodes(pls) == [None, 2, 1, 0]
    _check_round_trip(co, comp, frames, pls, False)


@gpu
@pytest.mark.parametrize("coder", ["zlib", "gpu"])
def test_motion_payload_is_never_longer_than_adaptive(pkg, coder):
    frames = _mixed_frames(64, 96, 3, np.uint8, 12, 17)
    frames += _pan_frames(64, 96, 3, np.uint8, 4, 3, noise=2)
    _, adapt = _compress(pkg, frames, 30, 4, coder, coding="adaptive")
    _, mot = _compress(pkg, frames, 30, 4, coder)
    vm = _vmodes(mot)
    assert 2 in vm and (0 in vm or 1 in vm)
    ivcmod = _ivc()
    t3, t4 = ivcmod._INTER_TAG_V3, ivcmod._INTER_TAG_V4
    for i, (a, b) in enumerate(zip(adapt, mot)):
        if vm[i] is None:
            assert a == b                                  # keyframes
        elif vm[i] == 2:
            assert len(b) < len(a), i
        else:
            assert a.startswith(t3) and b == t4 + a[len(t3):], i


@gpu
def test_value_coding_motion_is_accepted_and_others_are_not(pkg):
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=30)
    comp.value_coding = "motion-compensated"
    with pytest.raises(ValueError, match="value_coding"):
        comp.compress_video([np.zeros((16, 16, 3), np.uint8)] * 2)


# ------------------------------------------------------------------ counters: a motion group costs its field bytes and its split
@gpu
def test_counters_against_adaptive(pkg):
    """Per decoded group, against the same frames coded "adaptive": h2d_bytes grow by the group's field bytes (count x blocks x 2) when
    it holds a motion pair, d2h_bytes are equal, and kernel launches grow by (runs + motion pairs - 1), where runs are the maximal runs
    of non-motion pairs: the adaptive group launches tile count + tile scan + one sweep, the motion group tile count + tile scan + one
    sweep per run + one k_apply_motion per motion pair.  Each group is decoded on its own so that the counters are per group."""
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    h, w = 120, 160
    frames = _mixed_frames(h, w, 3, np.uint8, 14, 37)
    bs = 5
    _, ad = _compress(pkg, frames, 30, bs, coding="adaptive")
    _, mo = _compress(pkg, frames, 30, bs)
    vm = _vmodes(mo)
    assert 2 in vm and 1 in vm + _vmodes(ad)
    nblk = -(-h // 16) * -(-w // 16)
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=30, batch_size=bs)
    seen_motion = False
    for g0 in range(1, len(frames), bs):
        counts = {}
        for name, pls in (("adaptive", ad), ("motion", mo)):
            # the group's frames after a keyframe of its base frame, so that each group is one decode_masks + one apply_chain
            key = _compress(pkg, [frames[g0 - 1]], 30, bs, coding="plain")[1][0]
            L.rbf_reset_counters(ctx)
            dec = comp.decompress_video(compressed_frames=[key] + pls[g0:g0 + bs])
            counts[name] = [L.rbf_get_counter(ctx, k) for k in (b"kernel_launches", b"h2d_bytes", b"d2h_bytes")]
            assert all(np.array_equal(np.asarray(d), f) for d, f in zip(dec, frames[g0 - 1:g0 + bs]))
        modes = vm[g0:g0 + bs]
        mp = modes.count(2)
        runs = sum(1 for t, m in enumerate(modes) if m != 2 and (t == 0 or modes[t - 1] == 2))
        a, m = counts["adaptive"], counts["motion"]
        assert m[2] == a[2], (g0, counts)
        if mp:
            seen_motion = True
            assert m[1] - a[1] == len(modes) * nblk * 2, (g0, modes, counts)
            assert m[0] - a[0] == runs + mp - 1, (g0, modes, counts)
        else:
            assert m == a, (g0, counts)
    assert seen_motion
