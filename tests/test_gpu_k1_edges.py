"""K1, the frame-difference mask, against a plain numpy statement of the reference's mask (ivc:788-808) at every byte lane,
threshold edge, kernel and frame-size boundary; the full encode at the mask's extremes; and the default lossless GOP path on
chroma-only changes.

Every later stage (Bloom insert, query, witness, value gather, GOP decode) codes the mask K1 produced, so a wrong mask bit
survives every round trip.  The numpy reference below is pinned, case for case, to the fixtures taken from the original code
(frames_kat.json, gray_kat.json) by the CPU tests, and the GPU tests compare K1 with it.

Kernels reached (rbf_k1_threshold.cuh): one pair or a pair list that is not a chain -> k_threshold; a chain of >= 2 pairs ->
k_threshold_sweep; k1_variant 1 with npix >= TMA tile -> k_threshold_tma + k_threshold_tail (8-bit 1-channel frames are routed
away from TMA by the WPW <= 32 guard)."""
import contextlib
import math
import re
import zlib
from pathlib import Path

import numpy as np
import pytest

from tests.util import golden_json, golden_pair, gray_cube, gray_pair, sha

gpu = pytest.mark.gpu


# ------------------------------------------------------------------ the numpy reference (ivc:788-808)
def bgr2gray(a):
    """cv2.COLOR_BGR2GRAY of 8- and 16-bit samples: OpenCV's 15-bit fixed point (ivc:794-795)."""
    x = a.astype(np.uint32)
    return ((x[..., 0] * 3735 + x[..., 1] * 19235 + x[..., 2] * 9798 + 16384) >> 15).astype(a.dtype)


def ref_diff(prev, curr, gray=False):
    """-> (|Y_prev - Y_curr| exactly as ivc:801 computes it, in int16 with its wrap-around, as float64; anyd: some byte of the
    pixel differs).  Y is the single plane, channel 0, or the gray conversion of the three samples."""
    if prev.ndim == 2:
        yp, yc = prev, curr
    elif gray:
        yp, yc = bgr2gray(prev), bgr2gray(curr)
    else:
        yp, yc = prev[..., 0], curr[..., 0]
    diff = np.abs(yp.astype(np.int16) - yc.astype(np.int16))    # abs(int16(-32768)) stays -32768
    anyd = prev != curr
    if prev.ndim == 3:
        anyd = anyd.any(axis=2)
    return diff.astype(np.float64), anyd


def ref_mask(diff, anyd, thr, mask_mode=0):
    """-> (mask bool, ones, resid).  `diff > threshold` with the Python float (ivc:808): NaN and +-inf compare as in float64."""
    with np.errstate(invalid="ignore"):
        m = diff > float(thr)
    if mask_mode:
        m = m | anyd
    return m, int(m.sum()), int((anyd & ~m).sum())


def test_reference_reproduces_frames_kat():
    for rec in golden_json("frames_kat.json")["cases"]:
        prev, curr = golden_pair(rec)
        m, ones, _ = ref_mask(*ref_diff(prev, curr), rec["threshold"])
        assert ones == rec["ones"], rec["name"]
        assert sha(np.packbits(m.reshape(-1))) == rec["mask_sha256"], rec["name"]
        if "wrap_mask_head" in rec:
            assert [int(x) for x in m[0, :5]] == rec["wrap_mask_head"], rec["name"]


def test_reference_reproduces_gray_kat():
    g = golden_json("gray_kat.json")
    cube = gray_cube()
    assert sha(bgr2gray(cube)) == g["cube_u8_sha256"]
    assert sha(bgr2gray(cube.astype(np.uint16) * 257)) == g["cube_u16_sha256"]
    explicit = [rec for rec in g["cases"] if rec["threshold"] is not None]
    assert len(explicit) == len(g["cases"]) - 2                  # the two adaptive cases need the device median
    for rec in explicit:
        prev, curr = gray_pair(rec)
        assert sha(bgr2gray(curr)) == rec["gray_curr_sha256"], rec["name"]
        m, ones, _ = ref_mask(*ref_diff(prev, curr, gray=True), rec["threshold"])
        assert ones == rec["ones"], rec["name"]
        assert sha(np.packbits(m.reshape(-1))) == rec["mask_sha256"], rec["name"]


def test_reference_threshold_semantics():
    """The edges the kernels encode by hand: the int16 wrap (|dY| = 32768 is -32768, 65535 is 1), NaN and the infinities."""
    prev = np.array([[0, 65535, 0, 32768, 32767, 5]], dtype=np.uint16)
    curr = np.array([[32768, 0, 1, 0, 65535, 5]], dtype=np.uint16)
    diff, anyd = ref_diff(prev, curr)
    assert diff.tolist() == [[-32768.0, 1.0, 1.0, -32768.0, -32768.0, 0.0]]
    assert ref_mask(diff, anyd, -32768.0)[0].tolist() == [[False, True, True, False, False, True]]
    assert ref_mask(diff, anyd, -32768.5)[1] == 6
    assert ref_mask(diff, anyd, -1.0)[0].tolist() == [[False, True, True, False, False, True]]
    assert ref_mask(diff, anyd, math.nan)[1:] == (0, 5)
    assert ref_mask(diff, anyd, -math.inf)[1] == 6 and ref_mask(diff, anyd, math.inf)[1] == 0
    assert ref_mask(diff, anyd, math.nan, mask_mode=1)[1:] == (5, 0)


# ------------------------------------------------------------------ kernel geometry (pinned to the header below)
TMA_TILE_BYTES = 12288        # k_threshold_tma: bytes per frame per stage; TP = TMA_TILE_BYTES / PB pixels per tile
SW_TILE_PX = 4096             # k_threshold_sweep: pixels per tile
SW_STAGES = 4                 # k_threshold_sweep: ring slots
WARP_STAGE_PX = 1024          # k_threshold: a warp stages its 32 words only when all 1024 pixels lie in the frame


def test_kernel_constants_match_header():
    src = (Path(__file__).resolve().parents[1] / "new_bloom_filter_repo_b200" / "csrc" / "rbf_k1_threshold.cuh").read_text()

    def const(name):
        return re.search(r"constexpr\s+\w+\s+%s\s*=\s*([^;]+);" % name, src).group(1).strip()
    assert int(const("TMA_TILE_BYTES")) == TMA_TILE_BYTES
    assert const("SW_TILE_PX") == "32u * SW_THREADS" and 32 * int(const("SW_THREADS")) == SW_TILE_PX
    assert int(const("SW_STAGES")) == SW_STAGES
    assert int(const("TMA_THREADS")) == 256 and int(const("K1_THREADS")) == 256
    assert "(w | 31u) + 1u) * 32u <= npix" in src                 # the staging condition WARP_STAGE_PX stands for


# ------------------------------------------------------------------ byte-lane probe frames
FORMATS = {"u8x1": (1, np.uint8), "u16x1": (1, np.uint16), "u8x3": (3, np.uint8), "u16x3": (3, np.uint16)}
Y_EDGES = {np.uint8: (0, 1, 2, 126, 127, 128, 129, 253, 254, 255),
           np.uint16: (0, 1, 2, 126, 127, 128, 129, 253, 254, 255, 256, 257, 32766, 32767, 32768, 32769, 65534, 65535)}
Y_BASES = {np.uint8: (0, 1, 77, 255), np.uint16: (0x0000, 0x00ff, 0x0100, 0x1234, 0x7fff, 0x8000, 0xffff)}
# xor patterns of one chroma sample: each bit end of each byte; for 16-bit the low byte only, the high byte only, and both
C_XORS = {np.uint8: (0x01, 0x80), np.uint16: (0x0001, 0x0080, 0x0100, 0x8000, 0x0101)}


def _pb(fmt):
    c, dt = FORMATS[fmt]
    return c * np.dtype(dt).itemsize


def _y_pairs(dt):
    """(prev_y, curr_y): every |dY| of the edge set, prev above and below curr, from several bases (so that 16-bit changes hit the
    low byte only, the high byte only, and both)."""
    hi = np.iinfo(dt).max
    out = set()
    for d in Y_EDGES[dt]:
        for b in Y_BASES[dt]:
            lo = min(b, hi - d)
            out.add((lo, lo + d))
            out.add((lo + d, lo))
    return sorted(out)


def _chroma_xors(channels, dt):
    if channels == 1:
        return [()]
    out = [(0, 0)]
    for x in C_XORS[dt]:
        out += [(x, 0), (0, x)]
    out.append((C_XORS[dt][0], C_XORS[dt][-1]))
    return out


def templates(fmt):
    """(prev_y, curr_y, chroma xors): every Y pair with every chroma pattern, plus unchanged pixels for a fifth of the total."""
    c, dt = FORMATS[fmt]
    tp = [(yp, yc, cx) for yp, yc in _y_pairs(dt) for cx in _chroma_xors(c, dt)]
    return tp + [(b, b, _chroma_xors(c, dt)[0]) for b in Y_BASES[dt]] * (len(tp) // 4 // len(Y_BASES[dt]))


def probe_npix(fmt):
    """A ragged frame size whose full words hold every template at every position of a mask word."""
    return 32 * len(templates(fmt)) + 19


def probe_pair(fmt, npix, shift=0):
    """(prev, curr) [npix, C] (or [npix] for one channel).  Pixel i holds template (i // 32 + 7 * (i % 32) + shift) mod T, so
    once there are T whole words every template sits at every bit of a mask word and every byte lane of yuv8_group4, next to
    different templates (unchanged, chroma-only, Y changes) in the same word.  The ragged last word carries single-byte probes:
    its last pixel changes only byte PB-1 (the frame's last byte), the pixel before it only byte PB-2, and so on."""
    c, dt = FORMATS[fmt]
    hi = int(np.iinfo(dt).max) + 1
    tp = templates(fmt)
    T = len(tp)
    yp = np.array([t[0] for t in tp], dtype=dt)
    yc = np.array([t[1] for t in tp], dtype=dt)
    i = np.arange(npix, dtype=np.int64)
    idx = (i // 32 + 7 * (i % 32) + shift) % T
    prev = np.empty((npix, c), dtype=dt)
    curr = np.empty((npix, c), dtype=dt)
    prev[:, 0], curr[:, 0] = yp[idx], yc[idx]
    if c == 3:
        cx = np.array([t[2] for t in tp], dtype=dt)
        base = ((i[:, None] * np.array([40503, 9973]) + np.array([12345, 321])) % hi).astype(dt)
        prev[:, 1:] = base
        curr[:, 1:] = base ^ cx[idx]
    r = npix % 32
    if r:
        pb = _pb(fmt)
        pv, cv = prev.view(np.uint8).reshape(npix, pb), curr.view(np.uint8).reshape(npix, pb)
        for q in range(min(r, pb)):
            px = npix - 1 - q
            cv[px] = pv[px]
            cv[px, (pb - 1 - q + shift) % pb] ^= 0x80 if q % 2 else 0x01
    if c == 1:
        return prev[:, 0].copy(), curr[:, 0].copy()
    return prev, curr


def probe_chain(fmt, npix, nfr):
    """nfr frames [nfr, npix(, C)]: the probe pair, then frame t = frame t-2 with byte t % PB of the last pixel flipped, so every
    pair of the chain is the probe pair (either way round) and, over the chain, every byte of the last pixel changes."""
    p, c = probe_pair(fmt, npix)
    out = [p, c]
    pb = _pb(fmt)
    for t in range(2, nfr):
        f = out[t - 2].copy()
        f.view(np.uint8).reshape(npix, pb)[npix - 1, t % pb] ^= 0x40
        out.append(f)
    return np.stack(out[:nfr])


def _changed_bytes(prev, curr, pb):
    x = prev.view(np.uint8).reshape(-1, pb) != curr.view(np.uint8).reshape(-1, pb)
    return (x * (1 << np.arange(pb))).sum(axis=1)


@pytest.mark.parametrize("fmt", list(FORMATS))
def test_probe_pair_covers_every_lane_byte_and_delta(fmt):
    c, dt = FORMATS[fmt]
    isz = np.dtype(dt).itemsize
    pb = _pb(fmt)
    npix = probe_npix(fmt)
    prev, curr = probe_pair(fmt, npix)
    full = npix - npix % 32
    pos = np.arange(npix) % 32
    y0 = prev.reshape(npix, c)[:, 0].astype(np.int64)
    y1 = curr.reshape(npix, c)[:, 0].astype(np.int64)
    dy = y1 - y0
    cb = _changed_bytes(prev, curr, pb)
    ymask = (1 << isz) - 1
    chroma = cb >> isz                                          # changed bytes of samples 1, 2
    seen = set(zip(pos[:full].tolist(), dy[:full].tolist(), chroma[:full].tolist()))
    # every signed delta of the edge set at every bit of a mask word (so at every byte lane), crossed with every chroma pattern:
    # none, one chroma sample (16-bit: its low byte, its high byte, both), and both chroma samples
    deltas = {s * d for d in Y_EDGES[dt] for s in (1, -1)}
    chroma_pats = {0}
    if c == 3:
        one = {1, 2, 3} if isz == 2 else {1}
        chroma_pats |= one | {s << isz for s in one} | {1 | (3 << isz) if isz == 2 else 0b11}
    for p in range(32):
        for d in deltas:
            for ch in chroma_pats:
                assert (p, d, ch) in seen, (p, d, ch)
    # every single byte of the pixel changing alone, and for 16-bit Y its low byte only, its high byte only, and both
    for p in range(32):
        at = cb[:full][pos[:full] == p]
        for q in range(pb):
            assert (at == (1 << q)).any(), (p, q)
        ypats = {int(v) for v in (at & ymask)}
        assert ypats >= ({1, 2, 3} if isz == 2 else {1}), (p, ypats)
    # unsigned byte SIMD and the int16 wrap: a Y delta of 255 both ways, and 16-bit deltas that wrap
    assert {255, -255} <= set(dy.tolist())
    if isz == 2:
        assert {32768, -32768, 65535, -65535} <= set(dy.tolist())
        diff, _ = ref_diff(y0.astype(dt)[None], y1.astype(dt)[None])
        assert (diff == -32768).any() and (diff[0][np.abs(dy) == 65535] == 1).all()
    # interleaving: words that hold unchanged pixels, Y changes and (3 channels) chroma-only changes side by side
    words = cb[:full].reshape(-1, 32)
    mixed = (words == 0).any(axis=1) & ((words & ymask) != 0).any(axis=1)
    if c == 3:
        mixed &= (((words & ymask) == 0) & (words != 0)).any(axis=1)
    assert mixed.mean() > 0.1
    # the ragged last word: its last pixels change only the last byte, the one before it, ...
    assert npix % 32
    for q in range(min(npix % 32, pb)):
        assert cb[npix - 1 - q] == 1 << (pb - 1 - q), q


@pytest.mark.parametrize("fmt", list(FORMATS))
def test_probe_chain_pairs(fmt):
    pb = _pb(fmt)
    npix = 4097
    fr = probe_chain(fmt, npix, pb + 2)
    p, c = probe_pair(fmt, npix)
    assert np.array_equal(fr[0], p) and np.array_equal(fr[1], c)
    base = _changed_bytes(p, c, pb)
    last = 0
    for t in range(1, len(fr)):
        cb = _changed_bytes(fr[t - 1], fr[t], pb)
        assert np.array_equal(cb[:-1], base[:-1]), t            # every pair is the probe pair, either way round ...
        last |= int(cb[-1])
    assert last == (1 << pb) - 1                                # ... and every byte of the last pixel changes in some pair


# ------------------------------------------------------------------ thresholds and the sizes where the kernels change course
THRESHOLDS = [-math.inf, -1e12, -40000.5, -32769.0, -32768.5, -32768.0, -2.0, -1.5, -1.0, -0.5, 0.0, 0.5, 1.0, 126.5, 253.5,
              254.0, 254.5, 255.0, 256.0, 32767.0, 32768.0, 65535.0, 1e9, 1e12, math.inf, math.nan]
# one threshold per branch of threshold_to_int / k1_thr, for the size sweeps and the big frames
EDGE_THRESHOLDS = [-math.inf, -32768.5, -32768.0, -1.0, 0.0, 126.5, 254.0, 255.0, 32767.0, 1e12, math.nan]


def test_threshold_lists_reach_every_branch():
    """threshold_to_int: NaN, < -1 (16-bit: < -40000, floor), > 1e9, floor; k1_thr: < 0, 0..254, > 254."""
    for ths in (THRESHOLDS, EDGE_THRESHOLDS):
        assert any(math.isnan(t) for t in ths)
        assert any(t < -40000 for t in ths) and any(-40000 <= t < -1 for t in ths)
        assert any(t > 1e9 for t in ths) and any(-1 <= t <= 1e9 for t in ths)
        fl = {math.floor(t) for t in ths if -1 <= t <= 1e9}
        assert -1 in fl and 0 in fl and 254 in fl and 255 in fl and any(0 < f < 254 for f in fl)
        assert -32768.0 in ths and -32768.5 in ths             # |dY| = -32768 (16-bit wrap): not above -32768, above -32768.5


def _tp(fmt):
    return TMA_TILE_BYTES // _pb(fmt)


def _tiny_npix(fmt):
    return {1: 15, 2: 7, 3: 5, 6: 2}[_pb(fmt)]                   # a frame of fewer than 16 bytes


SIZE_CASES = [(fmt, npix) for fmt in FORMATS
              for npix in sorted({WARP_STAGE_PX - 1, WARP_STAGE_PX, WARP_STAGE_PX + 1, SW_TILE_PX - 1, SW_TILE_PX, SW_TILE_PX + 1,
                                  _tp(fmt) - 1, _tp(fmt), _tp(fmt) + 1, _tiny_npix(fmt), 31})]

# kernel -> (prev indices, curr indices, k1_variant)
KERNELS = {
    "pair": ([0], [1], 0),                                      # k_threshold, one pair
    "list": ([1, 0], [2, 2], 0),                                # k_threshold, pairs that are not a chain
    "chain2": ([0, 1], [1, 2], 0),                              # k_threshold_sweep: 3 frames
    "chain3": ([0, 1, 2], [1, 2, 3], 0),                        # 4 frames: a multiple of SW_STAGES
    "chain4": ([0, 1, 2, 3], [1, 2, 3, 4], 0),
    "chain5": ([0, 1, 2, 3, 4], [1, 2, 3, 4, 5], 0),
    "revisit": ([0, 1, 0], [1, 0, 1], 0),                       # a chain that comes back to frame 0
    "tma": ([0, 1, 2], [1, 2, 3], 1),                           # k_threshold_tma + tail when npix >= TP (else routed away)
}


def test_size_cases_hit_every_boundary():
    for fmt in FORMATS:
        sizes = {n for f, n in SIZE_CASES if f == fmt}
        assert {1023, 1024, 1025, 4095, 4096, 4097} <= sizes
        assert {_tp(fmt) - 1, _tp(fmt), _tp(fmt) + 1} <= sizes
        assert _tiny_npix(fmt) * _pb(fmt) < 16 and 31 in sizes
    assert any(len(p) % SW_STAGES == SW_STAGES - 1 for p, _, _ in KERNELS.values())     # nfr = P + 1 a multiple of SW_STAGES
    assert any((len(p) + 1) % SW_STAGES for p, _, _ in KERNELS.values())


# ------------------------------------------------------------------ GPU: K1 against the reference
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


@contextlib.contextmanager
def ctx_option(pkg, key, value, default):
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    pkg._cabi.check(L.rbf_set_option(ctx, key.encode(), int(value)), ctx)
    try:
        yield
    finally:
        pkg._cabi.check(L.rbf_set_option(ctx, key.encode(), int(default)), ctx)


def _as_frames(fmt, flat, h, w):
    c, _ = FORMATS[fmt]
    return flat.reshape((flat.shape[0], h, w, c) if c == 3 else (flat.shape[0], h, w))


def _check_k1(pkg, fmt, frames, kernels, thresholds, modes, ctas_per_sm=None):
    """Upload `frames` once; for every kernel, mode (mask_mode, gray) and threshold compare every mask bit, the padding bits past
    npix in the last mask byte, `ones` and `resid` with the reference."""
    c, dt = FORMATS[fmt]
    nfr, h, w = frames.shape[:3]
    npix = h * w
    st = pkg.FrameStream(h, w, c, dt, max_frames=nfr, max_pairs=8, k1_only=True)
    cache = {}
    try:
        st.upload(frames)
        for kname in kernels:
            prev_idx, curr_idx, variant = KERNELS[kname]
            if max(prev_idx + curr_idx) >= nfr:
                continue
            with contextlib.ExitStack() as es:
                es.enter_context(ctx_option(pkg, "k1_variant", variant, 0))
                if ctas_per_sm is not None:
                    es.enter_context(ctx_option(pkg, "k1_ctas_per_sm", ctas_per_sm, 32))
                for mask_mode, gray in modes:
                    st.set_option("mask_mode", mask_mode)
                    st.set_option("gray_mode", int(gray))
                    for thr in thresholds:
                        res = st.encode(prev_idx, curr_idx, thr)
                        _, _, mk = st.fetch_batch(0, len(prev_idx), want_masks=True)
                        for t, (a, b) in enumerate(zip(prev_idx, curr_idx)):
                            key = (a, b, gray)
                            if key not in cache:
                                cache[key] = ref_diff(frames[a], frames[b], gray)
                            em, eones, eresid = ref_mask(*cache[key], thr, mask_mode)
                            bits = np.unpackbits(mk[t], bitorder="little")
                            where = (fmt, npix, kname, mask_mode, gray, thr, t)
                            bad = np.flatnonzero(bits[:npix] != em.reshape(-1))
                            assert bad.size == 0, (where, "first wrong mask bits", bad[:8].tolist())
                            assert not bits[npix:].any(), (where, "padding bits past npix are set")
                            assert (res[t].ones, res[t].resid) == (eones, eresid), where
    finally:
        st.close()


def _modes(fmt):
    return [(0, False), (1, False)] + ([(0, True), (1, True)] if FORMATS[fmt][0] == 3 else [])


@gpu
@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("fmt", list(FORMATS))
def test_k1_probe_frames_every_threshold(pkg, fmt, kernel):
    """The full probe frames (every template at every mask bit and byte lane) at all 26 thresholds, both mask modes and gray."""
    npix = probe_npix(fmt)
    frames = _as_frames(fmt, probe_chain(fmt, npix, 6), 1, npix)
    _check_k1(pkg, fmt, frames, [kernel], THRESHOLDS, _modes(fmt))


@gpu
@pytest.mark.parametrize("fmt,npix", SIZE_CASES)
def test_k1_boundary_sizes(pkg, fmt, npix):
    """Warp staging (1023/1024/1025 px), the sweep tile (4095/4096/4097), the TMA tile (TP-1/TP/TP+1), frames under 16 bytes and
    under 32 pixels, through every kernel."""
    frames = _as_frames(fmt, probe_chain(fmt, npix, 6), 1, npix)
    _check_k1(pkg, fmt, frames, list(KERNELS), EDGE_THRESHOLDS, _modes(fmt))


@gpu
@pytest.mark.parametrize("fmt", list(FORMATS))
def test_k1_ragged_1080p_chain_one_cta_per_sm(pkg, fmt):
    """1080x1917 (2 070 360 px: neither whole tiles nor whole words) as a chain of 4 pairs with one sweep CTA per SM, so every
    CTA walks several tiles through the mbarrier ring; then through the TMA variant."""
    h, w = 1080, 1917
    frames = _as_frames(fmt, probe_chain(fmt, h * w, 5), h, w)
    _check_k1(pkg, fmt, frames, ["chain4"], [-32768.0, 0.0, 254.0, math.nan], [(0, False), (1, False)], ctas_per_sm=1)
    _check_k1(pkg, fmt, frames, ["tma", "list"], [0.0, 254.0], [(0, False), (1, False)])


@gpu
def test_k1_4k_chain(pkg):
    h, w = 2160, 3840
    frames = _as_frames("u8x3", probe_chain("u8x3", h * w, 4), h, w)
    _check_k1(pkg, "u8x3", frames, ["chain3", "tma"], [-1.0, 0.0, 254.0], [(0, False), (1, False), (0, True)])


# ------------------------------------------------------------------ GPU: the full encode at the mask's extremes
@gpu
@pytest.mark.parametrize("fmt", list(FORMATS))
@pytest.mark.parametrize("case", ["all", "empty", "first", "last"])
def test_encode_at_mask_extremes(pkg, co, fmt, case):
    """All ones (p = 1, raw), empty (raw), one pixel at index 0 and one at npix-1 (coded with a tiny l): (raw, l, k, wlen), the
    bitmap and the witness equal co.compress of the reference mask, and the GPU decode of every pair gives the mask back."""
    c, dt = FORMATS[fmt]
    h, w = 37, 53                                               # 1961 px: p = 1/1961 is above 0.0001, the last word is ragged
    npix = h * w
    rng = np.random.default_rng(7)
    shape = (h, w, c) if c == 3 else (h, w)
    prev = rng.integers(0, np.iinfo(dt).max + 1, shape).astype(dt)
    curr = prev.copy()
    fl = curr.reshape(npix, c)
    if case in ("all", "empty"):
        fl[rng.random(npix) < 0.3, 0] ^= 1
        thr = -math.inf if case == "all" else math.inf
    else:
        at = 0 if case == "first" else npix - 1
        fl[at, 0] = prev.reshape(npix, c)[at, 0] ^ 0x40         # |dY| = 64
        if c == 3:
            fl[1::7, 1] ^= 1                                    # chroma-only changes: residuals, not mask bits
        thr = 63.5
    st = pkg.FrameStream(h, w, c, dt, max_frames=2)
    try:
        st.upload(np.stack([prev, curr]))
        r = st.encode([0], [1], thr)[0]
        bms, wts, mks = st.fetch_batch(0, 1, want_masks=True)
        em, eones, eresid = ref_mask(*ref_diff(prev, curr), thr)
        flat = em.reshape(-1).astype(np.uint8)
        assert np.array_equal(np.unpackbits(mks[0], bitorder="little")[:npix], flat)
        assert (r.ones, r.resid) == (eones, eresid)
        assert eones == {"all": npix, "empty": 0}.get(case, 1)
        ob, ow, op, on, oratio, ok, ol = co.compress(flat)
        assert (r.raw, r.l, r.k, r.wlen) == (ok == 0, ol, ok, len(ow)), (case, r, ol, ok, len(ow))
        assert r.p == op and (case != "all" or r.p == 1.0)
        if not r.raw:
            assert 0 < r.l < 64, r.l                            # a one-pixel mask: a filter of a few dozen bits
            nb, nw = (ol + 7) // 8, (len(ow) + 7) // 8
            assert np.array_equal(bms[0, :nb], np.packbits(ob)) and not bms[0, nb:].any()
            assert np.array_equal(wts[0, :nw], np.packbits(ow)) and not wts[0, nw:].any()
            assert np.array_equal(co.decompress(ob, ow, npix, ok), flat)
        assert not st.decode_verify().any()
    finally:
        st.close()


# ------------------------------------------------------------------ GPU: the lossless GOP path on chroma-only changes
def gop_clip(kind, h, w):
    """f0; f1 chroma-only changes in every byte lane; f2 the chroma of every pixel (p = 1: a raw mask); f3 = f2; f4 one chroma
    change at the last pixel; f5 luma-only and luma+chroma changes.  16-bit clips change only the high or only the low byte of
    a chroma sample."""
    dt = np.uint16 if kind == "u16" else np.uint8
    rng = np.random.default_rng(11)
    npix = h * w
    i = np.arange(npix)
    f0 = rng.integers(0, np.iinfo(dt).max + 1, (npix, 3)).astype(dt)
    if dt == np.uint16:                                         # one bit of the low byte (odd pixels: of the high byte)
        xo = (np.where(i % 2, 0x0100, 0x0001) << (i // 2 % 8)).astype(dt)
    else:
        xo = (1 << (i % 8)).astype(dt)
    f1 = f0.copy()
    sel = (i % 9 == 1) | (i % 9 == 4)                           # every position mod 32, and p = 2/9: a coded mask
    f1[sel & (i % 2 == 0), 1] ^= xo[sel & (i % 2 == 0)]
    f1[sel & (i % 2 == 1), 2] ^= xo[sel & (i % 2 == 1)]
    f2 = f1.copy()
    f2[i, 1 + i % 2] ^= xo
    f3 = f2.copy()
    f4 = f3.copy()
    f4[npix - 1, 2] ^= xo[npix - 2]
    f5 = f4.copy()
    luma = i % 7 == 3
    f5[luma, 0] = f5[luma, 0] + dt(9)                          # |dY| = 9 (mod 2^bits)
    both = luma & (i % 2 == 0)
    f5[both, 1] ^= xo[both]
    return [f.reshape(h, w, 3) for f in (f0, f1, f2, f3, f4, f5)]


def _inter_mask(co, ivc, payload, n):
    p = ivc.ImprovedVideoCompressor._parse_inter(payload)
    if p.raw:
        mask = np.unpackbits(np.frombuffer(zlib.decompress(p.mask_bytes), dtype=np.uint8))[:n]
    else:
        bm = np.unpackbits(np.frombuffer(p.mask_bytes, dtype=np.uint8))[:p.l]
        wt = np.unpackbits(np.frombuffer(p.witness_bytes, dtype=np.uint8))[:p.wlen]
        mask = co.decompress(bm, wt, n, p.k)
    return p, mask


def _compress_gop(pkg, kind, frames, bs, coder, vc, mode):
    yuv = kind == "yuv"
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=30, batch_size=bs, use_direct_yuv=yuv)
    comp.entropy_coder, comp.value_coding = coder, vc
    comp.inter_frame_mode, comp.inter_frame_threshold = mode, 3.0
    ins = [pkg.YUVFrame(f.copy()) for f in frames] if yuv else [f.copy() for f in frames]
    stats = comp.compress_video(ins, input_color_space="YUV" if yuv else "BGR")
    pls = list(comp._last_compressed_frames)
    dec = comp.decompress_video(compressed_frames=pls)
    assert len(dec) == len(frames)
    for i, (d, f) in enumerate(zip(dec, frames)):
        assert hasattr(d, "yuv_info") == yuv, i
        dd = d.data if yuv else d
        assert dd.dtype == f.dtype and np.array_equal(dd, f), (mode, i)
    return stats, pls


GOP_CASES = ([(k, 37, 53, bs, coder, vc) for k in ("yuv", "bgr", "u16") for bs in (1, 2, 3)
              for coder in ("zlib", "gpu") for vc in ("plain", "adaptive")]
             + [("yuv", 1080, 1920, 2, "gpu", "adaptive"), ("bgr", 1080, 1920, 3, "zlib", "plain"),
                ("u16", 1080, 1920, 1, "gpu", "plain")])


@gpu
@pytest.mark.parametrize("kind,h,w,bs,coder,vc", GOP_CASES)
def test_lossless_gop_chroma_only_changes(pkg, co, kind, h, w, bs, coder, vc):
    from new_bloom_filter_repo_b200 import improved_video_compressor as ivc
    frames = gop_clip(kind, h, w)
    n = h * w
    refs = [ref_diff(frames[i - 1], frames[i]) for i in range(1, len(frames))]
    assert refs[1][1].all() and not refs[2][1].any() and refs[3][1].sum() == 1 and refs[3][1].reshape(-1)[-1]
    # lossless (default): every inter mask is exactly `some byte differs`
    stats, pls = _compress_gop(pkg, kind, frames, bs, coder, vc, "lossless")
    assert stats["keyframes"] == 1
    for i in range(1, len(frames)):
        assert pls[i][:len(ivc._INTER_TAG)] in ivc._INTER_TAGS, i
        p, mask = _inter_mask(co, ivc, pls[i], n)
        anyd = refs[i - 1][1].reshape(-1)
        bad = np.flatnonzero(mask != anyd)
        assert bad.size == 0, (i, "mask differs from anyd at", bad[:8].tolist())
        assert p.ones == int(anyd.sum()) and p.vcount == 3 * p.ones, i
        assert bool(p.raw) == (i in (2, 3) or (i == 4 and n >= 10000)), (i, p.raw)   # p = 1, p = 0, p = 1/n <= 0.0001
    # reference: the mask is |dY| > 3 on the first sample, and a frame with residuals falls back to a keyframe
    stats, pls = _compress_gop(pkg, kind, frames, bs, coder, vc, "reference")
    resid = [0] + [ref_mask(d, a, 3.0)[2] for d, a in refs]
    keys = [i for i in range(len(frames)) if i == 0 or resid[i]]
    assert keys == [0, 1, 2, 4]
    assert [i for i, pl in enumerate(pls) if pl[:len(ivc._INTER_TAG)] not in ivc._INTER_TAGS] == keys
    assert stats["keyframes"] == len(keys)
    for i in (3, 5):
        p, mask = _inter_mask(co, ivc, pls[i], n)
        em, eones, _ = ref_mask(*refs[i - 1], 3.0)
        assert np.array_equal(mask, em.reshape(-1)) and p.ones == eones, i
