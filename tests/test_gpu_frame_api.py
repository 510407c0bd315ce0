"""The per-frame VideoFrameCompressor API on the device (ivc:727-909) against plain numpy models of the reference's semantics:

  A  k_median5 (rbf_median_blur5) at every border, CTA edge and full-frame size, in u8 and u16;
  B  _estimate_noise_level / _adaptive_diff_threshold, bit for bit, and the clamp at and around its limits;
  C  _calculate_frame_diff in every branch, at the N1 gather's chunk edges;
  D  _apply_frame_diff at every mask value, value count and layout, on the device branch and the host branch;
  E  recorded outcomes of the real reference (tests/golden/frame_api_kat.json, tests/golden/make_golden.py).

The models are written from the reference's behaviour; cv2 checks the median model where it is installed.
"""
import numpy as np
import pytest

from oracle import rbf_oracle as po
from tests.util import golden_json, sha

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    import new_bloom_filter_repo_b200 as p
    info = p._cabi.device_info()
    assert info["cc"] == (9, 0), info
    return p


def launches(pkg):
    return pkg._cabi.lib().rbf_get_counter(pkg._cabi.ctx(), b"kernel_launches")


# ------------------------------------------------------------------ models
def model_median_rows(a: np.ndarray, r0: int, r1: int) -> np.ndarray:
    """Rows [r0, r1) of the 5x5 median with replicated borders: clamp the coordinates, gather the 25 samples, take the 13th smallest."""
    H, W = a.shape
    ys = np.clip(np.arange(r0, r1)[:, None] + np.arange(-2, 3)[None, :], 0, H - 1)          # [rows, 5]
    xs = np.clip(np.arange(W)[:, None] + np.arange(-2, 3)[None, :], 0, W - 1)               # [W, 5]
    win = a[ys[:, None, :, None], xs[None, :, None, :]].reshape(r1 - r0, W, 25)
    return np.partition(win, 12, axis=-1)[..., 12]


def model_median(a: np.ndarray) -> np.ndarray:
    return model_median_rows(a, 0, a.shape[0])


def model_noise(plane: np.ndarray):
    """ivc:738-746 with the model median; an (h, w, 1) plane meets cv2's (h, w) median in numpy's broadcast."""
    med = model_median(plane[:, :, 0] if plane.ndim == 3 else plane)
    return np.std(plane.astype(np.float32) - med.astype(np.float32))


def model_threshold(plane, tol, lo, hi):
    return max(lo, min(hi, model_noise(plane) * tol))                                         # ivc:762-764


def model_diff(prev, curr, thr, use_direct_yuv, yuv):
    """ivc:784-847 -> (mask, changed_values, density)."""
    is_color = prev.ndim > 2 and prev.shape[2] > 1
    gray = is_color and not (use_direct_yuv and prev.shape[2] >= 3)
    if is_color:
        cg = po.bgr2gray(curr) if gray else curr[:, :, 0]
    else:
        cg = curr
    if thr is None:
        thr = model_threshold(cg, 10.0, 3.0, 30.0)
    mask = po.frame_diff_mask(prev, curr, thr, gray=gray)
    idx = np.where(mask == 1)
    if is_color:
        vals = curr[idx[0], idx[1], :].reshape(-1)
        if use_direct_yuv and yuv:
            vals = vals.astype(np.uint8)                                                       # ivc:825
    else:
        vals = curr[idx]
    return mask, vals, np.sum(mask) / mask.size


def model_apply(base, mask, vals):
    """ivc:866-909 on a plain array: only mask == 1 counts; colour frames need pixels x channels values or keep the base; grayscale
    frames take numpy's assignment, which broadcasts one value and raises on any other count."""
    out = base.copy()
    idx = np.where(mask == 1)
    if base.ndim == 3 and base.shape[2] > 1:
        rows, cols = idx
        if len(vals) == len(rows) * base.shape[2]:
            pv = vals.reshape(-1, base.shape[2])
            for i in range(len(rows)):
                out[rows[i], cols[i]] = pv[i]
    elif len(idx[0]) > 0:
        out[idx] = vals
    return out


def outcome(fn):
    try:
        return fn(), None
    except Exception as e:
        return None, type(e)


# ------------------------------------------------------------------ A: the 5x5 median
def device_median(pkg, a):
    out = np.empty_like(a)
    pkg._cabi.check(pkg._cabi.lib().rbf_median_blur5(pkg._cabi.ctx(), pkg._cabi.ptr(a), a.shape[0], a.shape[1], a.dtype.itemsize,
                                                     pkg._cabi.ptr(out)), pkg._cabi.ctx())
    return out


def planes(shape, dtype, seed):
    """Uniform random, three-level ties, all-max and a plane of 0 / max / values >= 2^(bits-1) (a signed compare would misorder them)."""
    rng = np.random.default_rng(seed)
    hi = np.iinfo(dtype).max
    yield "random", rng.integers(0, hi + 1, shape).astype(dtype)
    yield "ties", rng.choice(np.array([0, hi // 2, hi], dtype), shape)
    yield "allmax", np.full(shape, hi, dtype)
    yield "signs", rng.choice(np.array([0, 1, hi // 2, hi // 2 + 1, hi - 1, hi], dtype), shape)


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16])
def test_median_every_small_size(pkg, dtype):
    """Every H, W in 1..6: every output sample sees a replicated border."""
    for h in range(1, 7):
        for w in range(1, 7):
            for kind, a in planes((h, w), dtype, 100 * h + w):
                assert np.array_equal(device_median(pkg, a), model_median(a)), (h, w, kind)


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16])
def test_median_cta_edges(pkg, dtype):
    """The 32 x 8 CTA tiles: one sample short of, exactly on and one past one and two tiles in each direction."""
    for h in (7, 8, 9, 15, 16, 17):
        for w in (31, 32, 33, 63, 64, 65):
            for kind, a in planes((h, w), dtype, 1000 * h + w):
                assert np.array_equal(device_median(pkg, a), model_median(a)), (h, w, kind)


@pytest.mark.parametrize("shape", [(45, 77), (270, 481), (1080, 1920), (2160, 3840), (4320, 7680)])
@pytest.mark.parametrize("dtype", [np.uint8, np.uint16])
def test_median_full_frames(pkg, shape, dtype):
    """Full frames against cv2.medianBlur where it is installed, else the borders and sampled interior rows against the model."""
    rng = np.random.default_rng(shape[0] + np.dtype(dtype).itemsize)
    hi = np.iinfo(dtype).max
    a = rng.integers(0, hi + 1, shape).astype(dtype)
    a[: shape[0] // 3] = rng.choice(np.array([0, hi // 2 + 1, hi], dtype), (shape[0] // 3, shape[1]))   # a tie-heavy band
    got = device_median(pkg, a)
    try:
        import cv2
    except ImportError:
        cv2 = None
    if cv2 is not None:
        assert np.array_equal(got, cv2.medianBlur(a, 5))
        return
    H, W = shape
    for r0 in (0, H - 3, H // 3 - 2, H // 2):                                  # top and bottom border rows, the band's edge, the middle
        assert np.array_equal(got[r0:r0 + 3], model_median_rows(a, r0, r0 + 3)), r0
    for c in (0, 1, W - 2, W - 1):                                             # left and right border columns, a band of rows at a time
        for r0 in range(0, H, 540):
            r1 = min(H, r0 + 540)
            assert np.array_equal(got[r0:r1, c], model_median_rows(a[:, max(0, c - 2):c + 3], r0, r1)[:, min(c, 2)]), (c, r0)


def test_median_bad_shapes_raise_without_launching(pkg):
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    a = np.zeros((4, 4), np.uint8)
    before = launches(pkg)
    for h, w, s in ((0, 4, 1), (4, 0, 1), (4, 4, 3), (4, 4, 4)):
        assert L.rbf_median_blur5(ctx, pkg._cabi.ptr(a), h, w, s, pkg._cabi.ptr(a)) != 0, (h, w, s)
    assert launches(pkg) == before


# ------------------------------------------------------------------ B: noise level and adaptive threshold
@pytest.mark.parametrize("shape,dtype", [((1, 1), np.uint8), ((5, 3), np.uint16), ((37, 53), np.uint8), ((64, 96), np.uint16),
                                         ((270, 481), np.uint8)])
def test_noise_level_bit_exact(pkg, shape, dtype):
    vfc = pkg.VideoFrameCompressor()
    for kind, y in planes(shape, dtype, shape[0] * shape[1]):
        got = vfc._estimate_noise_level(y)
        want = np.std(y.astype(np.float32) - model_median(y).astype(np.float32))
        assert type(got) is np.float32 and float(got).hex() == float(want).hex(), (kind, got, want)


def test_adaptive_threshold_clamp(pkg):
    """noise x tolerance below, on, between, on and above [min_diff_threshold, max_diff_threshold]; a flat plane has no noise."""
    y = next(planes((40, 56), np.uint8, 5))[1]
    noise = model_noise(y)
    assert noise > 0
    lo, hi = 3.0, 30.0
    for prod in (lo / 2, lo, (lo + hi) / 2, hi, hi * 2):
        tol = prod / float(noise)
        vfc = pkg.VideoFrameCompressor(noise_tolerance=tol, min_diff_threshold=lo, max_diff_threshold=hi)
        got, want = vfc._adaptive_diff_threshold(y), max(lo, min(hi, noise * tol))
        assert float(got).hex() == float(want).hex() and type(got) is type(want), (prod, got, want)
        assert lo <= got <= hi
    # the limits themselves taken from the product: the clamp picks the limit, as Python's max / min do
    prod = noise * 10.0
    for lo2, hi2 in ((float(prod), 30.0 + float(prod)), (float(prod) / 2, float(prod))):
        vfc = pkg.VideoFrameCompressor(noise_tolerance=10.0, min_diff_threshold=lo2, max_diff_threshold=hi2)
        got = vfc._adaptive_diff_threshold(y)
        assert float(got) == float(prod) and type(got) is type(max(lo2, min(hi2, prod)))
    flat = np.full((33, 65), 200, np.uint8)
    vfc = pkg.VideoFrameCompressor()
    assert float(vfc._estimate_noise_level(flat)) == 0.0 and vfc._adaptive_diff_threshold(flat) == vfc.min_diff_threshold


def test_noise_plane_layouts_that_raise(pkg):
    vfc = pkg.VideoFrameCompressor()
    for bad in (np.zeros((8, 8, 3), np.uint8), np.zeros(64, np.uint8), np.zeros((8, 8), np.float32), np.zeros((8, 8), np.int16)):
        with pytest.raises(NotImplementedError):
            vfc._estimate_noise_level(bad)
    with pytest.raises(ValueError):                       # (h, w, 1) - (h, w): numpy cannot broadcast 9 x 11 x 1 against 9 x 11
        vfc._estimate_noise_level(np.zeros((9, 11, 1), np.uint8))
    sq = next(planes((6, 6), np.uint8, 3))[1][:, :, None]                 # ... but it can a square plane: the reference's number
    assert float(vfc._estimate_noise_level(sq)).hex() == float(model_noise(sq)).hex()


# ------------------------------------------------------------------ C: _calculate_frame_diff
def frame_pair(shape, dtype, seed, p=0.3):
    rng = np.random.default_rng(seed)
    hi = np.iinfo(dtype).max + 1
    prev = rng.integers(0, hi, shape).astype(dtype)
    curr = prev.copy()
    sel = rng.random(shape[:2]) < p
    curr[sel] = (curr[sel].astype(np.int64) + rng.integers(1, 8, curr[sel].shape)) % hi   # small steps: the thresholds matter
    return prev, curr


BRANCHES = [("yuvframe", (3,), True, True), ("yuv_array", (3,), True, False), ("bgr", (3,), False, False), ("plane", (), False, False),
            ("hw1", (1,), False, False)]


def check_diff(pkg, prev, curr, thr, use_direct_yuv, yuv, label):
    vfc = pkg.VideoFrameCompressor(use_direct_yuv=use_direct_yuv)
    pf, cf = (pkg.YUVFrame(prev), pkg.YUVFrame(curr)) if yuv else (prev, curr)
    want, werr = outcome(lambda: model_diff(prev, curr, thr, use_direct_yuv, yuv))
    got, gerr = outcome(lambda: vfc._calculate_frame_diff(pf, cf, threshold=thr))
    assert gerr is werr, (label, gerr, werr)
    if werr is not None:
        return
    (m, v, d), (om, ov, od) = got, want
    assert m.shape == om.shape and m.dtype == np.uint8 and np.array_equal(m, om), label
    assert v.dtype == ov.dtype and v.tobytes() == ov.tobytes(), label
    assert float(d).hex() == float(od).hex(), (label, d, od)
    return got


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16])
@pytest.mark.parametrize("branch", BRANCHES, ids=[b[0] for b in BRANCHES])
def test_frame_diff_branches_and_thresholds(pkg, branch, dtype):
    _, tail, use_direct_yuv, yuv = branch
    for shape in ((37, 53), (12, 12), (1, 1), (2, 130)):
        prev, curr = frame_pair(shape + tail, dtype, shape[0] * shape[1])
        for thr in (None, 0, 3.0, 3.5):
            check_diff(pkg, prev, curr, thr, use_direct_yuv, yuv, (shape, thr))


def chunk_bounds(npix):
    """Pixel index where each of the N1 gather's chunks after the first begins (rbf_kernels.cu: gather_chunks, k_gather)."""
    nwords = (npix + 31) // 32
    ch = min(64, max(1, nwords // 4096))
    return [32 * (nwords * b // ch) for b in range(1, ch)]


def masked_pair(shape, dtype, flat_sel, seed):
    """prev random; curr moves every channel of the selected pixels by a quarter of the range (|dY| and |dgray| > 3)."""
    rng = np.random.default_rng(seed)
    hi = np.iinfo(dtype).max + 1
    prev = rng.integers(0, hi, shape).astype(dtype)
    curr = prev.copy()
    flat = curr.reshape(shape[0] * shape[1], -1)
    flat[flat_sel] = (flat[flat_sel].astype(np.int64) + hi // 4) % hi
    return prev, curr


@pytest.mark.parametrize("hw", [(32, 8191), (123, 2131), (511, 513), (512, 512), (481, 545), (2160, 3840), (4320, 7680)],
                         ids=lambda s: f"{s[0]}x{s[1]}")
def test_frame_diff_at_gather_chunk_edges(pkg, hw):
    """npix 262112 (1 chunk), 262113 (2: the first pixel of word 8191 opens chunk 2), 262143-262145 (2), 2160x3840 (63), 4320x7680
    (64, the cap).  Masks: the last pixel, every pixel, one chunk only, one pixel on each side of every chunk boundary."""
    npix = hw[0] * hw[1]
    bounds = chunk_bounds(npix)
    assert len(bounds) + 1 == {262112: 1, 8294400: 63, 33177600: 64}.get(npix, 2)
    edges = np.array(sorted({b for b in bounds} | {b - 1 for b in bounds}), dtype=np.int64)
    one_chunk = np.arange(bounds[0] if bounds else 0, bounds[1] if len(bounds) > 1 else npix)
    masks = {"last": np.array([npix - 1]), "all": slice(None), "one_chunk": one_chunk, "edges": edges}
    big = npix > 10 ** 7
    cases = [("bgr", (3,), False, False, np.uint8), ("plane", (), False, False, np.uint16), ("yuvframe", (3,), True, True, np.uint16)]
    for name, tail, use_direct_yuv, yuv, dtype in cases[:1] if big else cases:
        for mname, sel in masks.items():
            if big and mname == "one_chunk":
                continue
            prev, curr = masked_pair(hw + tail, dtype, sel, npix)
            got = check_diff(pkg, prev, curr, 3.0, use_direct_yuv, yuv, (name, mname))
            if mname == "all":
                assert got[0].all()
            if mname == "edges" and not big:                   # and the scatter puts the gathered values back where they came from
                vfc = pkg.VideoFrameCompressor(use_direct_yuv=use_direct_yuv)
                rec = vfc._apply_frame_diff(pkg.YUVFrame(prev) if yuv else prev, got[0], got[1].astype(dtype))
                want = model_apply(prev, got[0], got[1].astype(dtype))
                assert np.array_equal(np.asarray(rec.data if yuv else rec), want), name


# ------------------------------------------------------------------ D: _apply_frame_diff
H, W = 6, 7


def mask_kinds():
    out = {}
    m = np.zeros((H, W), np.uint8); m[[1, 3, 5], [1, 4, 6]] = 1; out["u8_01"] = m
    m = np.zeros((H, W), bool); m[[0, 2, 5], [0, 3, 6]] = True; out["bool"] = m
    m = np.zeros((H, W), np.uint8); m[1, 1] = 1; m[2, 2] = 255; m[4, 0] = 2; m[0, 6] = 1; out["u8_2_255"] = m
    m = np.zeros((H, W), np.int16); m[1, 1] = 1; m[2, 2] = 257; m[3, 3] = -1; m[5, 5] = 256; m[4, 4] = 1; out["i16_257_-1"] = m
    m = np.zeros((H, W), np.float64); m[1, 1] = 1.0; m[2, 2] = 0.5; m[5, 0] = 1.0; m[3, 6] = 1.5; out["f64_1_0.5"] = m
    out["empty"] = np.zeros((H, W), np.uint8)
    return out


LAYOUTS = [("g8", (H, W), np.uint8, False), ("g16", (H, W), np.uint16, False), ("hw1", (H, W, 1), np.uint8, False),
           ("c8", (H, W, 3), np.uint8, False), ("c16", (H, W, 3), np.uint16, False), ("c4", (H, W, 4), np.uint8, False),
           ("yuv8", (H, W, 3), np.uint8, True), ("yuv16", (H, W, 3), np.uint16, True)]
COUNTS = ("exact", "short", "long", "zero", "one")


@pytest.mark.parametrize("layout", LAYOUTS, ids=[l[0] for l in LAYOUTS])
def test_apply_frame_diff_matrix(pkg, layout):
    """Every mask kind x value count on one layout, with values of the frame's dtype (the device branch where the store holds the
    format) and as int64 (the host branch): both give the model's frame, or raise its exception."""
    name, shape, dtype, yuv = layout
    rng = np.random.default_rng(len(name) * 7 + len(shape))
    hi = np.iinfo(dtype).max + 1
    base = rng.integers(0, hi, shape).astype(dtype)
    ch = shape[2] if len(shape) == 3 and shape[2] > 1 else 1
    vdt = np.uint8 if yuv else dtype                       # a YUVFrame's values are u8 (ivc:825), whatever the frame's dtype
    for mname, mask in mask_kinds().items():
        if shape[-1:] == (1,):
            mask = mask[:, :, None]
        n = int(np.sum(mask == 1))
        for cname in COUNTS:
            k = {"exact": n, "short": n - 1, "long": n + 1, "zero": 0, "one": 1}[cname]
            if k < 0:
                continue
            vals = rng.integers(0, 256 if vdt == np.uint8 else hi, k * ch).astype(vdt)
            want, werr = outcome(lambda: model_apply(base, mask, vals))
            results = []
            for vv in (vals, vals.astype(np.int64)):
                vfc = pkg.VideoFrameCompressor(use_direct_yuv=yuv)
                frame = pkg.YUVFrame(base.copy()) if yuv else base.copy()
                got, gerr = outcome(lambda: vfc._apply_frame_diff(frame, mask, vv))
                label = (name, mname, cname, vv.dtype.name)
                assert gerr is werr, (label, gerr, werr)
                assert np.array_equal(np.asarray(frame.data if yuv else frame), base), label        # the base is not modified
                if werr is not None:
                    continue
                d = got.data if yuv else got
                assert type(got) is type(frame) and d.shape == base.shape and d.dtype == base.dtype, label
                assert np.array_equal(d, want), label
                if yuv:
                    for i, p in enumerate(("y_plane", "u_plane", "v_plane")):
                        assert np.array_equal(got.yuv_info[p], want[:, :, i]), (label, p)
                results.append(d)
            if len(results) == 2:
                assert np.array_equal(results[0], results[1])


def test_apply_frame_diff_hw1_with_hw_mask_follows_numpy(pkg):
    """An (h, w) mask on an (h, w, 1) frame indexes (N, 1) pixels: N values cannot be broadcast there unless N is 1."""
    base = np.arange(H * W, dtype=np.uint8).reshape(H, W, 1)
    m = np.zeros((H, W), np.uint8); m[1, 2] = m[4, 5] = 1
    vfc = pkg.VideoFrameCompressor()
    with pytest.raises(ValueError):
        vfc._apply_frame_diff(base, m, np.array([9, 8], np.uint8))
    m[4, 5] = 0
    assert np.array_equal(vfc._apply_frame_diff(base, m, np.array([9], np.uint8)), model_apply(base, m, np.array([9], np.uint8)))


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16])
@pytest.mark.parametrize("channels", [1, 3])
def test_stream_apply_diff_into_next_frame_contract(pkg, dtype, channels):
    """FrameStream.apply_diff, the layer under _apply_frame_diff: frame base + 1 (modulo the store, the last slot included) is the
    base with every non-zero mask entry set (any dtype, 256 and 0.5 included); values are C samples of the stream's dtype per set pixel
    or the output is the base unchanged; a mask of another size or values of another dtype raise before anything runs.  The output
    slot holds a third frame before each call, so a call that writes nothing fails."""
    rng = np.random.default_rng(channels + np.dtype(dtype).itemsize)
    hi = np.iinfo(dtype).max + 1
    shape = (19, 45) + ((channels,) if channels > 1 else ())
    base = rng.integers(0, hi, shape).astype(dtype)
    other = base ^ dtype(1)                                                              # differs from base in every sample
    st = pkg.FrameStream(19, 45, channels, dtype, max_frames=3)
    try:
        for mdt, vals in ((bool, (0, 1)), (np.uint8, (0, 1, 2, 255)), (np.int16, (0, 1, 256, 257, -1)), (np.float64, (0.0, 1.0, 0.5, -2.0))):
            mask = rng.choice(np.array(vals, dtype=mdt), (19, 45))
            setp = mask != 0
            n = int(setp.sum())
            v = rng.integers(0, hi, n * channels).astype(dtype)
            want = base.copy()
            want[setp] = v.reshape(-1, channels) if channels > 1 else v
            for b, out in ((0, 1), (2, 0)):                                              # 2 -> 0: the slots wrap
                st.upload(base, first=b)
                st.upload(other, first=out)
                assert st.apply_diff(b, mask, v) == n, (mdt, b)
                assert np.array_equal(st.download(out), want), (mdt, b)
                st.upload(other, first=out)
                assert st.apply_diff(b, mask, v[:-1]) == 0, (mdt, b)                     # one sample short: the base
                assert np.array_equal(st.download(out), base), (mdt, b)
        before = launches(pkg)
        with pytest.raises(ValueError):
            st.apply_diff(0, np.ones(19 * 45 - 1, np.uint8), np.zeros((19 * 45 - 1) * channels, dtype))
        with pytest.raises(ValueError):
            st.apply_diff(0, np.ones((19, 45), np.uint8), np.zeros(19 * 45 * channels, np.int64))
        assert launches(pkg) == before
    finally:
        st.close()


def test_apply_happy_path_launches_only_the_chain_sweep(pkg):
    """_calculate_frame_diff + _apply_frame_diff of a grayscale and a colour pair: the apply costs the one-pair K4c sweep only."""
    vfc = pkg.VideoFrameCompressor()
    for shape in ((64, 80), (64, 80, 3), (64, 80, 1)):
        prev, curr = frame_pair(shape, np.uint8, 3)
        mask, vals, _ = vfc._calculate_frame_diff(prev, curr, threshold=3.0)
        vfc._apply_frame_diff(prev, mask, vals)                                          # warm the cached stream
        before = launches(pkg)
        out = vfc._apply_frame_diff(prev, mask, vals)
        assert launches(pkg) - before == 3, shape                                        # k_tile_count, k_tile_scan, k_apply_sweep
        assert np.array_equal(out, model_apply(prev, mask, vals))


# ------------------------------------------------------------------ E: outcomes recorded from the real reference
def dec(d):
    return np.frombuffer(bytes.fromhex(d["hex"]), dtype=np.dtype(d["dtype"])).reshape(d["shape"]).copy()


KAT = golden_json("frame_api_kat.json")


@pytest.mark.parametrize("rec", KAT["apply"], ids=[r["name"] for r in KAT["apply"]])
def test_apply_frame_diff_against_reference(pkg, rec):
    base, mask, vals = dec(rec["base"]), dec(rec["mask"]), dec(rec["values"])
    vfc = pkg.VideoFrameCompressor(use_direct_yuv=rec["use_direct_yuv"])
    frame = pkg.YUVFrame(base.copy()) if rec["yuv"] else base.copy()
    got, err = outcome(lambda: vfc._apply_frame_diff(frame, mask, vals))
    if "error" in rec:
        assert err is not None and err.__name__ == rec["error"]
        return
    assert err is None, err
    d = got.data if rec["yuv"] else got
    assert list(d.shape) == rec["result_shape"] and d.dtype.name == rec["result_dtype"] and sha(d) == rec["result_sha256"]
    if rec["yuv"]:
        assert [sha(got.yuv_info[p]) for p in ("y_plane", "u_plane", "v_plane")] == rec["planes_sha256"]
    assert np.array_equal(np.asarray(frame.data if rec["yuv"] else frame), base) == rec["base_unchanged"]


@pytest.mark.parametrize("rec", KAT["diff"], ids=[r["name"] for r in KAT["diff"]])
def test_calculate_frame_diff_against_reference(pkg, rec):
    prev, curr = dec(rec["prev"]), dec(rec["curr"])
    vfc = pkg.VideoFrameCompressor(use_direct_yuv=rec["use_direct_yuv"])
    pf, cf = (pkg.YUVFrame(prev), pkg.YUVFrame(curr)) if rec["yuv"] else (prev, curr)
    got, err = outcome(lambda: vfc._calculate_frame_diff(pf, cf, threshold=rec["threshold"]))
    if "error" in rec:
        assert err is not None and err.__name__ == rec["error"]
        return
    assert err is None, err
    mask, changed, dens = got
    assert list(mask.shape) == rec["mask_shape"] and sha(mask) == rec["mask_sha256"]
    assert changed.dtype.name == rec["changed_dtype"] and len(changed) == rec["changed_len"] and sha(changed) == rec["changed_sha256"]
    assert float(dens).hex() == rec["density"]


@pytest.mark.parametrize("rec", KAT["noise"], ids=[r["name"] for r in KAT["noise"]])
def test_noise_level_against_reference(pkg, rec):
    plane = dec(rec["plane"])
    assert sha(device_median(pkg, plane)) == rec["median_sha256"]
    vfc = pkg.VideoFrameCompressor(noise_tolerance=rec["noise_tolerance"])
    nl = vfc._estimate_noise_level(plane)
    assert type(nl).__name__ == rec["noise_level_type"] and float(nl).hex() == rec["noise_level"]
    assert float(vfc._adaptive_diff_threshold(plane)).hex() == rec["threshold"]
