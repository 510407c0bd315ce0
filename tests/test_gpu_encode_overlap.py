"""The default resident-stream encode -- K1 of ranges 1.. on a few SMs beside K2 of the range before (encode_ranges, pipe_k1_sms)
-- against an explicit encode_ranges = 1 encode of the same frames, byte for byte: every result field, bitmap, witness and mask.

Each schedule runs on a context of its own, created here: the default one is left exactly as rbf_ctx_create made it, so no option
another test set on the process-wide context (and no RBF_* environment knob) decides what "default" means."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

R_DEFAULT = 2                        # encode_ranges of a fresh context; below 8 * R_DEFAULT pairs the encode is serial
THR = 3.0
P_MIX = (0.05, 0.02, 0.45, 0.1, 0.0, 0.2, 0.01, 0.03)    # coded, plus raw pairs: p >= p* = 0.32453 (0.45) and no change (0.0)
H1, W1 = 1080, 1921                  # 2 074 680 px: a ragged last mask word and a partial last K1 tile


@pytest.fixture(scope="module")
def pkg():
    import new_bloom_filter_repo_b200 as p
    assert p._cabi.device_info()["cc"] == (9, 0)
    return p


@pytest.fixture(scope="module")
def ctxs(pkg):
    """{"default": a fresh context, "serial": a fresh context with encode_ranges = 1}."""
    L = pkg._cabi.lib()
    dev = int(os.environ.get("RBF_DEVICE", os.environ.get("LOCAL_RANK", "0")))   # the device of _cabi.ctx()
    out = {}
    try:
        for name in ("default", "serial"):
            h = C.c_void_p()
            pkg._cabi.check(L.rbf_ctx_create(dev, C.byref(h)))
            out[name] = h
        pkg._cabi.check(L.rbf_set_option(out["serial"], b"encode_ranges", 1), out["serial"])
        yield out
    finally:
        for h in out.values():
            L.rbf_ctx_destroy(h)


def make_frames(p_seq, seed, h=H1, w=W1, channels=3, dtype=np.uint8):
    """Frame t = frame t-1 with a p_seq[t-1] share of its pixels moved by a quarter of the sample range (every sample), plus the
    low bit of one sample flipped in 1 % of the pixels (of a chroma sample for 3 channels): those differ without crossing the
    threshold, so the residual counts are not zero."""
    dt = np.dtype(dtype)
    rng = np.random.default_rng(seed)
    shape = (h, w, channels) if channels > 1 else (h, w)
    out = np.empty((len(p_seq) + 1,) + shape, dt)
    out[0] = rng.integers(0, np.iinfo(dt).max + 1, shape, dtype=dt)
    step = dt.type(np.iinfo(dt).max // 4 + 1)
    for t, p in enumerate(p_seq, 1):
        r = np.random.default_rng(seed + t)
        out[t] = out[t - 1]
        u = r.integers(0, 10000, (h, w), dtype=np.uint16)
        out[t][u < int(p * 10000)] += step                 # wraps modulo the sample range
        flip = u >= 9900
        if channels > 1:
            out[t][..., channels - 1][flip] ^= 1
        else:
            out[t][flip] ^= 1
    return out


def encode_on(pkg, h, frames, prev=None, curr=None, ko=None, lo=None):
    """One resident encode on context h -> (result fields, bitmap rows, witness rows, mask rows, kernels launched)."""
    L = pkg._cabi.lib()
    nfr = len(frames)
    P = nfr - 1 if prev is None else len(prev)
    channels = 1 if frames.ndim == 3 else frames.shape[3]
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(pkg._cabi, "ctx", lambda: h)            # a FrameStream takes its context from _cabi.ctx()
        st = pkg.FrameStream(frames.shape[1], frames.shape[2], channels, frames.dtype, max_frames=nfr, max_pairs=P)
        try:
            st.upload(frames)
            kw = {} if ko is None else dict(k_override=ko, l_override=lo)
            n0 = L.rbf_get_counter(h, b"kernel_launches")
            if prev is None:
                res = st.encode_consecutive(nfr, THR, **kw)
            else:
                res = st.encode(prev, curr, THR, **kw)
            launched = L.rbf_get_counter(h, b"kernel_launches") - n0
            bm, wt, mk = st.fetch_batch(0, P, want_masks=True)
            fields = [(r.n, r.ones, r.resid, r.raw, r.l, r.wlen, r.k.hex(), r.p.hex(), r.floor_k, r.act_T) for r in res]
            return fields, bm, wt, mk, launched
        finally:
            st.close()


def assert_same(pkg, ctxs, frames, split=True, **kw):
    """The default schedule and the serial one code every pair alike; split: the default one did split the encode."""
    d = encode_on(pkg, ctxs["default"], frames, **kw)
    s = encode_on(pkg, ctxs["serial"], frames, **kw)
    assert any(f[3] for f in s[0]) and not all(f[3] for f in s[0])       # raw and coded pairs
    assert d[0] == s[0]
    for what, a, b in zip(("bitmaps", "witnesses", "masks"), d[1:4], s[1:4]):
        assert a.shape == b.shape and np.array_equal(a, b), what
    if split:
        assert d[4] > s[4], ("the default encode did not split", d[4], s[4])
    else:
        assert d[4] == s[4], ("below 8 pairs per range the default encode is the serial one", d[4], s[4])


@pytest.fixture(scope="module")
def frames_4k():
    return make_frames([P_MIX[t % len(P_MIX)] for t in range(299)], 11, 2160, 3840)


def test_4k_299_pairs(pkg, ctxs, frames_4k):
    assert_same(pkg, ctxs, frames_4k)


@pytest.mark.parametrize("P", [8 * R_DEFAULT - 1, 8 * R_DEFAULT])
def test_4k_fallback_edge(pkg, ctxs, frames_4k, P):
    assert_same(pkg, ctxs, frames_4k[:P + 1], split=P >= 8 * R_DEFAULT)


@pytest.mark.parametrize("raw_range", ["first", "last", "every"])
def test_all_raw_range(pkg, ctxs, raw_range):
    P = 8 * R_DEFAULT * 2
    lo = [P * r // R_DEFAULT for r in range(R_DEFAULT + 1)]
    raw = {"first": range(lo[0], lo[1]), "last": range(lo[-2], lo[-1]), "every": range(P)}[raw_range]
    p = [(0.45 if i % 2 else 0.0) if i in raw else P_MIX[i % 2] for i in range(P)]
    if raw_range == "every":
        p[-1] = 0.05                                        # one coded pair, so that K3 and K3b run
    assert_same(pkg, ctxs, make_frames(p, 21))


def test_per_pair_overrides(pkg, ctxs):
    P, n = 8 * R_DEFAULT + 5, H1 * W1
    ks = [(0.5, 1.25, 2.0, 2.7, 3.5, 4.2, 0.0)[i % 7] for i in range(P)]          # 0.0: no override for that pair
    ls = [0 if i == 3 else int(n * (0.08 + 0.01 * (i % 20))) for i in range(P)]    # l = 0 forces raw
    assert_same(pkg, ctxs, make_frames([P_MIX[i % len(P_MIX)] for i in range(P)], 31), ko=ks, lo=ls)


@pytest.mark.parametrize("channels,dtype", [(3, np.uint16), (1, np.uint8), (1, np.uint16)], ids=["3ch-u16", "1ch-u8", "1ch-u16"])
def test_formats(pkg, ctxs, channels, dtype):
    P = 8 * R_DEFAULT + 3
    assert_same(pkg, ctxs, make_frames([P_MIX[i % len(P_MIX)] for i in range(P)], 41, channels=channels, dtype=dtype))


@pytest.mark.parametrize("name", ["swapped", "broken_at_range_boundary"])
def test_pair_list_not_a_chain(pkg, ctxs, name):
    P = 8 * R_DEFAULT * 2
    if name == "swapped":
        prev, curr = [t + 1 for t in range(P)], list(range(P))
    else:                                                  # one chain per range, broken exactly at the range boundary
        prev, curr = [t if t < P // 2 else t + 3 for t in range(P)], [t + 1 if t < P // 2 else t + 4 for t in range(P)]
    frames = make_frames([P_MIX[i % len(P_MIX)] for i in range(max(prev + curr))], 51)
    assert_same(pkg, ctxs, frames, prev=prev, curr=curr)
