"""K1 over chains of consecutive pairs (k_threshold_sweep: each frame tile is read once and compared as curr of one pair and
prev of the next) against the oracle, for every pixel format, gray and lossless modes, and ragged frame sizes; and a pair list
that is not a chain, which takes k_threshold.  Every mask bit and both counts are compared."""
import numpy as np
import pytest

from tests.util import synth_stream

pytestmark = pytest.mark.gpu


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


def _frames(h, w, channels, dtype, nfr, seed):
    f = synth_stream(h, w, nfr, seed, [0.05, 0.2, 0.0, 0.01, 0.4], dtype)
    f[3, h - 1, w - 1, 0] ^= 1                 # |dY| = 1 in the frame's last pixel: a residual, in the ragged last word
    if channels == 1:
        return np.ascontiguousarray(f[..., 0])
    f[2, 0, 0, 1] ^= 1                         # chroma-only change: residual unless mask_mode 1
    return f


def _expected(co, prev, curr, thr, mask_mode, gray):
    from oracle import rbf_oracle as po
    if gray:
        m = po.frame_diff_mask(prev, curr, thr, gray=True)
    else:
        m, ones = co.frame_diff_mask(prev, curr, thr)
        assert int(m.sum()) == ones
    anyd = (prev != curr).any(axis=2) if prev.ndim == 3 else prev != curr
    if mask_mode:
        m = m | anyd.astype(np.uint8)
    return m.reshape(-1), int(m.sum()), int((anyd & (m == 0)).sum())


# 1080x1917: 2 070 360 px, neither a multiple of the 4096-px tile nor of 32; (3, 5): a 15-byte frame, too small for a bulk copy
@pytest.mark.parametrize("shape,channels,dtype,thr,mask_mode,gray", [
    ((1080, 1917), 3, np.uint8, 3.0, 0, False),
    ((1080, 1917), 3, np.uint16, 3.0, 0, False),
    ((1080, 1917), 1, np.uint8, 3.0, 0, False),
    ((1080, 1917), 1, np.uint16, 3.0, 0, False),
    ((1080, 1917), 3, np.uint8, 7.0, 0, True),
    ((1080, 1917), 3, np.uint16, 7.0, 0, True),
    ((1080, 1917), 3, np.uint8, 3.0, 1, False),
    ((130, 4099), 1, np.uint16, 10.5, 1, False),
    ((33, 65), 3, np.uint16, 20000.0, 0, False),
    ((37, 53), 3, np.uint8, 0.0, 0, False),
    ((3, 5), 1, np.uint8, 3.0, 0, False),
])
def test_k1_chain_vs_oracle(pkg, co, shape, channels, dtype, thr, mask_mode, gray):
    h, w = shape
    nfr = 6
    frames = _frames(h, w, channels, dtype, nfr, seed=17)
    st = pkg.FrameStream(h, w, channels, dtype, max_frames=nfr, k1_only=True, mask_mode=mask_mode, gray_mode=gray)
    st.upload(frames)
    pair_lists = [(list(range(nfr - 1)), list(range(1, nfr))),       # the whole stream
                  ([1, 2, 3], [2, 3, 4]),                            # a chain that starts inside the stream
                  ([0, 1], [2, 2])]                                  # not a chain
    for prev_idx, curr_idx in pair_lists:
        res = st.encode(prev_idx, curr_idx, thr)
        for t, (a, b) in enumerate(zip(prev_idx, curr_idx)):
            em, eones, eresid = _expected(co, frames[a], frames[b], thr, mask_mode, gray)
            assert res[t].ones == eones and res[t].resid == eresid, (prev_idx, t)
            assert np.array_equal(st.fetch(t)[2], em), (prev_idx, t)
    st.close()
