"""K2 builds each frame's bit array in shared memory: CTA rank j of a cluster owns words [j*W, (j+1)*W), words beyond
the cluster's range are set in global memory, and frames that do not fill a whole wave of the GPU get several copies
that are OR-ed together.  These tests put filter sizes on every one of those edges and compare bit arrays and witnesses
with the C oracle, bit for bit."""
import numpy as np
import pytest

from tests.util import mask_for

pytestmark = pytest.mark.gpu

# words per CTA of the default build: K2_WORDS in csrc/rbf_k2_insert.cuh (one CTA of 32 warps per SM)
W = ((233472 - 1024 - 32 * 512 * 2) // 4) & ~15
N4K, N8K = 3840 * 2160, 7680 * 4320


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


def compress_both(pkg, co, m, k, l):
    ob, ow, op, on, oratio, ok, ol = co.compress(m, k_l_override=(k, l))
    assert ol == l
    bitmap, witness, p, nn, ratio = pkg.BloomFilterCompressor().compress(m, k_l_override=(k, l))
    assert len(bitmap) == l and np.array_equal(bitmap, ob)
    assert np.array_equal(np.array(witness, dtype=np.uint8), ow)
    return ob


@pytest.mark.parametrize("l", [32 * (W - 1), 32 * W - 5, 32 * W, 32 * W + 1, 32 * (W + 1)])
def test_cta_range_boundary(pkg, co, l):
    """l around one CTA's range: the array fits one CTA, just fills it, or has one word more (rank 1 or global memory)."""
    ob = compress_both(pkg, co, mask_for({"n": N4K, "p_gen": 0.05, "seed": 51}), 3.19, l)
    if l > 32 * W:                                   # bits in the last word of rank 0 and the first word after it
        assert ob[32 * W - 32:32 * W].any() and ob[32 * W:l].any()


@pytest.mark.parametrize("n,l", [(N4K, 32 * (2 * W) - 32), (N4K, 32 * (2 * W) + 32),
                                 (N8K, 32 * (8 * W) - 32), (N8K, 32 * (8 * W)), (N8K, 32 * (8 * W) + 32), (N8K, 1 << 24)])
def test_cluster_capacity_and_global_tail(pkg, co, n, l):
    """l at 2*W +- 1 word, where the shared-memory kernel hands arrays over to the RED.OR-into-L2 kernel, and at 8*W +- 1
    word (the largest cluster); l = 2^24 > 8*W keeps a large tail in global memory whatever the cluster size."""
    ob = compress_both(pkg, co, mask_for({"n": n, "p_gen": 0.05, "seed": 52}), 3.19, l)
    assert ob.any()


@pytest.mark.parametrize("n,p_gen,k,l", [(5000, 0.05, 2.5, 20), (5000, 0.05, 2.5, 31), (4096, 0.05, 3.19, 1000),
                                         (2_000_000, 0.2, 4.0, 64), (N4K, 0.3, 3.5, 4099), (101, 0.1, 3.19, 40)])
def test_small_and_saturated_filters(pkg, co, n, p_gen, k, l):
    """l < 32 and not a multiple of 32, saturated arrays (every copy of a small launch non-zero in every word), n = 101."""
    compress_both(pkg, co, mask_for({"n": n, "p_gen": p_gen, "seed": 53}), k, l)


@pytest.mark.parametrize("k", [0.6, 1.4])
def test_floor_k_zero_and_one(pkg, co, k):
    """floor(k) = 0 (only the activated probe) and floor(k) = 1, on an array spread over two CTAs."""
    compress_both(pkg, co, mask_for({"n": N4K, "p_gen": 0.05, "seed": 54}), k, 32 * W + 1000)


def test_century_and_digit_boundaries(pkg, co):
    """n = 101 and a mask set around centuries 0, 9/10, 99/100, 999/1000 and 9999/10000 (digit-count boundaries take
    the per-lane path), on an array spread over two CTAs."""
    n = N4K
    m = mask_for({"n": n, "p_gen": 0.02, "seed": 55})
    for c in (0, 10, 100, 1000, 10000, 80000):
        m[max(0, 100 * c - 300):100 * c + 300] = 1
    compress_both(pkg, co, m, 3.19, 32 * W + 77)


def _stream_vs_oracle(pkg, co, H, Wd, ls, seed):
    rng = np.random.default_rng(seed)
    F = len(ls)
    frames = rng.integers(0, 256, (F + 1, H, Wd, 3), dtype=np.uint8)
    for t in range(1, F + 1):                       # each frame: the previous one with ~5 % of the pixels changed
        keep = rng.random((H, Wd)) >= 0.05
        frames[t][keep] = frames[t - 1][keep]
    st = pkg.FrameStream(H, Wd, 3, np.uint8, max_frames=F + 1)
    try:
        st.upload(frames)
        ks = [3.19, 2.7, 1.4, 4.2][:F]
        res = st.encode(list(range(F)), list(range(1, F + 1)), 3.0, k_override=ks, l_override=ls)
        for t in range(F):
            bm, wt, mask = st.fetch(t)
            assert res[t].l == ls[t]
            ob, ow, *_ = co.compress(mask, k_l_override=(ks[t], ls[t]))
            assert np.array_equal(bm, np.packbits(ob)) and np.array_equal(wt, np.packbits(ow))
    finally:
        st.close()


def test_one_pair_stream_several_copies(pkg, co):
    """A 1-pair 4K encode: the GPU is filled with many copies of the one array, merged into it with RED.OR."""
    _stream_vs_oracle(pkg, co, 2160, 3840, [32 * W + 4097], 56)


def test_three_pair_stream_mixed_sizes(pkg, co):
    """A 3-pair encode whose frames have different l in one launch (two CTAs, one CTA, a few words), several copies each."""
    _stream_vs_oracle(pkg, co, 2160, 3840, [32 * W + 4097, 32 * W - 5, 1000], 57)


def test_frames_beyond_one_wave(pkg, co):
    """More pairs than the GPU holds clusters at once: whole waves take one copy per frame (plain stores), the frames of the
    last wave several copies (RED.OR merge), in one launch."""
    H, Wd, F = 480, 640, 140
    rng = np.random.default_rng(58)
    frames = np.repeat(rng.integers(0, 256, (1, H, Wd, 3), dtype=np.uint8), F + 1, axis=0)
    for t in range(1, F + 1):
        ch = rng.random((H, Wd)) < 0.05
        frames[t][ch] = frames[t][ch] ^ 0x80
    st = pkg.FrameStream(H, Wd, 3, np.uint8, max_frames=F + 1)
    try:
        st.upload(frames)
        res = st.encode_consecutive(F + 1, 3.0)
        for t in range(F):
            bm, wt, mask = st.fetch(t)
            ob, ow, op, on, oratio, ok, ol = co.compress(mask)
            assert (res[t].l, len(ow)) == (ol, res[t].wlen)
            assert np.array_equal(bm, np.packbits(ob)) and np.array_equal(wt, np.packbits(ow))
    finally:
        st.close()
