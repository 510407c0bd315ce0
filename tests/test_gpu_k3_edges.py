"""K3, the Bloom query, against the C oracle at every kernel formulation, filter size, shared/L2 split, index-digit edge and
launch shape.

K3 decides for every position of every frame whether it passes the Bloom test (ivc:116-138).  Its formulations
(rbf_k3_query.cuh): `query_variant` 0 the per-lane kernel k_query; 1 the staged rings k_query2 (also the home of every filter
beyond 2^24 bits); 5 the decade tiles k_query4 (half-decade tiles for 2^23 < l <= 2^24); 6 half-decade tiles for every l <= 2^24.
The oracle's filter_check (oracle/rbf_oracle.c) hashes str(i) with the full XXH64 and takes a 64-bit `%` per position: it shares
nothing with the century/decade decomposition, Barrett reduction, tiles or rings.

Probes:
  * the pass mask -- a bit array decoded with an all-ones witness of n bits gives back exactly the pass mask, and the witness
    bits consumed are the pass count.  No encode is needed, so the bit array is free: any fill, any l (also l >= n).
  * the encode -- bitmap, witness and witness length of the whole coder for a given (k, l).
The options are context-global; every test restores the defaults (query_variant 5, query_warps 0, query_smem_bytes 0)."""
import contextlib
import ctypes as C
import os
import re
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CSRC = Path(__file__).resolve().parents[1] / "new_bloom_filter_repo_b200" / "csrc"
VARIANTS = (0, 1, 5, 6)
DEFAULTS = (("query_variant", 5), ("query_warps", 0), ("query_smem_bytes", 0))


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
def options(pkg, ctx=None, **opts):
    L = pkg._cabi.lib()
    c = ctx if ctx is not None else pkg._cabi.ctx()
    try:
        for k, v in opts.items():
            pkg._cabi.check(L.rbf_set_option(c, k.encode(), int(v)), c)
        yield
    finally:
        for k, v in DEFAULTS:
            L.rbf_set_option(c, k.encode(), v)


def rand_bits(rng, l, fill):
    """One byte per bit, as the coder takes them.  Fill 0.5: np.unpackbits of random bytes; l <= 3: a fixed non-empty pattern."""
    if l <= 3:
        return np.array([1, 0, 1][:l], dtype=np.uint8)
    if fill == 0.5:
        return np.unpackbits(rng.integers(0, 256, (l + 7) // 8, dtype=np.uint8))[:l]
    return (rng.random(l) < fill).astype(np.uint8)


def gpu_pass(pkg, bits, n, k, ctx=None):
    """-> (pass mask uint8[n], pass count) from rbf_decompress_mask with an all-ones witness of n bits."""
    cabi = pkg._cabi
    c = ctx if ctx is not None else cabi.ctx()
    bits = np.ascontiguousarray(bits, dtype=np.uint8)
    wit = np.ones(n, dtype=np.uint8)
    out = np.empty(n, dtype=np.uint8)
    consumed = C.c_uint64()
    sd = cabi.seeds_struct(cabi.IVC_SEEDS)
    cabi.check(cabi.lib().rbf_decompress_mask(c, cabi.ptr(bits), bits.size, cabi.ptr(wit), n, n, float(k), C.byref(sd),
                                              cabi.ptr(out), C.byref(consumed)), c)
    return out, int(consumed.value)


def oracle_pass(co, bits, n, k):
    """The same probe through orc_decompress_kl (c_oracle.decompress drops the count)."""
    bits = np.ascontiguousarray(bits, dtype=np.uint8)
    wit = np.ones(n, dtype=np.uint8)
    out = np.empty(n, dtype=np.uint8)
    j = co.lib().orc_decompress_kl(co._ptr(bits), bits.size, co._ptr(wit), n, n, float(k), *[int(s) for s in co.IVC_SEEDS],
                                   co._ptr(out))
    return out, int(j)


def gpu_compress(pkg, m, k, l):
    """rbf_compress_mask with an explicit (k, l) (what BloomFilterCompressor.compress(m, k_l_override=(k, l)) calls)
    -> (bitmap uint8[l], witness uint8[wlen], info)."""
    cabi = pkg._cabi
    c = cabi.ctx()
    m = np.ascontiguousarray(m, dtype=np.uint8)
    info = cabi.MaskInfo()
    bitmap = np.empty(max(l, 1), dtype=np.uint8)
    witness = np.empty(m.size, dtype=np.uint8)
    sd = cabi.seeds_struct(cabi.IVC_SEEDS)
    cabi.check(cabi.lib().rbf_compress_mask(c, cabi.ptr(m), m.size, C.byref(sd), float(k), int(l), C.byref(info), cabi.ptr(bitmap),
                                            cabi.ptr(witness)), c)
    assert not info.raw and info.l == l
    return bitmap[:l], witness[:info.wlen], info


def same(got, want, what):
    if not np.array_equal(got, want):
        d = np.flatnonzero(np.asarray(got) != np.asarray(want))
        raise AssertionError("%s: %d positions differ, first %s (got %s, want %s)" % (what, d.size, d[:8].tolist(),
                                                                                   np.asarray(got)[d[:8]].tolist(),
                                                                                   np.asarray(want)[d[:8]].tolist()))


def check_pass(pkg, co, bits, n, k, variant, what, want=None, ctx=None, **opts):
    want = want if want is not None else oracle_pass(co, bits, n, k)
    with options(pkg, ctx, query_variant=variant, **opts):
        got, cnt = gpu_pass(pkg, bits, n, k, ctx)
    same(got, want[0], "%s: pass mask" % what)
    assert cnt == want[1], (what, cnt, want[1])
    return want


def check_encode(pkg, co, m, k, l, variant, what, want=None, **opts):
    if want is None:
        ob, ow, *_ = co.compress(m, k_l_override=(k, l))
        want = (ob, ow)
    with options(pkg, query_variant=variant, **opts):
        bm, wt, info = gpu_compress(pkg, m, k, l)
    same(bm, want[0], "%s: bitmap" % what)
    assert info.wlen == len(want[1]), (what, info.wlen, len(want[1]))
    same(wt, want[1], "%s: witness" % what)
    return want


# ------------------------------------------------------------------ A. filter regimes
# floor(k) 0 (with and without activation), 1, 2, 3 (straight-line stage B), >= 4 (the general probe loop with k_query2's early
# exit), with and without activation; n crosses 10^6 (centuries of 4 and 5 digits)
N_A = 1_000_037
L_A = 400_009
K_A = (0.0, 0.37, 1.0, 1.62, 2.0, 2.5, 3.0, 3.19, 4.0, 4.71, 7.0, 11.3)


@pytest.fixture(scope="module")
def regimes(co):
    rng = np.random.default_rng(301)
    arrays = {f: rand_bits(rng, L_A, f) for f in (0.0, 0.02, 0.5, 0.98, 1.0)}
    cases = [(k, f) for k in K_A for f in (0.02, 0.5, 0.98)] + [(3.19, 0.0), (3.19, 1.0)]
    want = {(k, f): oracle_pass(co, arrays[f], N_A, k) for k, f in cases}
    masks = {p: (rng.random(N_A) < p).astype(np.uint8) for p in (0.01, 0.3)}
    enc = {(k, p): co.compress(masks[p], k_l_override=(k, L_A))[:2] for k in K_A if k > 0 for p in masks}
    return arrays, want, masks, enc


@pytest.mark.parametrize("variant", VARIANTS)
def test_filter_regimes_pass_mask(pkg, co, regimes, variant):
    arrays, want, _, _ = regimes
    for (k, f), w in want.items():
        check_pass(pkg, co, arrays[f], N_A, k, variant, "v%d k=%r fill=%r" % (variant, k, f), want=w)
    # the sparse and dense arrays really are sparse and dense where it matters: few / most positions pass stage A
    assert want[(1.0, 0.02)][1] < N_A // 20 and want[(1.0, 0.98)][1] > N_A * 9 // 10
    assert want[(0.0, 0.5)][1] == N_A                        # k = 0: no probe at all, every position passes


@pytest.mark.parametrize("variant", VARIANTS)
def test_filter_regimes_encode(pkg, co, regimes, variant):
    _, _, masks, enc = regimes
    for (k, p), w in enc.items():
        check_encode(pkg, co, masks[p], k, L_A, variant, "v%d k=%r p=%r" % (variant, k, p), want=w)


# ------------------------------------------------------------------ B. filter sizes
# each side of make_fastmod's m >= 2 and power-of-two branches, 32-bit words, the TY = 10 / 5 switch at 2^23 and the tile / ring
# switch at 2^24
N_B = 300_007
L_B = (1, 2, 3, 31, 32, 33, 127, 128, 129, 4096, 2 ** 20, 2 ** 20 + 1, 2 ** 23 - 1, 2 ** 23, 2 ** 23 + 1, 2 ** 24 - 1, 2 ** 24,
       2 ** 24 + 1)


@pytest.mark.parametrize("l", L_B)
def test_filter_sizes_pass_mask(pkg, co, l):
    bits = rand_bits(np.random.default_rng(l), l, 0.5)
    for k in (2.5, 3.19):
        want = oracle_pass(co, bits, N_B, k)
        for v in VARIANTS:
            check_pass(pkg, co, bits, N_B, k, v, "v%d l=%d k=%r" % (v, l, k), want=want)


# ------------------------------------------------------------------ C. the shared-memory / L2 split
def _expr(src, pattern, **names):
    """Evaluate the integer constant expression `pattern` captures in `src`, C integer division."""
    mt = re.search(pattern, src)
    assert mt, pattern
    return eval(mt.group(1).replace("/", "//"), {"__builtins__": {}}, names)


def query_layout():
    """Fixed shared bytes of each formulation and the launcher's shared-memory ceiling, from the headers."""
    q = (CSRC / "rbf_k3_query.cuh").read_text()
    kc = (CSRC / "rbf_kernels.cu").read_text()
    ring = _expr(q, r"constexpr int Q2_RING = (\d+);")
    q2_warps = _expr(q, r"constexpr int Q2_WARPS = (\d+);")
    q2_ww = _expr(q, r"constexpr int Q2_WARP_WORDS = ([^;]+);", Q2_RING=ring)
    table = _expr(q, r"constexpr int Q4_TABLE_WORDS = (\d+);")
    q4_warps = _expr(q, r"#define RBF_Q4_WARPS (\d+)")

    def q4_ww(ty):
        buf = _expr(q, r"static constexpr int BUF = ([^;]+);", TY=ty)
        return _expr(q, r"static constexpr int WARP_WORDS = ([^;]+);", BUF=buf, Q2_RING=ring)

    smem_max = _expr(kc, r"int query_max_smem_bytes\(\) \{ return ([^;]+);")
    return dict(q2=4 * q2_warps * q2_ww, q4=lambda warps, ty: 4 * (table + warps * q4_ww(ty)), q4_warps=q4_warps, max=smem_max)


def test_query_layout_constants():
    """The layout this file derives from the headers, against the numbers of the default build: a change of layout must be
    looked at here (the boundaries of test_shared_l2_boundary move with it)."""
    lay = query_layout()
    assert lay["q2"] == 4 * 24 * 544 and lay["q4_warps"] == 28 and lay["max"] == 231424
    assert lay["q4"](28, 10) == 4 * (32 + 28 * 608) and lay["q4"](28, 5) == 4 * (32 + 28 * 448)


N_C, L_C = 2_000_003, 1_000_003


def _smem_cases(lay, variant, warps, need):
    """query_smem_bytes that make the bit array fit exactly, fall one 16 B granule short, or leave all but the launcher's
    minimum (qbytes + 1024; 16 B for the per-lane kernel) to L2."""
    if variant == 0:
        q = 0
    elif variant == 1:
        q = lay["q2"]
    else:
        q = lay["q4"](warps or lay["q4_warps"], 5 if variant == 6 else 10)
    exact = q + need
    assert exact <= (lay["max"] & ~15) and q % 16 == 0
    return (("exact", exact), ("short", exact - 16), ("minimum", 16))


@pytest.mark.parametrize("variant,warps", [(0, 0), (1, 0), (5, 4), (5, 7), (5, 28), (6, 4), (6, 7), (6, 28)])
def test_shared_l2_boundary(pkg, co, variant, warps):
    """A ragged l whose bit array fits the shared memory exactly, misses its last 16 B granule (probed through L2), or is
    nearly all in L2; the tile kernel with 4, 7 and 28 warps per CTA (its fixed shared bytes change with them)."""
    lay = query_layout()
    need = 4 * ((((L_C + 31) >> 5) + 3) & ~3)                # the launcher's need_words, in bytes
    rng = np.random.default_rng(401)
    bits = rand_bits(rng, L_C, 0.5)
    m = (rng.random(N_C) < 0.1).astype(np.uint8)
    want_p = oracle_pass(co, bits, N_C, 3.19)
    ob, ow, *_ = co.compress(m, k_l_override=(3.19, L_C))
    for name, smem in _smem_cases(lay, variant, warps, need):
        what = "v%d warps=%d smem=%s(%d)" % (variant, warps, name, smem)
        check_pass(pkg, co, bits, N_C, 3.19, variant, what, want=want_p, query_warps=warps, query_smem_bytes=smem)
        check_encode(pkg, co, m, 3.19, L_C, variant, what, want=(ob, ow), query_warps=warps, query_smem_bytes=smem)


# ------------------------------------------------------------------ D. index-digit boundaries
def _tile_slab_offset(c, total, sm, warps):
    """Offset of century c inside its 32-century slab in a one-frame launch of the tile kernel (launch_query's grid, k_query4's
    split of the centuries over CTAs, and of a CTA's centuries over its warps in slabs of 32)."""
    grid = max(1, min(sm, -(-total // (32 * warps))))
    b = c * grid // total
    while total * (b + 1) // grid <= c:
        b += 1
    while total * b // grid > c:
        b -= 1
    return (c - total * b // grid) % 32


def _digit_cases():
    for d in range(1, 8):
        b = 10 ** d
        for v in (1, 63, 64, 65, 99):
            yield (v if v > b else b + v) if b == 10 else b + v


@pytest.mark.parametrize("n", list(_digit_cases()))
def test_index_digit_boundaries(pkg, co, n):
    """n just past 10^d: the last century holds the first indices of d+1 digits (a new hash kind or string length) and 1, 63,
    64, 65 or 99 valid positions.  It shares its slab with the last centuries of d digits (the per-lane route); the tile kernel
    also runs with 7 warps per CTA, which changes the grid and the slabs' placement once the frame has more than 224 centuries."""
    bits = rand_bits(np.random.default_rng(n), 100_003, 0.5)
    want = oracle_pass(co, bits, n, 3.19)
    for v in VARIANTS:
        for w in ((0, 7) if v >= 5 else (0,)):
            check_pass(pkg, co, bits, n, 3.19, v, "v%d n=%d warps=%d" % (v, n, w), want=want, query_warps=w)


@pytest.mark.parametrize("d", [4, 5, 6, 7])
def test_index_digit_boundary_at_slab_start(pkg, co, d):
    """The first century of d+1-digit indices at the start of a slab of the tile kernel (a uniform slab of the new kind right
    behind a uniform slab of the old one): the frame length and the warps per CTA are searched so that a CTA's slabs put
    century 10^(d-2) first; the last century is ragged (63 valid positions)."""
    sm = pkg._cabi.device_info()["sm_count"]
    cb = 10 ** (d - 2)
    found = next(((cb + t + 1, w) for t in range(32, 20000) for w in range(4, 29)
                  if _tile_slab_offset(cb, cb + t + 1, sm, w) == 0), None)
    assert found, d
    total, w = found
    n = 100 * (total - 1) + 63
    bits = rand_bits(np.random.default_rng(d), 100_003, 0.5)
    want = oracle_pass(co, bits, n, 3.19)
    for v in (5, 6):
        check_pass(pkg, co, bits, n, 3.19, v, "v%d n=%d warps=%d" % (v, n, w), want=want, query_warps=w)


N_D = 100_004_321           # indices >= 10^8: 9 characters, centuries of 7 digits, hash kind K_8B
L_D = (2 ** 23 - 15, 2 ** 24 - 3)


@pytest.fixture(scope="module")
def past_1e8(co):
    """A sparse mask that is set everywhere within 3000 positions of 10^8 and at the end, a bit array per l, and the oracle's
    encode and pass mask for both.  The four oracle runs take several seconds each; ctypes releases the GIL, so they run
    side by side."""
    rng = np.random.default_rng(501)
    m = np.zeros(N_D, dtype=np.uint8)
    m[rng.integers(0, N_D, N_D // 100)] = 1
    m[10 ** 8 - 3000:10 ** 8 + 3000] = 1
    m[N_D - 3000:] = 1
    bits = {l: rand_bits(np.random.default_rng(l), l, 0.5) for l in L_D}
    co.lib()
    with ThreadPoolExecutor(4) as ex:
        enc = {l: ex.submit(co.compress, m, k_l_override=(3.19, l)) for l in L_D}
        pas = {l: ex.submit(oracle_pass, co, bits[l], N_D, 3.19) for l in L_D}
        return m, bits, {l: enc[l].result()[:2] for l in L_D}, {l: pas[l].result() for l in L_D}


@pytest.mark.parametrize("l", L_D)
def test_indices_past_1e8(pkg, co, past_1e8, l):
    """Encode and pass mask at n = 100 004 321 against the full oracle: l <= 2^23 (decade tiles) and 2^23 < l <= 2^24
    (half-decade tiles)."""
    m, bits, enc, pas = past_1e8
    for v in (1, 5, 6):
        check_encode(pkg, co, m, 3.19, l, v, "v%d l=%d" % (v, l), want=enc[l])
        check_pass(pkg, co, bits[l], N_D, 3.19, v, "v%d l=%d" % (v, l), want=pas[l])


# ------------------------------------------------------------------ E. filters of 2^30 bits and more
@pytest.fixture
def own_ctx(pkg):
    """A context of its own: its device scratch (about 5 GB at l = 2^32 - 5) is released when the group is done."""
    L = pkg._cabi.lib()
    h = C.c_void_p()
    pkg._cabi.check(L.rbf_ctx_create(int(os.environ.get("RBF_DEVICE", os.environ.get("LOCAL_RANK", "0"))), C.byref(h)))
    yield h
    L.rbf_ctx_destroy(h)


@pytest.mark.parametrize("l", [2 ** 30, 2 ** 30 + 1, 2 ** 32 - 5])
def test_large_filters(pkg, co, own_ctx, l):
    """l = 2^30 (the last Barrett size), 2^30 + 1 (exact 64-bit `%`), 2^32 - 5 (sums of two indices wrap 32 bits in addmod,
    and (l + 31) >> 5 wraps in uint32).  One host array of l bytes serves the GPU call and the oracle."""
    n = 250_007
    bits = rand_bits(np.random.default_rng(601), l, 0.5)
    try:
        for k in (2.5, 4.0):
            want = oracle_pass(co, bits, n, k)
            for v in (0, 1, 5):
                check_pass(pkg, co, bits, n, k, v, "v%d l=%d k=%r" % (v, l, k), want=want, ctx=own_ctx)
    finally:
        del bits


# ------------------------------------------------------------------ F. heterogeneous launches
# one K3 launch over frames with different l, floor(k) and activation, raw pairs (no centuries in the work list) first, in the
# middle and last.  (k, l, mask density); l = 0 or l >= n and a density >= P* make raw pairs.
H_F, W_F = 540, 960
N_F = H_F * W_F
SPREAD = [(1.0, 0, 0.05), (0.37, 1, 0.02), (1.0, 2, 0.05), (2.0, 64, 0.1), (2.5, 2 ** 16, 0.05), (3.19, 1000, 0.4),
          (3.0, N_F - 1, 0.03), (3.19, 40_009, 0.05), (4.0, 2 ** 16, 0.01), (4.71, N_F - 17, 0.2), (5.0, 64, 0.05),
          (6.5, 2, 0.05), (7.0, 250_007, 0.05), (2.5, N_F, 0.05)]


def _spread_frames():
    rng = np.random.default_rng(701)
    masks = [(rng.random(N_F) < p).astype(np.uint8) for _, _, p in SPREAD]
    frames = np.zeros((len(SPREAD) + 1, H_F, W_F), dtype=np.uint8)
    for t, m in enumerate(masks):                          # |dY| = 128 exactly where the mask is set
        frames[t + 1] = frames[t] ^ (m.reshape(H_F, W_F) << 7)
    return masks, frames


def test_heterogeneous_encode(pkg, co):
    masks, frames = _spread_frames()
    F = len(SPREAD)
    st = pkg.FrameStream(H_F, W_F, 1, np.uint8, max_frames=F + 1)
    try:
        st.upload(frames)
        for v in VARIANTS:
            with options(pkg, query_variant=v):
                res = st.encode(list(range(F)), list(range(1, F + 1)), 3.0, k_override=[s[0] for s in SPREAD],
                                l_override=[s[1] for s in SPREAD])
            raw = []
            for t, ((k, l, _), r) in enumerate(zip(SPREAD, res)):
                bm, wt, mask = st.fetch(t)
                same(mask, masks[t], "v%d pair %d: mask" % (v, t))
                ob, ow, op, on, oratio, ok, ol = co.compress(masks[t], k_l_override=(k, l))
                raw.append(r.raw)
                if ok == 0:
                    assert r.raw and r.l == 0, (v, t, r)
                    continue
                assert (r.l, r.k, r.wlen) == (ol, ok, len(ow)), (v, t, r)
                same(bm, np.packbits(ob), "v%d pair %d: bitmap" % (v, t))
                same(wt, np.packbits(ow), "v%d pair %d: witness" % (v, t))
            assert raw[0] and raw[5] and raw[-1] and sum(raw) == 3
            with options(pkg, query_variant=v):
                assert not st.decode_verify().any(), v
    finally:
        st.close()


def test_heterogeneous_decode_masks(pkg, co):
    """FrameStream.decode_masks over the same spread, random bit arrays, all-ones witnesses: consumed[i] is the oracle's pass
    count, and every decoded mask is read back through apply_chain (pair i writes the value i + 1 onto a zero frame)."""
    rng = np.random.default_rng(702)
    F = len(SPREAD)
    nb = (N_F + 7) // 8
    raw = [ol == 0 or ol >= N_F or p >= 0.32453 for _, ol, p in SPREAD]
    bslot = (nb + 15) // 16 * 16
    bms = np.zeros((F, bslot), dtype=np.uint8)
    wts = np.full((F, bslot), 0xFF, dtype=np.uint8)
    want = []
    for i, (k, l, _) in enumerate(SPREAD):
        if raw[i]:
            m = (rng.random(N_F) < 0.3).astype(np.uint8)
            bms[i, :nb] = np.packbits(m)
            want.append((m, 0))
        else:
            bits = rand_bits(rng, l, 0.5)
            bms[i, :(l + 7) // 8] = np.packbits(bits)
            want.append(oracle_pass(co, bits, N_F, k))
    st = pkg.FrameStream(H_F, W_F, 1, np.uint8, max_frames=F + 1, max_pairs=F, k1_only=True)
    try:
        for v in VARIANTS:
            with options(pkg, query_variant=v):
                consumed, ones = st.decode_masks(bms, wts, [0 if r else s[1] for r, s in zip(raw, SPREAD)],
                                                 [0 if r else N_F for r in raw], [s[0] for s in SPREAD], raw)
            assert list(consumed) == [w[1] for w in want], v
            assert list(ones) == [int(w[0].sum()) for w in want], v
            st.upload(np.zeros((H_F, W_F), dtype=np.uint8), first=0)
            applied = st.apply_chain(0, [np.full(int(ones[i]), i + 1, dtype=np.uint8) for i in range(F)])
            assert list(applied) == list(ones), v
            got = st.download_batch(1, F)
            for i in range(F):
                same((got[i].reshape(-1) == i + 1).astype(np.uint8), want[i][0], "v%d pair %d: decoded mask" % (v, i))
    finally:
        st.close()


# ------------------------------------------------------------------ G. witness chunks (K3b / K4b) and witness lengths
def _witness_chunks(F, ncent, sm):
    """K3b / K4b chunks per frame (launch_witness / launch_expand): >= 8 waves of the GPU, >= 4096 centuries a chunk, <= 32."""
    return max(1, min(-(-16 * sm // F), ncent // 4096, 32))


@pytest.mark.parametrize("ncent", [8191, 8192, 8193, 140_000])
def test_witness_chunks(pkg, co, ncent):
    """One frame of 1, 2, 2 and 32 (capped) chunks; the last century is ragged.  Witness and length against the oracle, and the
    decode with the exact witness, one bit short (IndexError, as the reference's list index) and 64 bits to spare."""
    n = 100 * ncent - 37
    sm = pkg._cabi.device_info()["sm_count"]
    assert _witness_chunks(1, ncent, sm) == {8191: 1, 8192: 2, 8193: 2}.get(ncent, 32)
    m = (np.random.default_rng(ncent).random(n) < 0.05).astype(np.uint8)
    ob, ow, op, on, oratio, ok, ol = co.compress(m)
    assert ok > 0
    comp = pkg.BloomFilterCompressor()
    for v in VARIANTS:
        check_encode(pkg, co, m, ok, ol, v, "v%d ncent=%d" % (v, ncent), want=(ob, ow))
        with options(pkg, query_variant=v):
            same(comp.decompress(ob, ow, n, ok), m, "v%d ncent=%d: decode" % (v, ncent))
            with pytest.raises(IndexError):
                comp.decompress(ob, ow[:-1], n, ok)
            same(comp.decompress(ob, np.concatenate([ow, np.zeros(64, np.uint8)]), n, ok), m, "v%d ncent=%d: +64" % (v, ncent))


def test_witness_chunks_follow_pair_count(pkg, co):
    """A stream with enough pairs that the chunk count per frame drops below its one-frame value (the pairs alternate between
    two masks over three frames): every pair's bitmap and witness against the oracle, and the batched decode round trip."""
    H, W = 3201, 4096
    n = H * W
    ncent = (n + 99) // 100
    sm = pkg._cabi.device_info()["sm_count"]
    F = 96
    assert _witness_chunks(F, ncent, sm) < _witness_chunks(1, ncent, sm) == 32
    rng = np.random.default_rng(801)
    masks = [(rng.random(n) < p).astype(np.uint8) for p in (0.05, 0.02)]
    frames = np.zeros((3, H, W), dtype=np.uint8)
    for t in range(2):
        frames[t + 1] = frames[t] ^ (masks[t].reshape(H, W) << 7)
    want = [co.compress(m) for m in masks]
    st = pkg.FrameStream(H, W, 1, np.uint8, max_frames=3, max_pairs=F)
    try:
        st.upload(frames)
        res = st.encode([0, 1] * (F // 2), [1, 2] * (F // 2), 3.0)
        bms, wts, _ = st.fetch_batch(0, F)
        for t, r in enumerate(res):
            ob, ow, op, on, oratio, ok, ol = want[t % 2]
            assert (r.l, r.k, r.wlen) == (ol, ok, len(ow)), (t, r)
            same(bms[t, :(ol + 7) // 8], np.packbits(ob), "pair %d: bitmap" % t)
            same(wts[t, :(len(ow) + 7) // 8], np.packbits(ow), "pair %d: witness" % t)
        assert not st.decode_verify().any()
    finally:
        st.close()
