"""The item-keyed Bloom filters on the device -- IndexRationalBloomFilter (ivc:39-138), RationalBloomFilter and
StandardBloomFilter (rbf:9-214), i.e. k_items_u32 / k_items_str and the k_pack_bytes / k_unpack_bits pair behind the
bit_array getter and setter -- compared bit for bit with two references:

  * oracle/rbf_oracle.py: plain Python, unbounded-int `(h1 + i*h2) % m`, the reference's `bit_array[idx] == 0` tests.
    Used for small cases and for the set of bit positions of filters too large to materialise twice.
  * oracle/c_oracle.py (filter_add_strings / filter_check_strings over str(item)): used for batches.

StandardBloomFilter's model is `xxh64(str(item), seed=i) % m` for i < k (rbf:25-41).

Groups (GPU): A index route, B string route, C filter sizes (both sides of the exact-`%` size 2^30 + 1 and of the
33-bit `addmod` carry at 2^31), D k regimes, E batches longer than one grid-stride pass, F bit-array I/O, G bit arrays
holding bytes other than 0 and 1.  The CPU part checks that the case lists reach what they claim to reach.
"""
import math
import os
import random

import numpy as np
import pytest

from oracle import rbf_oracle as ro
from oracle.rbf_oracle import BC_SEEDS, IVC_SEEDS, rbf_seeds

U32 = 2 ** 32


@pytest.fixture(scope="module")
def co():
    from oracle import c_oracle
    c_oracle.build()
    return c_oracle


@pytest.fixture(scope="module")
def pkg():
    import new_bloom_filter_repo_b200 as p
    info = p._cabi.device_info()
    assert info["cc"] == (9, 0), info
    return p


# ------------------------------------------------------------------ case lists
def century_kind(i: int):
    """make_century's rule (csrc/rbf_hash.cuh) restated: the century hq = i // 100 has strings of L = digits(hq) + 2
    characters (century 0: L = 2, its first decade one character), and L alone picks where the last two digits fall in
    XXH64's lane order.  -> (kind, length of str(i))."""
    hq = i // 100
    L = 2 if hq == 0 else len(str(hq)) + 2
    kind = {4: "K_44", 5: "K_4B", 8: "K_88", 9: "K_8B"}.get(L, "K_BB")
    return kind, (1 if i < 10 else L)


def index_cases(seed=11):
    """name -> uint32 items of group A."""
    edges = set()
    for d in range(1, 10):
        for v in (10 ** d - 1, 10 ** d):
            c = v // 100
            edges.update(range(c * 100, c * 100 + 100))
    rng = np.random.default_rng(seed)
    strat = [rng.integers(0 if d == 1 else 10 ** (d - 1), min(10 ** d, U32), 10_000, dtype=np.uint64) for d in range(1, 11)]
    return {
        "all_0_12000": np.arange(12_001, dtype=np.uint32),
        "century_edges": np.array(sorted(edges), dtype=np.uint32),
        "billion": np.arange(10 ** 9, 10 ** 9 + 301, dtype=np.uint32),
        "top": np.arange(U32 - 300, U32, dtype=np.uint64).astype(np.uint32),
        "stratified": np.concatenate(strat).astype(np.uint32),
    }


def index_non_members(members, seed=12, per_digits=2_000):
    rng = np.random.default_rng(seed)
    cand = np.concatenate([rng.integers(0 if d == 1 else 10 ** (d - 1), min(10 ** d, U32), per_digits, dtype=np.uint64)
                           for d in range(1, 11)]).astype(np.uint32)
    return cand[~np.isin(cand, members)]


STR_LENGTHS = list(range(81)) + [127, 128, 129, 1000, 4097]
UTF8_ITEMS = ["\u00e9", "\u00f1and\u00fa", "\u20ac", "\u65e5\u672c\u8a9e", "\U0001F600", "\U0001D11E clef",
              "e\u0301", "a\u0300\u0301\u0302", "\u00e9" * 40, "\U0001F600" * 9, "\u20ac" * 11,
              "\u03a9\u2248\u00e7\u221a", "\U0001F1EB\U0001F1F7", "x\U0001F600y\u20acz\u00e9" * 5]
NUL_ITEMS = ["\0", "a\0", "\0b", "abc\0def", "\0" * 32, "x" * 31 + "\0", "\0" * 4097]


def _rand_str(rng, n, alphabet=None):
    if alphabet is None:
        return "".join(chr(rng.randrange(1, 128)) for _ in range(n))
    return "".join(rng.choice(alphabet) for _ in range(n))


def string_cases(seed=5):
    """-> (items, length of each content item or None for a pad, last-byte partners).  For every length of STR_LENGTHS,
    16 contents packed so that their starts (in the blob of the concatenated UTF-8 items) fall on every offset mod 16;
    pad items of 1..15 bytes shift the next start.  Then multi-byte UTF-8, embedded NULs, and strings whose partner
    (kept out of the filter) differs only in the last byte."""
    rng = random.Random(seed)
    items, tags, pos = [], [], 0

    def push(s, tag):
        nonlocal pos
        items.append(s)
        tags.append(tag)
        pos += len(s.encode("utf-8"))

    alphabets = [None, "abcdefghijklmnopqrstuvwxyz", "0123456789", "".join(map(chr, range(32, 127)))]
    for L in STR_LENGTHS:
        for r in range(16):
            pad = (r - pos) % 16
            if pad:
                push(_rand_str(rng, pad), None)
            push(_rand_str(rng, L, alphabets[r % 4]), L)
    for s in UTF8_ITEMS + NUL_ITEMS:
        push(s, None)
    partners = []
    for L in list(range(1, 41)) + [63, 64, 65, 100, 1000]:
        s = _rand_str(rng, L, "abcdefghijklmnopqrstuvwxyz")
        push(s, None)
        partners.append(s[:-1] + chr(ord(s[-1]) ^ 1))
    return items, tags, partners


def string_non_members(members, seed=6, count=10_000):
    rng = random.Random(seed)
    ms = set(members)
    out = []
    while len(out) < count:
        s = _rand_str(rng, rng.randrange(0, 120), None if rng.random() < 0.5 else "abcdefghijklmnopqrstuvwxyz0123456789")
        if s not in ms:
            out.append(s)
    out += ["\u00fc" * n for n in range(1, 30)] + ["\0" * n for n in (2, 3, 33)]
    return [s for s in out if s not in ms]


def xxh64_tail_class(n: int):
    """Where XXH64 ends on an n-byte input: ("short", n) below 32 bytes -- 8-byte lanes, an optional 4-byte lane and
    single bytes -- or ("stripes", n mod 32) after whole 32-byte stripes."""
    return ("short", n) if n < 32 else ("stripes", n % 32)


FAST_MOD_MAX = 2 ** 30        # FastMod takes the Barrett path for 2 <= m <= 2^30, the exact 64-bit `%` otherwise
SIZES = [1, 2, 3, 31, 32, 33, 2 ** 24 - 1, 2 ** 24 + 1, 2 ** 30 - 1, 2 ** 30, 2 ** 30 + 1, 2 ** 31 - 1, 2 ** 31 + 1,
         U32 - 5, U32 - 1]
SMALL_SIZE = 2 ** 24 + 1      # up to here a case compares the whole bit array; above it, the set of set positions

K_STARS = [0.0, 0.1, 0.5, 0.999999, 1.0, 2.3, 3.0, 12.99]
K_STANDARD = [0, 1, 2, 7, 33, 64]
ODD_BYTES = np.array([2, 3, 128, 255], dtype=np.uint8)


def strs(items):
    return [x if isinstance(x, str) else str(x) for x in (items.tolist() if isinstance(items, np.ndarray) else items)]


def grid_passes(count: int, block: int, sm_count: int) -> int:
    """Grid-stride passes of a launch sized by grid_for (csrc/rbf_kernels.cu): at most 16 CTAs per SM."""
    grid = max(1, min((count + block - 1) // block, 16 * sm_count))
    return -(-count // (grid * block))


def c_bits(co, m, k, seeds, items):
    bits = np.zeros(m, dtype=np.uint8)
    if len(items):
        co.filter_add_strings(bits, k, seeds, strs(items))
    return bits


def ro_positions(m, k, seeds, items):
    """Set positions of rbf_oracle's filter after adding items, without materialising a bit array."""
    f = ro.RationalBloomFilter.__new__(ro.RationalBloomFilter)
    f.size, f.k_star, f.floor_k = m, k, math.floor(k)
    f.p_activation = k - f.floor_k
    f.h1_seed, f.h2_seed, f.act_seed = seeds
    pos = set()
    for it in items:
        for i in range(f.floor_k):
            pos.add(f._get_hash_indices(it, i))
        if f._determine_activation(it):
            pos.add(f._get_hash_indices(it, f.floor_k))
    return pos


def std_positions(co, m, k, items):
    return {co.xxh64(s.encode("utf-8"), i) % m for s in strs(items) for i in range(k)}


def std_contains(co, bits, k, items):
    m = len(bits)
    return np.array([all(bits[co.xxh64(s.encode("utf-8"), i) % m] for i in range(k)) for s in strs(items)], dtype=bool)


def odd_bitmap(bits01, seed):
    """The 0/1 array with every 1 replaced by one of 2, 3, 128, 255."""
    rng = np.random.default_rng(seed)
    return np.where(bits01 != 0, ODD_BYTES[rng.integers(0, 4, len(bits01))], 0).astype(np.uint8)


def launches(pkg):
    return pkg._cabi.lib().rbf_get_counter(pkg._cabi.ctx(), b"kernel_launches")


# ------------------------------------------------------------------ CPU: the case lists reach their edges
def test_string_cases_reach_every_xxh64_tail_class():
    items, tags, partners = string_cases()
    lens = {len(s.encode("utf-8")) for s in items + partners}
    classes = {xxh64_tail_class(n) for n in lens}
    assert {("short", n) for n in range(32)} <= classes               # < 4, the 4-byte lane, every residue of 8..31
    assert {("stripes", r) for r in range(32)} <= classes             # 32-byte stripes plus each tail
    assert 0 in lens and 32 in lens and 4097 in lens
    assert any(n % 8 >= 4 for n in lens if n < 32) and any(n % 32 % 8 >= 4 for n in lens if n >= 32)
    # every content length starts at every offset mod 16 of the packed blob
    offs = np.concatenate([[0], np.cumsum([len(s.encode("utf-8")) for s in items])])
    for L in STR_LENGTHS:
        starts = {int(offs[j]) % 16 for j, t in enumerate(tags) if t == L}
        assert starts == set(range(16)), L
    # 2-, 3- and 4-byte code points, combining marks and NULs reach the device
    blob = "".join(items)
    widths = {len(ch.encode("utf-8")) for ch in blob}
    assert widths == {1, 2, 3, 4}
    assert "\u0301" in blob and "\0" in blob
    assert all(len(a) == len(b) and a[:-1] == b[:-1] and a != b for a, b in zip(items[-len(partners):], partners))


def test_index_cases_reach_every_century_kind():
    cases = index_cases()
    items = np.unique(np.concatenate(list(cases.values())))
    for i in (0, 9, 10, 99, 100, 999, 1000, 99_999_999, 100_000_000, 999_999_999, 10 ** 9, U32 - 1):
        kind, L = century_kind(i)
        assert L == len(str(i)), i
    kinds = {century_kind(int(i)) for i in items}
    assert {("K_BB", L) for L in (1, 2, 3, 6, 7, 10)} <= kinds
    assert {("K_4B", 5), ("K_8B", 9), ("K_44", 4), ("K_88", 8)} <= kinds
    counts = np.bincount([len(str(int(i))) for i in cases["stratified"]], minlength=11)
    assert (counts[1:] >= 10_000).all(), counts
    for d in range(1, 10):                                         # both sides of every digit-count boundary
        assert 10 ** d - 1 in items and 10 ** d in items
    assert 10 ** 9 + 300 in items and U32 - 300 in items and U32 - 1 in items


def test_sizes_straddle_the_exact_mod_and_carry_edges():
    assert 1 in SIZES                                              # m = 1 takes the exact `%` too
    assert max(m for m in SIZES if m <= FAST_MOD_MAX) == FAST_MOD_MAX and FAST_MOD_MAX + 1 in SIZES
    assert any(2 <= m < 2 ** 24 for m in SIZES) and any(FAST_MOD_MAX < m < 2 ** 31 for m in SIZES)
    assert any(m > 2 ** 31 for m in SIZES) and 2 ** 31 - 1 in SIZES and U32 - 1 in SIZES
    assert max(SIZES) < U32 and min(SIZES) >= 1
    assert grid_passes(2_000_003, 256, 132) > 1 and grid_passes(700_001, 128, 132) > 1


def test_oracles_agree_on_non01_bitmaps(co):
    """A bit array byte counts as set when it is non-zero, in rbf_oracle (`== 0`, ivc:129,135) and in the C oracle
    (`!bits[idx]`) alike; a numpy bool array reads the same."""
    m, k = 4_000, 2.6
    members = list(range(0, 3_000, 7))
    bits = c_bits(co, m, k, IVC_SEEDS, members)
    odd = odd_bitmap(bits, 1)
    assert set(np.unique(odd)) - {0} <= set(ODD_BYTES.tolist()) and len(set(np.unique(odd)) - {0}) == 4
    probes = list(range(3_000))
    want = co.filter_check_strings(odd, k, IVC_SEEDS, strs(probes)).astype(bool)
    assert np.array_equal(want, co.filter_check_strings(bits, k, IVC_SEEDS, strs(probes)).astype(bool))
    assert np.array_equal(want, co.filter_check_strings(odd.astype(bool).astype(np.uint8), k, IVC_SEEDS, strs(probes)).astype(bool))
    for bm in (odd, odd.astype(bool)):
        f = ro.RationalBloomFilter(m, k, IVC_SEEDS)
        f.bit_array = bm
        assert np.array_equal(want, [f.check_index(i) for i in probes])
    assert want[members].all() and not want.all()
    # BloomFilterCompressor.decompress (ivc:268-307) on such a bitmap
    rng = np.random.default_rng(2)
    mask = (rng.random(2_000) < 0.06).astype(np.uint8)
    b, w = co.compress_kl(mask, 2.2, 300)
    odd_b = odd_bitmap(b, 3)
    out_c = co.decompress(odd_b, w, len(mask), 2.2)
    assert np.array_equal(out_c, mask)
    assert np.array_equal(ro.decompress(odd_b, list(w), len(mask), 2.2), mask)


# ------------------------------------------------------------------ A. index route
A_FILTERS = [(1_000_003, 2.3, IVC_SEEDS), (1 << 20, 3.7, BC_SEEDS), (524_287, 4.6, rbf_seeds(4.6))]


@pytest.mark.gpu
def test_a_index_route_vs_oracles(pkg, co):
    cases = index_cases()
    members = np.concatenate(list(cases.values()))
    non = index_non_members(members)
    assert len(non) >= 10_000
    for m, k, seeds in A_FILTERS:
        f = pkg.IndexRationalBloomFilter(m, k, seeds)
        for name in cases:                                         # one call per case
            f.add_indices(cases[name])
        want = c_bits(co, m, k, seeds, members)
        got = f.bit_array
        assert np.array_equal(got, want), (m, k, seeds, np.flatnonzero(got != want)[:8])
        assert f.check_indices(members).all()
        chk = f.check_indices(non)
        assert np.array_equal(chk, co.filter_check_strings(want, k, seeds, strs(non)).astype(bool)), (m, k)
        assert not chk.all()
        # the string route over str(i) sets the same bits
        g = pkg.IndexRationalBloomFilter(m, k, seeds)
        g._dev.add_strings(strs(members))
        assert np.array_equal(g.bit_array, want)
        assert np.array_equal(g._dev.check_strings(strs(non)).astype(bool), chk)
    # the digit-count edges against the pure-Python oracle, as a set of positions
    edge = np.concatenate([cases["century_edges"], cases["billion"], cases["top"]])
    for m, k, seeds in A_FILTERS:
        f = pkg.IndexRationalBloomFilter(m, k, seeds)
        f.add_indices(edge)
        assert set(np.flatnonzero(f.bit_array).tolist()) == ro_positions(m, k, seeds, edge.tolist()), (m, k)


# ------------------------------------------------------------------ B. string route
B_RATIONAL = [(200_003, 2.3), (65_536, 5.5), (4_099, 1.0)]
B_STANDARD = [(200_003, 3), (65_536, 7)]


@pytest.mark.gpu
def test_b_string_route_both_classes(pkg, co):
    items, _, partners = string_cases()
    non = string_non_members(items) + [p for p in partners if p not in set(items)]
    assert len(non) >= 10_000
    for m, k in B_RATIONAL:
        f = pkg.RationalBloomFilter(m, k)
        f.add_many(items[:100])
        for s in items[100:110]:
            f.add(s)                                               # the reference's one-item signature
        f.add_many(items[110:])
        want = c_bits(co, m, k, rbf_seeds(k), items)
        got = np.array(f.bit_array, dtype=np.uint8)
        assert np.array_equal(got, want), (m, k, np.flatnonzero(got != want)[:8])
        assert f.contains_many(items).all() and f.contains(items[-1])
        chk = f.contains_many(non)
        assert np.array_equal(chk, co.filter_check_strings(want, k, rbf_seeds(k), non).astype(bool)), (m, k)
        assert not chk.all()
    small = [s for s in items if len(s) <= 40][:300] + UTF8_ITEMS + NUL_ITEMS[:-1]
    f = pkg.RationalBloomFilter(50_021, 2.3)
    f.add_many(small)
    assert set(np.flatnonzero(f.bit_array).tolist()) == ro_positions(50_021, 2.3, rbf_seeds(2.3), small)
    for m, k in B_STANDARD:
        f = pkg.StandardBloomFilter(m, k)
        f.add_many(items)
        got = np.array(f.bit_array, dtype=np.uint8)
        assert set(np.flatnonzero(got).tolist()) == std_positions(co, m, k, items), (m, k)
        assert f.contains_many(items).all()
        chk = f.contains_many(non)
        assert np.array_equal(chk, std_contains(co, got, k, non)), (m, k)
        assert not chk.all()


# ------------------------------------------------------------------ C. filter sizes
C_INDICES = np.array(sorted({0, 7, 42, 99, 100, 12_345, 999_999, 10 ** 6, 87_654_321, 99_999_999, 10 ** 8, 999_999_999,
                             10 ** 9, 3_000_000_000, U32 - 1} | set(range(1_000, 1_200)) | set(range(U32 - 150, U32 - 1))),
                     dtype=np.uint32)
C_STRINGS = ["s%d" % i for i in range(60)] + ["", "x" * 32, "y" * 47, "\u00e9\u20ac\U0001F600"] + ["z" * n for n in range(1, 36)]
C_K = 3.5


def _size_case(pkg, co, m):
    """Index filter (u32 and string routes) and a k = 3 standard filter of size m against the models."""
    rng = np.random.default_rng(m % 1000)
    non = rng.integers(0, U32, 12_000, dtype=np.uint64).astype(np.uint32)
    non = non[~np.isin(non, C_INDICES)]
    non_s = ["q%d" % i for i in range(2_000)]
    f = pkg.IndexRationalBloomFilter(m, C_K)
    f.add_indices(C_INDICES)
    f.add_indices(np.array(C_STRINGS, dtype=object))
    assert f.check_indices(C_INDICES).all() and f.check_indices(np.array(C_STRINGS, dtype=object)).all()
    members = strs(C_INDICES) + C_STRINGS
    got = f._dev.get_bits()
    if m <= SMALL_SIZE:
        want = c_bits(co, m, C_K, IVC_SEEDS, members)
        assert np.array_equal(got, want), m
    else:
        assert set(np.flatnonzero(got).tolist()) == ro_positions(m, C_K, IVC_SEEDS, members), m
    assert np.array_equal(f.check_indices(non), co.filter_check_strings(got, C_K, IVC_SEEDS, strs(non)).astype(bool)), m
    assert np.array_equal(f._dev.check_strings(non_s).astype(bool), co.filter_check_strings(got, C_K, IVC_SEEDS, non_s).astype(bool))
    del got, f
    s = pkg.StandardBloomFilter(m, 3)
    s.add_many(members)
    got = s._dev.get_bits()
    assert set(np.flatnonzero(got).tolist()) == std_positions(co, m, 3, members), m
    assert s.contains_many(members).all()
    probe = strs(non[:10_000])
    assert np.array_equal(s.contains_many(probe), std_contains(co, got, 3, probe)), m
    del got, s


@pytest.mark.gpu
@pytest.mark.parametrize("m", [m for m in SIZES if m <= 2 ** 30])
def test_c_filter_sizes(pkg, co, m):
    _size_case(pkg, co, m)


@pytest.mark.gpu
def test_c_filter_sizes_above_2_30(pkg, co):
    """Every size above 2^30 takes the exact 64-bit `%`, and above 2^31 the probe walk's sum carries into bit 32.  One
    get_bits host buffer of up to 4 GiB at a time."""
    for m in [m for m in SIZES if m > 2 ** 30]:
        _size_case(pkg, co, m)


@pytest.mark.gpu
def test_c_sizes_0_and_2_32_raise(pkg):
    for cls, arg in ((pkg.IndexRationalBloomFilter, 2.3), (pkg.RationalBloomFilter, 2.3), (pkg.StandardBloomFilter, 3)):
        with pytest.raises(ValueError):
            cls(0, arg)
        with pytest.raises(pkg._cabi.RbfError, match=r"outside \[1, 2\^32\)"):
            cls(U32, arg)


# ------------------------------------------------------------------ D. k regimes
@pytest.mark.gpu
@pytest.mark.parametrize("k", K_STARS + [40.5])
def test_d_rational_k(pkg, co, k):
    m = 7 if k == 40.5 else 100_003                                # k* = 40.5 on m = 7: the probe walk wraps the array
    idx = np.arange(0, 3_000 * 37, 37, dtype=np.uint32)
    words = ["w%d" % i for i in range(3_000)]
    non_i = np.arange(1, 12_000 * 37, 37, dtype=np.uint32)
    non_w = ["v%d" % i for i in range(12_000)]
    f = pkg.IndexRationalBloomFilter(m, k)
    f.add_indices(idx)
    g = pkg.RationalBloomFilter(m, k)
    g.add_many(words)
    for dev, seeds, mem, non, check in ((f, IVC_SEEDS, idx, non_i, f.check_indices), (g, rbf_seeds(k), words, non_w, g.contains_many)):
        want = c_bits(co, m, k, seeds, mem)
        got = np.array(dev.bit_array, dtype=np.uint8)
        assert np.array_equal(got, want), (k, seeds)
        few = pkg.IndexRationalBloomFilter(m, k, seeds)
        few.add_indices(np.array(strs(mem[:150]), dtype=object) if dev is g else mem[:150])
        assert set(np.flatnonzero(few.bit_array).tolist()) == ro_positions(m, k, seeds, strs(mem[:150])), (k, seeds)
        assert check(mem).all()
        chk = check(non)
        assert np.array_equal(chk, co.filter_check_strings(want, k, seeds, strs(non)).astype(bool)), (k, seeds)
        if k == 0:
            assert not got.any() and chk.all()                     # no probe at all: nothing set, everything passes
        elif m > 7 and k >= 1:
            assert not chk.all()


@pytest.mark.gpu
@pytest.mark.parametrize("k", K_STANDARD)
def test_d_standard_k(pkg, co, k):
    m = 100_003
    items = ["i%d" % i for i in range(2_000)]
    non = ["n%d" % i for i in range(10_000)]
    f = pkg.StandardBloomFilter(m, k)
    f.add_many(items)
    got = np.array(f.bit_array, dtype=np.uint8)
    assert set(np.flatnonzero(got).tolist()) == std_positions(co, m, k, items)
    assert f.contains_many(items).all()
    chk = f.contains_many(non)
    assert np.array_equal(chk, std_contains(co, got, k, non))
    if k == 0:
        assert not got.any() and chk.all()
    else:
        assert not chk.all()
    if k:                                                          # the device's contains, not the class's k == 0 shortcut
        assert np.array_equal(f._dev.check_strings(non, standard_k=k).astype(bool), chk)


# ------------------------------------------------------------------ E. batches longer than one grid pass
@pytest.mark.gpu
def test_e_index_batch_past_one_grid_pass(pkg, co):
    sm = pkg._cabi.device_info()["sm_count"]
    n, m, k = 2_000_003, 2 ** 24 + 1, 2.3
    assert grid_passes(n, 256, sm) > 1
    rng = np.random.default_rng(21)
    items = rng.integers(0, U32, n, dtype=np.uint64).astype(np.uint32)
    f = pkg.IndexRationalBloomFilter(m, k)
    f.add_indices(items)
    want = c_bits(co, m, k, IVC_SEEDS, items)
    assert np.array_equal(f.bit_array, want)
    # the same items in 7 uneven calls, with duplicates across and within calls
    cuts = np.sort(rng.choice(np.arange(1, n), 6, replace=False))
    g = pkg.IndexRationalBloomFilter(m, k)
    for part in np.split(items, cuts):
        g.add_indices(np.concatenate([part, part[: len(part) // 3]]))
    assert np.array_equal(g.bit_array, want)
    h = pkg.IndexRationalBloomFilter(m, k)
    h.add_indices(np.concatenate([items, items[::-5]]))
    assert np.array_equal(h.bit_array, want)
    # one check call over members and non-members mixed
    probe = np.concatenate([items[: n // 2], rng.integers(0, U32, n - n // 2, dtype=np.uint64).astype(np.uint32)])
    rng.shuffle(probe)
    chk = f.check_indices(probe)
    assert np.array_equal(chk, co.filter_check_strings(want, k, IVC_SEEDS, strs(probe)).astype(bool))
    assert f.check_indices(items).all()


@pytest.mark.gpu
def test_e_string_batch_past_one_grid_pass(pkg, co):
    sm = pkg._cabi.device_info()["sm_count"]
    n, m, k = 700_001, 4_000_037, 2.3
    assert grid_passes(n, 128, sm) > 1
    rng = random.Random(22)
    items = ["%x:%s" % (i, "ab" * rng.randrange(0, 20)) for i in range(n)]
    f = pkg.RationalBloomFilter(m, k)
    f.add_many(items)
    want = c_bits(co, m, k, rbf_seeds(k), items)
    assert np.array_equal(np.array(f.bit_array, dtype=np.uint8), want)
    g = pkg.RationalBloomFilter(m, k)
    cuts = sorted(rng.sample(range(1, n), 6))
    for a, b in zip([0] + cuts, cuts + [n]):
        g.add_many(items[a:b] + items[a:b:4])
    assert np.array_equal(np.array(g.bit_array, dtype=np.uint8), want)
    probe = items[::2] + ["%x!" % i for i in range(n - len(items[::2]))]
    rng.shuffle(probe)
    chk = f.contains_many(probe)
    assert np.array_equal(chk, co.filter_check_strings(want, k, rbf_seeds(k), probe).astype(bool))
    assert f.contains_many(items).all()
    # the standard filter strides the same loop
    s = pkg.StandardBloomFilter(m, 2)
    s.add_many(items)
    got = np.array(s.bit_array, dtype=np.uint8)
    assert set(np.flatnonzero(got).tolist()) == std_positions(co, m, 2, items)
    assert s.contains_many(items).all()
    assert np.array_equal(s.contains_many(probe), std_contains(co, got, 2, probe))


@pytest.mark.gpu
def test_e_empty_batch_launches_nothing(pkg):
    f = pkg.IndexRationalBloomFilter(1000, 2.3)
    r = pkg.RationalBloomFilter(1000, 2.3)
    s = pkg.StandardBloomFilter(1000, 3)
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    items, out = np.zeros(1, dtype=np.uint32), np.zeros(1, dtype=np.uint8)
    offs = np.zeros(1, dtype=np.uint64)
    before = launches(pkg)
    f.add_indices([])
    assert f.check_indices(np.zeros(0, dtype=np.uint32)).shape == (0,)
    r.add_many([])
    assert r.contains_many([]).shape == (0,)
    s.add_many([])
    assert s.contains_many([]).shape == (0,)
    for dev in (f._dev, r._dev, s._dev):                           # count = 0 through the C ABI itself
        h = dev._h
        pkg._cabi.check(L.rbf_filter_add_indices(h, pkg._cabi.ptr(items), 0), ctx)
        pkg._cabi.check(L.rbf_filter_check_indices(h, pkg._cabi.ptr(items), 0, pkg._cabi.ptr(out)), ctx)
        for sk in (0, 3):
            pkg._cabi.check(L.rbf_filter_add_strings(h, pkg._cabi.ptr(out), pkg._cabi.ptr(offs), 0, sk), ctx)
            pkg._cabi.check(L.rbf_filter_check_strings(h, pkg._cabi.ptr(out), pkg._cabi.ptr(offs), 0, sk, pkg._cabi.ptr(out)), ctx)
    assert launches(pkg) == before
    assert not f.bit_array.any() and not any(r.bit_array) and not any(s.bit_array)


# ------------------------------------------------------------------ F. bit-array I/O
def _fits(m):
    try:
        host = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    except (ValueError, OSError):
        host = 0
    return m <= SMALL_SIZE or 4 * m < host


def _random01(rng, m):
    return np.unpackbits(np.frombuffer(rng.bytes((m + 7) // 8), dtype=np.uint8), count=m)


@pytest.mark.gpu
def test_f_set_get_roundtrip_every_size(pkg):
    rng = np.random.default_rng(31)
    done = []
    for m in SIZES:
        if not _fits(m):
            continue
        f = pkg.IndexRationalBloomFilter(m, 2.3)
        a = _random01(rng, m)
        if m <= 33:
            a[-1] = 1                                              # the last bit of a partial word
        f.bit_array = a
        b = f._dev.get_bits()
        for s in range(0, m, 1 << 28):                             # no 4 GiB temporary
            assert np.array_equal(a[s:s + (1 << 28)], b[s:s + (1 << 28)]), (m, s)
        done.append(m)
        del a, b, f
    assert max(done) > 2 ** 31, done


@pytest.mark.gpu
def test_f_setter_replaces_then_add_ors(pkg, co):
    m, k = 70_001, 2.3
    rng = np.random.default_rng(32)
    items = rng.integers(0, 10 ** 7, 5_000).astype(np.uint32)
    pattern = _random01(rng, m) & _random01(rng, m)                # about a quarter set
    f = pkg.IndexRationalBloomFilter(m, k)
    f.add_indices(items)
    assert f.bit_array.any()
    f.bit_array = pattern                                          # replaces, does not OR
    assert np.array_equal(f.bit_array, pattern)
    f.bit_array = np.zeros(m, dtype=np.uint8)
    assert not f.bit_array.any()
    f.bit_array = pattern
    f.add_indices(items)                                           # add after the setter ORs on top
    assert np.array_equal(f.bit_array, pattern | c_bits(co, m, k, IVC_SEEDS, items))
    for cls, arg in ((pkg.RationalBloomFilter, k), (pkg.StandardBloomFilter, 3)):
        g = cls(m, arg)
        g.add_many(["a", "b", "c"])
        g.bit_array = pattern.tolist()                             # the string classes keep a list (rbf:23)
        assert g.bit_array == pattern.tolist()
        g.add_many(strs(items))
        ref = c_bits(co, m, k, rbf_seeds(k), items) if cls is pkg.RationalBloomFilter else None
        if ref is not None:
            assert np.array_equal(np.array(g.bit_array, dtype=np.uint8), pattern | ref)
        else:
            assert set(np.flatnonzero(g.bit_array).tolist()) == set(np.flatnonzero(pattern).tolist()) | std_positions(co, m, 3, items)
    for bad in (np.zeros(m - 1, np.uint8), np.zeros(m + 1, np.uint8), np.zeros((1, m), np.uint8), []):
        with pytest.raises(ValueError):
            f.bit_array = bad
    assert np.array_equal(f.bit_array, pattern | c_bits(co, m, k, IVC_SEEDS, items))
    snap = f.bit_array
    assert not snap.flags.writeable
    with pytest.raises(ValueError):
        snap[0] = 1
    with pytest.raises(ValueError):
        f.bit_array[1] = 0


# ------------------------------------------------------------------ G. bit arrays holding bytes other than 0 and 1
@pytest.mark.gpu
def test_g_non01_bit_array_bytes_read_as_set(pkg, co):
    """The reference tests `bit_array[idx] == 0` (ivc:129,135; rbf:39,172,179): any non-zero byte is set.  get_bits
    afterwards returns 0/1 -- the device stores bits, not bytes."""
    m, k = 5_000, 2.6
    members = np.arange(0, 4_000, 9, dtype=np.uint32)
    bits = c_bits(co, m, k, IVC_SEEDS, members)
    odd = odd_bitmap(bits, 41)
    probes = np.arange(20_000, dtype=np.uint32)
    want = co.filter_check_strings(odd, k, IVC_SEEDS, strs(probes)).astype(bool)
    pyf = ro.RationalBloomFilter(m, k, IVC_SEEDS)
    pyf.bit_array = odd
    assert np.array_equal(want[:3_000], [pyf.check_index(int(i)) for i in probes[:3_000]])
    assert want[members].all() and not want.all()
    for bm in (odd, odd.astype(bool), odd.tolist()):
        f = pkg.IndexRationalBloomFilter(m, k)
        f.bit_array = bm
        assert np.array_equal(f.check_indices(probes), want)
        assert f.check_index(int(members[3])) and f.check_indices(np.array(["-4", "x"], dtype=object)).tolist() == \
            co.filter_check_strings(odd, k, IVC_SEEDS, ["-4", "x"]).astype(bool).tolist()
        assert np.array_equal(f.bit_array, bits)                   # read back as 0/1
    words = ["w%d" % i for i in range(500)]
    non = ["v%d" % i for i in range(10_000)]
    rb = c_bits(co, m, k, rbf_seeds(k), words)
    odd_r = odd_bitmap(rb, 42)
    g = pkg.RationalBloomFilter(m, k)
    g.bit_array = odd_r.tolist()
    assert np.array_equal(g.contains_many(words + non), co.filter_check_strings(odd_r, k, rbf_seeds(k), words + non).astype(bool))
    assert g.bit_array == rb.tolist()
    s = pkg.StandardBloomFilter(m, 3)
    sb = np.zeros(m, dtype=np.uint8)
    sb[sorted(std_positions(co, m, 3, words))] = 1
    odd_s = odd_bitmap(sb, 43)
    s.bit_array = odd_s
    res = s.contains_many(words + non)
    assert res[:len(words)].all() and np.array_equal(res, std_contains(co, odd_s, 3, words + non))
    assert not res.all()


@pytest.mark.gpu
def test_g_decompress_non01_bitmap(pkg, co):
    """BloomFilterCompressor.decompress assigns the caller's bitmap to the filter (ivc:290): bytes 2, 3, 128 and 255 are
    set bits, so the mask decodes as it does from the 0/1 bitmap."""
    rng = np.random.default_rng(51)
    for n, p, k, l in ((20_000, 0.05, 2.3, 3_000), (1_000, 0.1, 1.6, 150), (131_077, 0.02, 4.2, 9_001)):
        mask = (rng.random(n) < p).astype(np.uint8)
        bits, wit = co.compress_kl(mask, k, l)
        assert len(wit)
        odd = odd_bitmap(bits, n)
        want = co.decompress(odd, wit, n, k)
        assert np.array_equal(want, mask)
        for bm in (odd, odd.astype(bool)):
            out = pkg.BloomFilterCompressor().decompress(bm, list(wit), n, k)
            assert np.array_equal(out, want), (n, k, l)
        if n <= 1_000:
            assert np.array_equal(ro.decompress(odd, list(wit), n, k), want)
