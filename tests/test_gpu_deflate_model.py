"""The device zlib coder (csrc/rbf_deflate.cuh) byte for byte against tests/deflate_model.py, the pinned stream of its layout
comment: hash chains, the 16-candidate search, the greedy parse, the trees and run-length coded header, the dynamic / stored
decision, and the host batching of zlib_batch across waves of 2 x sm_count segments.

CPU tests: every model stream inflates to its input, and every constructed input reaches the case it was built for (the
assertions are on the model's facts, so a wrongly built input fails here, not silently on the GPU).
GPU tests: every stream of deflate.compress_many / FrameStream.zlib_changed / compress_video(entropy_coder="gpu") equals the
model's bytes (4K keyframes: equal to each buffer coded alone; see test_compress_video_keyframes)."""
import ctypes as C
import functools
import heapq
import struct
import zlib

import numpy as np
import pytest

from tests import deflate_model as M
from tests.util import synth_stream

SEG = M.SEG
FILL = 8                         # filler bytes 0..7; word bodies 0x10..0x6f; heads (unique per segment) 0x80..0xff
END_ORIG, END_COPY, END_THIRD, PRE, PRE2 = 0x78, 0x79, 0x7B, 0x7A, 0x7C


@pytest.fixture(scope="module")
def cabi():
    from new_bloom_filter_repo_b200 import build, _cabi
    build.build()
    return _cabi


@functools.lru_cache(maxsize=None)
def _hash_table():
    x = np.arange(1 << 24, dtype=np.uint32)
    return (x * np.uint32(M.HASH_MUL)) >> np.uint32(20)


def _colliding_triples(triple: bytes, n: int, rng):
    """n distinct 3-byte strings with bytes in 0x10..0x6f whose hash equals triple's."""
    h = M.hashes(np.frombuffer(triple, np.uint8))[0]
    x = np.nonzero(_hash_table() == h)[0]
    b = np.stack([x & 255, (x >> 8) & 255, x >> 16], axis=1)
    ok = ((b >= 0x10) & (b < 0x70)).all(axis=1)
    pick = rng.choice(np.nonzero(ok)[0], n, replace=False)
    return [bytes(b[k].astype(np.uint8)) for k in pick]


class _Seg:
    """One segment under construction: random filler with placed, protected words.  want: (pos, length, dist) tokens
    (dist 0: a literal); scrub() then rewrites filler until no unplanned position between a copy and its original shares
    the copy's hash."""

    def __init__(self, size, seed):
        self.rng = np.random.default_rng(seed)
        self.b = self.rng.integers(0, FILL, size, dtype=np.uint8)
        self.prot = np.zeros(size, bool)
        self.heads = iter(range(0x80, 0x100))
        self.want, self.clean = [], []

    def free(self, lo, hi):
        return lo >= 0 and hi <= self.b.size and not self.prot[lo:hi].any()

    def place(self, pos, data):
        data = np.frombuffer(bytes(data), np.uint8)
        assert self.free(pos, pos + data.size), (pos, data.size)
        self.b[pos:pos + data.size] = data
        self.prot[pos:pos + data.size] = True

    def word(self, n):
        return bytes([next(self.heads)]) + self.rng.integers(0x10, 0x70, n - 1, dtype=np.uint8).tobytes()

    def spans(self, o, dist, length):
        if dist >= length + 3:
            return [(o, o + length + 1), (o + dist - 2, o + dist + length + 1)]
        return [(o - 1, o + dist + length + 1)]

    def copy(self, o, dist, length, found=True, allowed=()):
        """A match of `length` at o + dist whose only candidate is o (periodic content when the two overlap)."""
        if dist >= length + 3:
            r = self.word(length)
            self.place(o, r + bytes([END_ORIG]))
            self.place(o + dist - 2, bytes([PRE, PRE]) + r + bytes([END_COPY]))
        else:
            w = self.word(dist)
            self.place(o - 1, bytes([PRE]) + (w * (length // dist + 2))[:dist + length] + bytes([END_COPY]))
        c = o + dist
        self.want.append((c, length if found else 0, dist if found else 0))
        self.clean.append((o, c, set(allowed)))
        return c

    def fit(self, dist, length, start=1, step=7):
        o = start
        while not all(self.free(lo, hi) for lo, hi in self.spans(o, dist, length)):
            o += step
            assert o + dist + length < self.b.size, "segment full"
        return self.copy(o, dist, length)

    def scrub(self):
        for _ in range(400):
            h = M.hashes(self.b)
            bad = []
            for o, c, allowed in self.clean:
                ps = o + 1 + np.nonzero(h[o + 1:c] == h[c])[0]
                bad += [p for p in ps.tolist() if p not in allowed and not self.prot[p:p + 3].all()]
            if not bad:
                return self
            for p in bad:
                q = [k for k in range(p, p + 3) if not self.prot[k]]
                k = q[int(self.rng.integers(len(q)))]
                self.b[k] = (int(self.b[k]) + 1 + int(self.rng.integers(FILL - 1))) % FILL
        raise AssertionError("scrub did not converge")

    def bytes(self):
        return self.scrub().b.tobytes()


def _tokens_ok(seg, want):
    mp = dict(zip(seg.match_pos.tolist(), zip(seg.match_len.tolist(), seg.match_dist.tolist())))
    lit = set(seg.lit_pos.tolist())
    for p, ln, d in want:
        if ln:
            assert mp.get(p) == (ln, d), ("match", p, ln, d, mp.get(p))
        else:
            assert p in lit, ("literal", p, mp.get(p))


def _same_hash_between(b, o, c):
    h = M.hashes(np.frombuffer(b, np.uint8))
    return int(np.count_nonzero(h[o + 1:c] == h[c]))


def _huffman_cost(freqs):
    """Total bits of an optimal Huffman code with no length limit (heapq)."""
    h = [int(f) for f in freqs if f]
    heapq.heapify(h)
    cost = 0
    while len(h) > 1:
        w = heapq.heappop(h) + heapq.heappop(h)
        cost += w
        heapq.heappush(h, w)
    return cost


def _zero_runs(lens):
    runs, r = [], 0
    for v in list(lens) + [1]:
        if v == 0:
            r += 1
        elif r:
            runs.append(r)
            r = 0
    return runs


LENS = sorted({x for s, b in enumerate(M.LEN_BASE) for x in (b, min(257 if s == 27 else 258, b + (1 << M.LEN_EXTRA[s]) - 1))})
DISTS = sorted({x for s, b in enumerate(M.DIST_BASE) for x in (b, b + (1 << M.DIST_EXTRA[s]) - 1)})


# ------------------------------------------------------------------ the inputs and the case each must reach
def _case_chain(n):
    s = _Seg(4000, 100 + n)
    t = s.word(8)
    o = 100
    s.place(o, t + bytes([END_ORIG]))
    pos = [200 + 40 * k for k in range(n)]
    for p, tri in zip(pos, _colliding_triples(t[:3], n, s.rng)):
        s.place(p, tri)
    c = 200 + 40 * n + 50
    s.place(c - 2, bytes([PRE, PRE]) + t + bytes([END_COPY]))
    s.want.append((c, 8, c - o) if n < M.DEPTH else (c, 0, 0))
    s.clean.append((o, c, set(pos)))
    b = s.bytes()

    def check(segs):
        assert _same_hash_between(b, o, c) == n          # the match is candidate n + 1
        _tokens_ok(segs[0], s.want)
    return b, check


def _case_window(dist):
    s = _Seg(40000, dist)
    c = s.copy(100, dist, 8, found=dist <= M.WINDOW)
    b = s.bytes()

    def check(segs):
        assert M.chains(np.frombuffer(b, np.uint8))[c] == (dist if dist <= M.WINDOW else 0)   # a direct link, or none
        _tokens_ok(segs[0], s.want)
    return b, check


def _seg_case(build, extra=None):
    def make():
        s = build()
        b = s.bytes()

        def check(segs):
            assert len(segs) == 1 and segs[0].dynamic
            _tokens_ok(segs[0], s.want)
            if extra:
                extra(s, segs[0])
        return b, check
    return make


def _in_warp():
    s = _Seg(SEG, 7)
    cur = 10
    for d in range(1, 32):
        for res in (31, 0):
            o = cur + (res - cur - d) % 32
            c = s.copy(o, d, d + 5)
            assert c % 32 == res
            cur = c + d + 40
    return s


def _ties():
    s = _Seg(SEG, 8)
    o = 64
    for ln in (3, 4, 5, 6, 7):                       # all three copies inside one 32-position step of the chain builder
        sp = ln + 3
        r = s.word(ln)
        s.place(o, r + bytes([END_ORIG]))
        s.place(o + sp - 2, bytes([PRE, PRE]) + r + bytes([END_THIRD]))
        s.place(o + 2 * sp - 2, bytes([PRE2, PRE2]) + r + bytes([END_COPY]))
        s.want += [(o + sp, ln, sp), (o + 2 * sp, ln, sp)]
        s.clean.append((o, o + 2 * sp, {o + sp}))
        o += 64
    for ln, sp in ((3, 1000), (10, 1000), (40, 5000), (200, 300)):
        o = o + 64
        r = s.word(ln)
        s.place(o, r + bytes([END_ORIG]))
        s.place(o + sp - 2, bytes([PRE, PRE]) + r + bytes([END_THIRD]))
        s.place(o + 2 * sp - 2, bytes([PRE2, PRE2]) + r + bytes([END_COPY]))
        s.want += [(o + sp, ln, sp), (o + 2 * sp, ln, sp)]
        s.clean.append((o, o + 2 * sp, {o + sp}))
        o += 2 * sp + ln
    # a 258 match at the first candidate with an equally long, farther copy behind it
    y = s.word(300)
    o = 20000
    s.place(o, y + bytes([END_ORIG]))
    s.place(o + 500 - 2, bytes([PRE, PRE]) + y + bytes([END_THIRD]))
    s.place(o + 1000 - 2, bytes([PRE2, PRE2]) + y + bytes([END_COPY]))
    s.want += [(o + 500, 258, 500), (o + 1000, 258, 500), (o + 1258, 42, 500)]
    s.clean.append((o, o + 1000, {o + 500}))
    return s


def _lengths():
    s = _Seg(SEG, 9)
    for k, ln in enumerate(LENS):
        s.fit(ln + 20 + k % 5, ln, start=1)
        s.fit(5 + k % 3, ln, start=30000)               # overlapping (periodic) copies
    return s


def _distances(part):
    s = _Seg(SEG, 10 + part)
    ds = [d for k, d in enumerate(DISTS) if k % 2 == part]
    for k, d in enumerate(sorted(ds, reverse=True)):
        s.fit(d, 3 + k % 9, start=1, step=5)
    return s


def _all_symbols():
    s = _Seg(SEG, 12)
    for d in sorted(M.DIST_BASE, reverse=True):
        s.fit(d, 6, start=1, step=5)
    for ln in M.LEN_BASE:
        s.fit(ln + 7, ln, start=1, step=5)
    perm = s.rng.permutation(256).astype(np.uint8).tobytes()
    o = 1
    while not s.free(o - 3, o + 259):
        o += 16
    s.place(o, perm)
    return s


def _all_symbols_check(s, seg):
    assert seg.hlit == 286 and seg.hdist == 30
    assert (seg.ll_hist > 0).all() and (seg.d_hist > 0).all()


def _chunk_edges():
    s = _Seg(SEG, 13)
    lens = (3, 4, 10, 100, 258, 257, 3, 258, 5, 64, 255, 3, 200, 7, 258)
    for k in range(1, 16):
        c = 4096 * k - 2 + (k % 2)
        ln = lens[k - 1]
        s.copy(c - 700, 700, ln)
    for k in range(8):                                   # matches ending on a 32-position word boundary
        ln = 5 + 11 * k
        c = 1024 * (k + 1) + 600
        c += (-(c + ln)) % 32
        while not all(s.free(lo, hi) for lo, hi in s.spans(c - 300, 300, ln)):
            c += 32
        s.copy(c - 300, 300, ln)
    return s


def _chunk_check(s, seg):
    for c, ln, d in s.want:
        if c % 4096 >= 4094:
            assert c // 4096 != (c + ln - 1) // 4096
    assert sum((c + ln) % 32 == 0 for c, ln, d in s.want) >= 8


def _back_to_back():
    rng = np.random.default_rng(14)
    blk = rng.integers(0x10, 0x70, 1500, dtype=np.uint8).tobytes()
    return (rng.integers(0, FILL, 300, dtype=np.uint8).tobytes() + blk * 40)[:SEG]


def _back_to_back_check(segs):
    s = segs[0]
    ends = s.match_pos + s.match_len
    chained = np.isin(ends[:-1], s.match_pos)
    crossing = (s.match_pos // 4096) != ((ends - 1) // 4096)
    assert chained.sum() > 100 and crossing.sum() >= 10 and (crossing[1:] & chained).sum() >= 10


def _tail(L, last_lits):
    s = _Seg(L, 15 + L)
    r = s.word(300)
    o = max(100, L - 20000)
    s.place(o, r + bytes([END_ORIG]))
    if last_lits:
        c = L - 52
        s.place(c - 2, bytes([PRE, PRE]) + r[:50] + bytes([END_COPY, r[0]]))
        s.want += [(c, 50, c - o), (L - 2, 0, 0), (L - 1, 0, 0)]
    else:
        c = L - 100                                      # maxlen = 100 < 258
        s.place(c - 2, bytes([PRE, PRE]) + r[:100])
        s.want.append((c, 100, c - o))
    s.clean.append((o, c, set()))
    return s


def _across_segments():
    first = _tail(SEG, False).bytes()
    return first + first[-3000:] + first[:3000]


def _across_check(segs):
    data = _across_segments()
    assert len(segs) == 2 and segs[0].dynamic and segs[1].dynamic
    assert data[SEG:SEG + 3000] == data[SEG - 3000:SEG]     # reaching back 3000 bytes would find a 258 match at once
    s = segs[1]
    assert s.match_pos.size > 100 and (s.match_pos >= s.match_dist).all()   # matches, none before the segment start
    assert {0, 1, 2} <= set(s.lit_pos.tolist())


def _de_bruijn(k, n):
    a, seq = [0] * k * n, []

    def db(t, p):
        if t > n:
            if n % p == 0:
                seq.extend(a[1:p + 1])
        else:
            a[t] = a[t - p]
            db(t + 1, p)
            for j in range(a[t - p] + 1, k):
                a[t] = j
                db(t + 1, t)
    db(1, 1)
    return seq


def _fib_bytes():
    """A counter 0..16383 written as (k >> 7, k & 127) byte pairs: 128 byte values, 256 times each, and almost no repeated
    3-byte string, so nearly every byte is a literal.  Between pairs go 13 more byte values (128..) with counts 1, 2, 3, 5,
    ..., 377; with the end-of-block code as the other 1 they form a Fibonacci chain below the counter bytes, so the
    optimal tree is deeper than 15 and the limit must bind."""
    fib = [1, 2]
    while len(fib) < 13:
        fib.append(fib[-1] + fib[-2])
    k = np.arange(16384)
    pairs = np.stack([k >> 7, k & 127], axis=1).astype(np.uint8).reshape(-1)
    rng = np.random.default_rng(1)
    g = rng.permutation(np.repeat(np.arange(128, 128 + len(fib)), fib)).astype(np.uint8)
    slots = np.sort(rng.choice(16383, g.size, replace=False)) + 1          # one insertion per gap between pairs
    parts = np.split(pairs, 2 * slots)
    return b"".join(p.tobytes() + (bytes([x]) if i < g.size else b"") for i, (p, x) in enumerate(zip(parts, list(g) + [0])))


def _present(values, n, seed, weights=None):
    rng = np.random.default_rng(seed)
    v = np.array(values, np.uint8)
    p = None if weights is None else np.array(weights, float) / np.sum(weights)
    return rng.choice(v, n, p=p).tobytes()


def _zero_runs_input(gaps, seed):
    vals, x = [0], 0
    for g in gaps:
        x += g + 1
        vals.append(x)
    return _present(vals, 6000, seed), gaps


def _repeats_input():
    # blocks of consecutive byte values with one frequency per block: equal code lengths inside a block
    vals, w, x = [], [], 0
    for k, size in enumerate((4, 5, 7, 8, 10, 11)):
        vals += list(range(x, x + size))
        w += [2 ** k] * size
        x += size + 2
    return _present(vals, 20000, 17, w)


def _size_search(target_excess, L, seed0):
    """Seed search: uniform random bytes over 233..237 values sit near the dynamic / stored break-even; find dyn_bytes - bound
    == excess."""
    for seed in range(seed0, seed0 + 400):
        b = np.random.default_rng(seed).integers(0, 233 + seed % 5, L, dtype=np.uint8)
        s = M.segment(b.tobytes())
        if s.dyn_bytes - s.bound == target_excess:
            return b.tobytes()
    return None


@functools.lru_cache(maxsize=None)
def cases():
    cs = {}
    for n in (14, 15, 16):
        cs["chain_%d_colliding" % n] = _case_chain(n)
    for d in (32767, 32768, 32769):
        cs["window_%d" % d] = _case_window(d)
    cs["in_warp_distances"] = _seg_case(_in_warp)()
    cs["ties_nearest"] = _seg_case(_ties)()
    cs["every_length"] = _seg_case(_lengths)()
    cs["every_distance_a"] = _seg_case(lambda: _distances(0))()
    cs["every_distance_b"] = _seg_case(lambda: _distances(1))()
    cs["all_286_and_30"] = _seg_case(_all_symbols, _all_symbols_check)()
    cs["chunk_edges"] = _seg_case(_chunk_edges, _chunk_check)()
    cs["back_to_back"] = (_back_to_back(), _back_to_back_check)
    for L, lits in ((5000, False), (5000, True), (SEG, False), (SEG, True), (4099, True)):
        cs["tail_%d_%s" % (L, "lits" if lits else "match")] = _seg_case(functools.partial(_tail, L, lits))()
    cs["across_segments"] = (_across_segments(), _across_check)
    rng = np.random.default_rng(18)
    low = lambda n: rng.integers(0, 12, n, dtype=np.uint8).tobytes()          # noqa: E731
    for n in [1, 2, 3, 4, 65535, 65536, 65537, 2 * SEG - 1, 2 * SEG + 1] + [4096 * k + e for k in range(1, 17) for e in (-1, 1)]:
        cs["len_%d" % n] = (low(n), None)
    for n in (1, 3, 100, 65535, 65536, 65537):
        cs["random_%d" % n] = (rng.integers(0, 256, n, dtype=np.uint8).tobytes(), None)
    cs["empty"] = (b"", None)
    cs["single_literal"] = (b"A" * 3000, None)
    cs["no_match"] = (bytes(0x30 + x for x in _de_bruijn(16, 3)), None)
    cs["fibonacci"] = (_fib_bytes(), None)
    cs["zero_runs_3_10_11_138"] = _zero_runs_input((3, 10, 11, 138), 19)
    cs["zero_runs_139"] = _zero_runs_input((139,), 20)
    cs["zero_runs_149"] = _zero_runs_input((149,), 21)
    cs["nonzero_repeats"] = (_repeats_input(), None)
    mix = b"".join(low(SEG) if k % 2 else rng.integers(0, 256, SEG, dtype=np.uint8).tobytes() for k in range(5))
    cs["mixture"] = (mix + low(1000), None)
    return cs


def _check_case(name):
    data, check = cases()[name]
    z, segs = M.compress(data)
    d = zlib.decompressobj()
    assert d.decompress(z) + d.flush() == data and d.eof and d.unused_data == b""
    from new_bloom_filter_repo_b200 import _cabi
    assert len(z) <= _cabi.zlib_bound(len(data))
    if callable(check):
        check(segs)
    return z, segs


CASE_NAMES = ["chain_14_colliding", "chain_15_colliding", "chain_16_colliding", "window_32767", "window_32768", "window_32769",
              "in_warp_distances", "ties_nearest", "every_length", "every_distance_a", "every_distance_b", "all_286_and_30",
              "chunk_edges", "back_to_back", "tail_5000_match", "tail_5000_lits", "tail_65536_match", "tail_65536_lits",
              "tail_4099_lits", "across_segments", "empty", "single_literal", "no_match", "fibonacci", "zero_runs_3_10_11_138",
              "zero_runs_139", "zero_runs_149", "nonzero_repeats", "mixture"]


@pytest.mark.parametrize("name", CASE_NAMES)
def test_model_stream_inflates_and_reaches_its_case(cabi, name):
    _check_case(name)


def test_model_lengths_and_random_inputs_inflate(cabi):
    for name in cases():
        if name.startswith(("len_", "random_")):
            z, segs = _check_case(name)
            if name.startswith("random_") and len(cases()[name][0]) > 100:
                assert not any(s.dynamic for s in segs)


def test_model_empty_stream(cabi):
    assert M.compress(b"")[0] == bytes.fromhex("789c030000000001")


def test_every_length_and_distance_symbol_at_both_ends(cabi):
    got_l, got_d = set(), set()
    for name in ("every_length", "every_distance_a", "every_distance_b"):
        for s in M.compress(cases()[name][0])[1]:
            got_l |= set(s.match_len.tolist())
            got_d |= set(s.match_dist.tolist())
    assert set(LENS) <= got_l and set(DISTS) <= got_d
    assert len(LENS) == 8 + 2 * 20 + 1 and len(DISTS) == 4 + 2 * 26       # 3..10, 258 and distances 1..4 have one value


def test_trees_and_header_cases(cabi):
    segs = {k: M.compress(cases()[k][0])[1] for k in ("single_literal", "no_match", "fibonacci", "zero_runs_3_10_11_138",
                                                      "zero_runs_139", "zero_runs_149", "nonzero_repeats")}
    sl, nm = segs["single_literal"][0], segs["no_match"][0]
    assert sl.dynamic and np.count_nonzero(sl.d_hist) == 1 and np.count_nonzero(sl.d_len) == 2       # one distance + the added code
    assert nm.dynamic and nm.d_hist.sum() == 0 and list(nm.d_len[:2]) == [1, 1] and nm.hdist == 2
    fb = segs["fibonacci"][0]
    assert fb.dynamic and fb.ll_len.max() == 15 and fb.hclen == 19                         # the 15-bit limit binds:
    assert int((fb.ll_hist * fb.ll_len).sum()) > _huffman_cost(fb.ll_hist)                  # the optimum is out of reach
    runs = set()
    rle = set()
    for k in ("zero_runs_3_10_11_138", "zero_runs_139", "zero_runs_149", "nonzero_repeats"):
        s = segs[k][0]
        assert s.dynamic
        runs |= set(_zero_runs(list(s.ll_len[:s.hlit]) + list(s.d_len[:s.hdist])))
        rle |= set(zip(s.rle_sym, s.rle_ext))
    assert {3, 10, 11, 138, 139, 149} <= runs
    assert {(16, 0), (16, 3), (17, 0), (17, 7), (18, 0), (18, 127)} <= rle, sorted(x for x in rle if x[0] >= 16)
    assert any(s.hclen < 19 for v in segs.values() for s in v)


def test_size_decision_cases(cabi):
    mixed = M.compress(cases()["mixture"][0])[1]
    assert [s.dynamic for s in mixed] == [False, True, False, True, False, True]
    tie = M.compress(_tie_input(0))[1][0]
    over = M.compress(_tie_input(1))[1][0]
    assert tie.dyn_bytes == tie.bound and tie.dynamic
    assert over.dyn_bytes == over.bound + 1 and not over.dynamic


@functools.lru_cache(maxsize=None)
def _tie_input(excess):
    b = _size_search(excess, 3000, 1000 * (excess + 1))
    assert b is not None, "no seed with dyn_bytes - bound == %d" % excess
    return b


# ------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def pkg():
    import new_bloom_filter_repo_b200 as p
    assert p._cabi.device_info()["cc"] == (9, 0)
    return p


def _assert_model(got: bytes, data, what=""):
    want, segs = M.compress(data)
    if got != want:
        pytest.fail("%s: %s" % (what, M.first_difference(got, want, segs)))


def _batch(pkg, bufs, capacity=None, guard=0):
    """rbf_zlib_compress_batch with an explicit capacity; -> (rc, out array incl. guard bytes, offsets)."""
    _cabi = pkg._cabi
    views = [np.frombuffer(b, np.uint8) if len(b) else np.zeros(0, np.uint8) for b in bufs]
    n = len(views)
    lens = np.array([v.size for v in views], np.uint64)
    srcs = (C.c_void_p * n)(*[v.ctypes.data if v.size else None for v in views])
    cap = sum(_cabi.zlib_bound(int(x)) for x in lens) if capacity is None else capacity
    out = np.full(cap + guard, 0xA5, np.uint8)
    offs = np.zeros(n + 1, np.uint64)
    rc = _cabi.lib().rbf_zlib_compress_batch(_cabi.ctx(), n, srcs, _cabi.ptr(lens), 0, _cabi.ptr(out), cap, _cabi.ptr(offs))
    return rc, out, offs


@pytest.mark.gpu
def test_streams_equal_model(pkg):
    names = list(cases())
    datas = [cases()[k][0] for k in names] + [_tie_input(0), _tie_input(1)]
    names += ["dyn_equals_bound", "dyn_one_over_bound"]
    zs = pkg.deflate.compress_many(datas)
    for k, d, z in zip(names, datas, zs):
        _assert_model(z, d, k)


def _wave_segments(seed):
    """Seven distinct 64 KiB segments (low-entropy, text-like, random, runs): a cycle of them never lines up with a wave."""
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 6, SEG, dtype=np.uint8).tobytes(),
            (b"segment %d of the wave test " % seed * 3000)[:SEG],
            rng.integers(0, 256, SEG, dtype=np.uint8).tobytes(),
            np.repeat(rng.integers(0, 256, SEG // 64, dtype=np.uint8), 64).tobytes(),
            rng.integers(0, 40, SEG, dtype=np.uint8).tobytes(),
            np.resize(rng.integers(0, 256, 977, dtype=np.uint8), SEG).tobytes(),
            rng.integers(100, 104, SEG, dtype=np.uint8).tobytes()]


def _cycle(n_bytes, k0, seed=0):
    segs = _wave_segments(seed)
    return b"".join(segs[(k0 + k) % 7] for k in range((n_bytes + SEG - 1) // SEG))[:n_bytes]


@pytest.mark.gpu
def test_one_buffer_across_two_wave_boundaries(pkg):
    W = 2 * pkg._cabi.device_info()["sm_count"]
    data = _cycle((2 * W + 3) * SEG + 5, 0)
    z = pkg.deflate.compress(data)
    _assert_model(z, data, "%d segments" % (2 * W + 4))
    assert zlib.decompress(z) == data


def _wave_batch(W):
    """> 2W streams: a wave boundary inside a multi-segment stream (W), between streams and on an empty stream (2W)."""
    singles = [b"\x07", _cycle(65535, 1), _cycle(SEG, 2), b"", _cycle(777, 3), _cycle(SEG, 4)]
    bufs = [singles[k % 6] if k % 6 != 4 else _cycle(100 + k, k) for k in range(W - 1)]
    bufs.append(_cycle(2 * SEG + 1, 5))                             # segments W-1, W, W+1
    bufs += [singles[k % 6] for k in range(W - 2)]                  # through segment 2W - 1
    bufs.append(b"")                                                # segment 2W: the first of the third wave
    bufs += [_cycle(SEG + 1, 6), b"", b"\x00", _cycle(5 * SEG - 3, 0), _cycle(65537, 2)] + [singles[k % 6] for k in range(20)]
    nseg = [max(1, -(-len(b) // SEG)) for b in bufs]
    first = np.cumsum([0] + nseg[:-1])
    assert len(bufs) > 2 * W
    assert first[W - 1] == W - 1 and nseg[W - 1] == 3                # W falls inside that stream
    assert first[2 * W - 2] == 2 * W and bufs[2 * W - 2] == b""      # 2W falls between streams, on an empty one
    return bufs


@pytest.mark.gpu
def test_batch_across_waves(pkg):
    W = 2 * pkg._cabi.device_info()["sm_count"]
    bufs = _wave_batch(W)
    rc, out, offs = _batch(pkg, bufs)
    pkg._cabi.check(rc, pkg._cabi.ctx())
    pos = 0
    alone = {}
    for i, b in enumerate(bufs):
        want, segs = M.compress(b)
        assert int(offs[i]) == pos, (i, int(offs[i]), pos)            # contiguous
        got = out[pos:pos + len(want)].tobytes()
        if got != want:
            pytest.fail("stream %d (%d bytes): %s" % (i, len(b), M.first_difference(got, want, segs)))
        pos += len(want)
        if b not in alone:
            alone[b] = pkg.deflate.compress(b)
        assert alone[b] == want
    assert int(offs[len(bufs)]) == pos


@pytest.mark.gpu
def test_output_capacity_exact_and_one_short(pkg):
    W = 2 * pkg._cabi.device_info()["sm_count"]
    bufs = _wave_batch(W)
    need = sum(len(M.compress(b)[0]) for b in bufs)
    rc, out, offs = _batch(pkg, bufs, capacity=need, guard=64)
    pkg._cabi.check(rc, pkg._cabi.ctx())
    assert int(offs[-1]) == need and (out[need:] == 0xA5).all()
    assert out[:need].tobytes() == b"".join(M.compress(b)[0] for b in bufs)
    rc, out, offs = _batch(pkg, bufs, capacity=need - 1, guard=64)
    assert rc != 0
    assert (out[need - 1:] == 0xA5).all()                          # nothing written at or past the capacity


def _changed_stream(pkg, h, w, ch, dtype, frames, mask_mode=1):
    st = pkg.FrameStream(h, w, ch, dtype, max_frames=len(frames), mask_mode=mask_mode)
    st.upload(frames if ch > 1 else frames[..., 0].copy())
    st.encode_consecutive(len(frames), 0.0)
    return st


@pytest.mark.gpu
@pytest.mark.parametrize("ch,dtype", [(1, np.uint8), (3, np.uint8), (3, np.uint16)])
def test_zlib_changed_unaligned_sources(pkg, ch, dtype):
    fr = synth_stream(67, 131, 7, 40 + ch, [0.013, 0.2, 0.0007, 0.05, 0.31, 0.003], dtype=dtype)
    st = _changed_stream(pkg, 67, 131, ch, dtype, fr)
    try:
        voff = st.changed_offsets()
        assert any(int(v) % 16 for v in voff[1:-1])                    # later pairs start off a 16 B boundary
        gathered = st.gather_changed()
        zs = st.zlib_changed()
        for j, (g, z) in enumerate(zip(gathered, zs)):
            _assert_model(z, g.tobytes(), "pair %d" % j)
            assert zlib.decompress(z) == g.tobytes()
    finally:
        st.close()


@pytest.mark.gpu
def test_zlib_changed_4k_group_crosses_waves(pkg):
    W = 2 * pkg._cabi.device_info()["sm_count"]
    fr = synth_stream(2160, 3840, 30, 50, [0.05])
    st = _changed_stream(pkg, 2160, 3840, 3, np.uint8, fr, mask_mode=0)
    try:
        voff = st.changed_offsets()
        nseg = sum(-(-int(voff[i + 1] - voff[i]) // SEG) for i in range(29))
        assert nseg > W
        gathered = st.gather_changed()
        zs = st.zlib_changed()
        for j, (g, z) in enumerate(zip(gathered, zs)):
            _assert_model(z, g.tobytes(), "pair %d" % j)
    finally:
        st.close()


def _keyframe_blobs(payload):
    h, w, isz = struct.unpack_from("<III", payload, 0)
    pos = 12
    (n,) = struct.unpack_from("<I", payload, pos)
    blobs = [payload[pos + 4:pos + 4 + n]]
    pos += 4 + n
    if payload[pos]:
        (fl,) = struct.unpack_from("<H", payload, pos + 1)
        pos += 3 + fl
        for _ in range(3):
            (n,) = struct.unpack_from("<I", payload, pos)
            blobs.append(payload[pos + 4:pos + 4 + n])
            pos += 4 + n + 8
    return blobs


@pytest.mark.gpu
@pytest.mark.parametrize("hw", [(1080, 1920), (2160, 3840)])
def test_compress_video_keyframes(pkg, hw):
    """1080p: every keyframe blob equals the model.  4K (about 760 segments per keyframe): each blob equals its buffer coded
    alone, which the wave tests above tie to the model."""
    frames = [f for f in synth_stream(hw[0], hw[1], 3, 60, [0.05, 0.5])]
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=2)
    comp.entropy_coder = "gpu"
    comp.compress_video(frames, input_color_space="YUV")
    payloads = list(comp._last_compressed_frames)
    for fi in (0, 2):
        raws = pkg.fixed_video_compressor.keyframe_raws(frames[fi])
        blobs = _keyframe_blobs(payloads[fi])
        assert len(blobs) == len(raws) == 4
        for r, z in zip(raws, blobs):
            if hw[0] <= 1080:
                _assert_model(z, r, "keyframe %d" % fi)
            else:
                assert z == pkg.deflate.compress(r)
            assert zlib.decompress(z) == r
    dec = comp.decompress_video(compressed_frames=payloads)
    assert comp.verify_lossless(frames, dec)["lossless"]
