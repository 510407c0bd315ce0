"""A plain numpy/Python model of the device zlib coder's pinned stream (csrc/rbf_deflate.cuh, file header).

compress(data) -> (stream, segments): the exact bytes the layout comment describes, and per 64 KiB segment the facts the
tests assert on (tokens, code lengths, the run-length coded header, hlit / hdist / hclen, dynamic or stored, dyn_bytes).
Nothing here comes from the kernels except the host build of the length-limited code builder
(_cabi.deflate_code_lengths), which tests/test_gpu_deflate.py checks against an unconstrained Huffman code.
"""
from __future__ import annotations

import functools
import zlib
from dataclasses import dataclass, field

import numpy as np

SEG = 65536
WINDOW = 32768
DEPTH = 16
MAX_MATCH = 258
HASH_MUL = 2654435761
CL_ORDER = (16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)

# RFC 1951 3.2.5
LEN_BASE = (3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258)
LEN_EXTRA = (0,) * 8 + (1,) * 4 + (2,) * 4 + (3,) * 4 + (4,) * 4 + (5,) * 4 + (0,)
DIST_BASE = (1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577)
DIST_EXTRA = (0, 0, 0, 0) + tuple(e for e in range(1, 14) for _ in (0, 1))

_LEN_SYM = np.zeros(MAX_MATCH + 1, np.int64)
for _s, _b in enumerate(LEN_BASE):
    _LEN_SYM[_b:] = 257 + _s
_DIST_SYM = np.zeros(WINDOW + 1, np.int64)
for _s, _b in enumerate(DIST_BASE):
    _DIST_SYM[_b:] = _s
_LL_EXTRA = np.zeros(286, np.int64)
_LL_EXTRA[257:] = LEN_EXTRA
_LL_BASE = np.zeros(286, np.int64)
_LL_BASE[257:] = LEN_BASE
_D_EXTRA = np.array(DIST_EXTRA, np.int64)
_D_BASE = np.array(DIST_BASE, np.int64)


def len_sym(n):
    return _LEN_SYM[n]


def dist_sym(d):
    return _DIST_SYM[d]


def seg_bound(n: int) -> int:
    """Stored blocks (one, two at 65536 bytes) plus the sync flush: the most a segment of n bytes may take."""
    return 0 if n == 0 else n + 5 * (2 if n > 65535 else 1) + 5


def hashes(b: np.ndarray) -> np.ndarray:
    """12-bit hash of the 3-byte prefix at every position i with i + 2 < len(b)."""
    if b.size < 3:
        return np.zeros(0, np.int64)
    x = b[:-2].astype(np.uint64) | (b[1:-1].astype(np.uint64) << 8) | (b[2:].astype(np.uint64) << 16)
    return (((x * HASH_MUL) & 0xFFFFFFFF) >> 20).astype(np.int64)


def chains(b: np.ndarray) -> np.ndarray:
    """prev[i]: distance to the nearest earlier position with the same hash, 0 if none within WINDOW."""
    prev = np.zeros(b.size, np.int64)
    h = hashes(b)
    if h.size < 2:
        return prev
    order = np.argsort(h, kind="stable")
    d = order[1:] - order[:-1]
    prev[order[1:]] = np.where((h[order[1:]] == h[order[:-1]]) & (d <= WINDOW), d, 0)
    return prev


def _words(b: np.ndarray) -> np.ndarray:
    """w[p]: the 8 bytes at p as a little-endian uint64 (zero past the end)."""
    pad = np.concatenate([b, np.zeros(MAX_MATCH + 16, np.uint8)])
    return np.lib.stride_tricks.sliding_window_view(pad, 8).copy().view("<u8").reshape(-1)


def _lcp(w: np.ndarray, i: np.ndarray, j: np.ndarray, cap: np.ndarray) -> np.ndarray:
    n = np.zeros(i.size, np.int64)
    act = np.arange(i.size)
    while act.size:
        x = w[i[act] + n[act]] ^ w[j[act] + n[act]]
        done = x != 0
        low = x[done] & (~x[done] + np.uint64(1))
        n[act[done]] += np.log2(low.astype(np.float64)).astype(np.int64) >> 3
        go = act[~done]
        n[go] += 8
        act = go[n[go] < cap[go]]
    return np.minimum(n, cap)


def search(b: np.ndarray, prev: np.ndarray):
    """Longest match (>= 3) among the first DEPTH chain candidates within WINDOW, nearest on ties: (length, distance)."""
    L = b.size
    maxlen = np.minimum(L - np.arange(L), MAX_MATCH)
    blen = np.zeros(L, np.int64)
    bdist = np.zeros(L, np.int64)
    w = _words(b)
    idx = np.nonzero((prev != 0) & (maxlen >= 3))[0]
    cum = prev[idx].copy()
    for _ in range(DEPTH):
        live = (cum <= WINDOW) & (cum != 0) & (blen[idx] < maxlen[idx])
        idx, cum = idx[live], cum[live]
        if idx.size == 0:
            break
        j = idx - cum
        ln = _lcp(w, idx, j, maxlen[idx])
        better = (ln >= 3) & (ln > blen[idx])
        blen[idx[better]] = ln[better]
        bdist[idx[better]] = cum[better]
        d = prev[j]
        cum = np.where(d != 0, cum + d, 0)
    return blen, bdist


def parse(blen: np.ndarray):
    """Greedy parse: a match where the search found one, else a literal.  -> match starts, literal positions."""
    cand = np.nonzero(blen)[0]
    starts = []
    pos, L = 0, blen.size
    while True:
        k = int(np.searchsorted(cand, pos))                  # the next position at or after pos with a match
        if k >= cand.size:
            break
        c = int(cand[k])
        starts.append(c)
        pos = c + int(blen[c])
    ms = np.array(starts, np.int64)
    cover = np.zeros(L + 1, np.int64)
    np.add.at(cover, ms, 1)
    np.add.at(cover, ms + blen[ms], -1)
    lit = np.nonzero(np.cumsum(cover[:L]) == 0)[0]
    return ms, lit


def canonical(lengths) -> np.ndarray:
    """Canonical codes, bit-reversed for deflate's LSB-first order."""
    lengths = [int(x) for x in lengths]
    count = [0] * 16
    for n in lengths:
        if n:
            count[n] += 1
    nxt, code = [0] * 16, 0
    for n in range(1, 16):
        code = (code + count[n - 1]) << 1
        nxt[n] = code
    out = np.zeros(len(lengths), np.int64)
    for s, n in enumerate(lengths):
        if n:
            c = nxt[n]
            nxt[n] += 1
            out[s] = int(format(c, "0%db" % n)[::-1], 2)
    return out


def rle_lengths(lens):
    """Run-length code of the code lengths: 18 for zero runs 11..138, 17 for 3..10, 16 for 3..6 repeats of the last."""
    syms, ext = [], []
    i, n = 0, len(lens)
    while i < n:
        v = lens[i]
        run = 1
        while i + run < n and lens[i + run] == v:
            run += 1
        i += run
        if v == 0:
            while run >= 11:
                r = min(run, 138)
                syms.append(18); ext.append(r - 11); run -= r
            if run >= 3:
                syms.append(17); ext.append(run - 3); run = 0
        else:
            syms.append(v); ext.append(0); run -= 1
            while run >= 3:
                r = min(run, 6)
                syms.append(16); ext.append(r - 3); run -= r
        syms += [v] * run
        ext += [0] * run
    return syms, ext


def _pack(vals, nbits) -> bytes:
    """Concatenate fields LSB first; pad the last byte with zeros."""
    vals = np.asarray(vals, np.int64)
    nbits = np.asarray(nbits, np.int64)
    keep = nbits > 0
    vals, nbits = vals[keep], nbits[keep]
    total = int(nbits.sum())
    fi = np.repeat(np.arange(vals.size), nbits)
    off = np.arange(total) - np.repeat(np.cumsum(nbits) - nbits, nbits)
    bits = ((vals[fi] >> off) & 1).astype(np.uint8)
    return np.packbits(bits, bitorder="little").tobytes()


def _stored(b: bytes) -> bytes:
    out = []
    for k in range(0, max(len(b), 1), 65535):
        part = b[k:k + 65535]
        n = len(part)
        out.append(bytes([0, n & 255, n >> 8, ~n & 255, (~n >> 8) & 255]) + part)
    return b"".join(out) + b"\x00\x00\x00\xff\xff"


@dataclass
class Segment:
    length: int
    dynamic: bool
    dyn_bytes: int
    bound: int
    match_pos: np.ndarray
    match_len: np.ndarray
    match_dist: np.ndarray
    lit_pos: np.ndarray
    ll_hist: np.ndarray
    d_hist: np.ndarray
    ll_len: np.ndarray
    d_len: np.ndarray
    cl_len: np.ndarray
    rle_sym: list
    rle_ext: list
    hlit: int
    hdist: int
    hclen: int
    hdr_bits: int
    body_bits: int
    out: bytes
    token_pos: np.ndarray = field(default=None)      # every token start, in order
    token_bit: np.ndarray = field(default=None)      # bit offset of each token in `out` (dynamic blocks)

    def token_at_byte(self, byte: int) -> str:
        """The token whose code covers byte `byte` of this segment's output, for mismatch reports."""
        if not self.dynamic:
            return "stored block byte %d" % byte
        k = int(np.searchsorted(self.token_bit, 8 * byte, side="right")) - 1
        if k < 0:
            return "header (hlit %d hdist %d hclen %d)" % (self.hlit, self.hdist, self.hclen)
        p = int(self.token_pos[k])
        m = int(np.searchsorted(self.match_pos, p))
        if m < self.match_pos.size and self.match_pos[m] == p:
            return "match at %d: length %d distance %d" % (p, self.match_len[m], self.match_dist[m])
        return "literal at %d" % p


def _code_lengths(freqs, max_bits):
    from new_bloom_filter_repo_b200 import _cabi
    return _cabi.deflate_code_lengths(np.asarray(freqs, np.uint32), max_bits).astype(np.int64)


@functools.lru_cache(maxsize=32)             # a few segments recur (the wave tests cycle through seven)
def segment(data: bytes) -> Segment:
    """Code one segment (1..65536 bytes)."""
    b = np.frombuffer(data, np.uint8)
    L = b.size
    assert 0 < L <= SEG
    blen, bdist = search(b, chains(b))
    ms, lit = parse(blen)
    ml, md = blen[ms], bdist[ms]
    ll_hist = np.bincount(b[lit], minlength=286) + np.bincount(_LEN_SYM[ml], minlength=286)
    ll_hist[256] += 1
    d_hist = np.bincount(_DIST_SYM[md], minlength=30)
    ll_len = _code_lengths(ll_hist, 15)
    d_len = _code_lengths(d_hist, 15)
    hlit = 286
    while hlit > 257 and ll_len[hlit - 1] == 0:
        hlit -= 1
    hdist = 30
    while hdist > 1 and d_len[hdist - 1] == 0:
        hdist -= 1
    syms, ext = rle_lengths([int(x) for x in ll_len[:hlit]] + [int(x) for x in d_len[:hdist]])
    cl_len = _code_lengths(np.bincount(syms, minlength=19), 7)
    hclen = 19
    while hclen > 4 and cl_len[CL_ORDER[hclen - 1]] == 0:
        hclen -= 1
    xbits = {16: 2, 17: 3, 18: 7}
    hdr = 3 + 5 + 5 + 4 + 3 * hclen + sum(int(cl_len[s]) + xbits.get(s, 0) for s in syms)
    body = int((ll_hist * (ll_len + _LL_EXTRA)).sum() + (d_hist * (d_len + _D_EXTRA)).sum())
    dyn_bytes = (hdr + body + 3 + 7) // 8 + 4
    bound = seg_bound(L)
    dynamic = dyn_bytes <= bound and dyn_bytes <= SEG
    tok = np.sort(np.concatenate([ms, lit]))
    seg = Segment(L, dynamic, dyn_bytes, bound, ms, ml, md, lit, ll_hist, d_hist, ll_len, d_len, cl_len, syms, ext,
                  hlit, hdist, hclen, hdr, body, b"", tok)
    if not dynamic:
        seg.out = _stored(data)
        return seg
    llc, dc, clc = canonical(ll_len), canonical(d_len), canonical(cl_len)
    hv = [4, hlit - 257, hdist - 1, hclen - 4] + [int(cl_len[CL_ORDER[k]]) for k in range(hclen)]
    hn = [3, 5, 5, 4] + [3] * hclen
    for s, e in zip(syms, ext):
        hv += [int(clc[s]), e]
        hn += [int(cl_len[s]), xbits.get(s, 0)]
    # tokens: four fields each (literals use the first only)
    f_val = np.zeros((tok.size, 4), np.int64)
    f_len = np.zeros((tok.size, 4), np.int64)
    is_m = np.zeros(L, bool)
    is_m[ms] = True
    mi = np.zeros(L, np.int64)
    mi[ms] = np.arange(ms.size)
    lt = tok[~is_m[tok]]
    lrow = np.nonzero(~is_m[tok])[0]
    f_val[lrow, 0] = llc[b[lt]]
    f_len[lrow, 0] = ll_len[b[lt]]
    mrow = np.nonzero(is_m[tok])[0]
    k = mi[tok[mrow]]
    ls, ds = _LEN_SYM[ml[k]], _DIST_SYM[md[k]]
    f_val[mrow, 0], f_len[mrow, 0] = llc[ls], ll_len[ls]
    f_val[mrow, 1], f_len[mrow, 1] = ml[k] - _LL_BASE[ls], _LL_EXTRA[ls]
    f_val[mrow, 2], f_len[mrow, 2] = dc[ds], d_len[ds]
    f_val[mrow, 3], f_len[mrow, 3] = md[k] - _D_BASE[ds], _D_EXTRA[ds]
    tbits = f_len.sum(axis=1)
    seg.token_bit = hdr + np.cumsum(tbits) - tbits
    vals = np.concatenate([np.array(hv, np.int64), f_val.reshape(-1), [llc[256], 0]])
    lens = np.concatenate([np.array(hn, np.int64), f_len.reshape(-1), [ll_len[256], 3]])
    assert int(lens.sum()) == hdr + body + 3
    seg.out = _pack(vals, lens) + b"\x00\x00\xff\xff"
    assert len(seg.out) == dyn_bytes
    return seg


def compress(data):
    """-> (zlib stream, [Segment]) of the device coder's layout for `data` (bytes-like)."""
    data = bytes(memoryview(data).cast("B"))
    segs = [segment(data[k:k + SEG]) for k in range(0, len(data), SEG)]
    adler = zlib.adler32(data)
    return b"\x78\x9c" + b"".join(s.out for s in segs) + b"\x03\x00" + adler.to_bytes(4, "big"), segs


def first_difference(got: bytes, want: bytes, segs) -> str:
    """Where `got` first differs from the model stream `want`: the segment, the byte in it and the model's token there."""
    n = min(len(got), len(want))
    diff = next((k for k in range(n) if got[k] != want[k]), n)
    pos = 2
    for si, s in enumerate(segs):
        if diff < pos + len(s.out):
            return "segment %d (%s), byte %d of it (stream byte %d): model has %s; lengths %d vs %d" % (
                si, "dynamic" if s.dynamic else "stored", diff - pos, diff, s.token_at_byte(diff - pos), len(got), len(want))
        pos += len(s.out)
    return "trailer, stream byte %d; lengths %d vs %d" % (diff, len(got), len(want))
