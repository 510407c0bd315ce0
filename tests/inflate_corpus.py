"""Streams for the GPU inflater's tests (tests/test_inflate_corpus.py on the CPU, tests/test_gpu_inflate_corpus.py on the GPU),
from producers other than the device coder:

zlib_streams()    zlib 1.3 driven into the segment layout (layout()): levels, memLevels, strategies and window sizes over random
                  data, text, long runs, u16 ramps, random-then-text segments and stored data holding 00 00 FF FF; plus streams
                  flushed at other intervals, which are outside the layout.
crafted_streams() hand-built segments of the shapes zlib does not write (Writer / dynamic()), each alone and behind full
                  64 KiB segments.
split_streams()   segment starts on and beside the scan's job boundaries (2 + k * 8192).
cap_stream(n)     one stored segment with n planted 00 00 FF FF markers.
Each corpus entry is (name, stream).  zlib.decompress is the reference for every stream's bytes.
"""
from __future__ import annotations

import itertools
import zlib

import numpy as np

from tests import inflate_model as im
from tests.test_inflate_segment import _text

SEG = 65536
SIZES = (0, 1, 65535, 65536, 65537, 3 * SEG + 1)
LEVELS = (1, 4, 6, 9, 0)
MEMLEVELS = (1, 8, 9)
STRATEGIES = (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED)
WBITS = (9, 15)
SCAN_CHUNK = 8192                      # kInflateScanChunk: positions per k_inflate_scan job


def layout(data: bytes, level=6, memlevel=8, strategy=zlib.Z_DEFAULT_STRATEGY, wbits=15, step=SEG) -> bytes:
    """zlib's stream of data, with a full flush (00 00 FF FF, match state reset) after every `step` bytes and the header
    rewritten to 78 9C.  For step 64 KiB and level >= 1 that is the device layout, except where zlib writes a fixed block."""
    co = zlib.compressobj(level, zlib.DEFLATED, wbits, memlevel, strategy)
    out = b"".join(co.compress(data[i:i + step]) + co.flush(zlib.Z_FULL_FLUSH) for i in range(0, len(data), step) or [0])
    out += co.flush(zlib.Z_FINISH)
    return b"\x78\x9c" + out[2:]


# ---------------------------------------------------------------- data
def _random(n, rng):
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes()


def _runs(n, rng):
    """Runs longer than 258 (matches of 258 at distance 1) between short random stretches."""
    out = bytearray()
    while len(out) < n:
        out += bytes([int(rng.integers(0, 256))]) * int(rng.integers(259, 2000)) + _random(int(rng.integers(1, 40)), rng)
    return bytes(out[:n])


def _ramp(n, rng):
    return (np.arange(n // 2 + 1) * int(rng.integers(1, 7)) + int(rng.integers(0, 65536))).astype(np.uint16).tobytes()[:n]


def _rand_text(n, rng):
    """Per 64 KiB: 20000 random bytes, then text: stored and Huffman blocks in one segment."""
    return b"".join(_random(20000, rng) + _text(SEG - 20000, int(rng.integers(1 << 30))) for _ in range(n // SEG + 1))[:n]


def _planted(n, rng):
    """Random bytes (stored blocks) holding 00 00 FF FF every 4099 bytes and right before each 64 KiB boundary."""
    b = bytearray(_random(n, rng))
    for off in list(range(7, n - 4, 4099)) + list(range(SEG - 4, n - 4, SEG)):
        b[off:off + 4] = im.MARKER
    return bytes(b)


KINDS = {"random": _random, "text": lambda n, rng: _text(n, int(rng.integers(1 << 30))), "runs": _runs, "ramp": _ramp,
         "randtext": _rand_text, "planted": _planted}


def zlib_streams():
    """A fixed subset of level x memLevel x strategy x wbits over every kind and size: each kind and size once, with the
    settings cycled so that each setting occurs with several kinds; then the other flush intervals."""
    rng = np.random.default_rng(60)
    out = []
    for i, (kind, n) in enumerate(itertools.product(KINDS, SIZES)):
        level, mem, strat, wb = LEVELS[i % 5], MEMLEVELS[i % 3], STRATEGIES[(i // 2) % 5], WBITS[(i // 3) % 2]
        if n > 2 * SEG and mem == 1:
            mem = 9                                  # keeps the model's work down: memLevel 1 writes a block per 128 symbols
        out.append(("%s-%d-L%d-M%d-S%d-W%d" % (kind, n, level, mem, strat, wb), layout(KINDS[kind](n, rng), level, mem, strat, wb)))
    text = _text(2 * SEG + 300, 61)
    for mem in MEMLEVELS:                            # many blocks per segment, at every level
        for level in (1, 6, 9):
            out.append(("text-M%d-L%d" % (mem, level), layout(text[:SEG + 5000], level, mem)))
    out.append(("randtext-M1", layout(_rand_text(SEG + 10, rng), 6, 1)))
    for kind in KINDS:                               # several segments each, at zlib's defaults
        out.append(("%s-%d-default" % (kind, 3 * SEG + 1), layout(KINDS[kind](3 * SEG + 1, rng))))
    for step in (32768, SEG - 1, SEG + 1):           # other flush intervals: outside the layout
        out.append(("text-step%d" % step, layout(text, 6, 8, step=step)))
    return out


# ---------------------------------------------------------------- hand-built segments
class Writer:
    """LSB-first bit writer into a bytearray (stored blocks of 64 KiB go in as bytes)."""

    def __init__(self):
        self.buf, self.acc, self.n = bytearray(), 0, 0

    def put(self, v, nb):
        self.acc |= (v & ((1 << nb) - 1)) << self.n
        self.n += nb
        while self.n >= 8:
            self.buf.append(self.acc & 255)
            self.acc >>= 8
            self.n -= 8

    def align(self):
        if self.n:
            self.put(0, 8 - self.n)

    def stored(self, data: bytes):
        self.put(0, 3)
        self.align()
        n = len(data)
        self.buf += bytes([n & 255, n >> 8, ~n & 255, (~n >> 8) & 255]) + data

    def bytes(self):
        assert self.n == 0
        return bytes(self.buf)


def lengths(n, maxlen):
    """Sorted lengths of a complete code of n symbols whose longest code has exactly maxlen bits."""
    L = [1, 1]
    while max(L) < maxlen:                           # a staircase down to maxlen
        L.remove(max(L))
        L += [max(L) + 1] * 2 if L else [2, 2]
    while len(L) < n:                                # then split the shortest leaves
        s = min(x for x in L if x < maxlen)
        L.remove(s)
        L += [s + 1] * 2
    assert len(L) == n and sum(2.0 ** -x for x in L) == 1.0
    return sorted(L)


def assign(syms, maxlen):
    """{sym: length}: a complete code over syms, the last ones in `syms` getting the longest codes."""
    if len(syms) == 1:
        return {syms[0]: 1}
    return dict(zip(syms, lengths(len(syms), maxlen)))


def _rev_codes(lens):
    count = [0] * 16
    for x in lens:
        count[x] += 1
    count[0] = 0
    nxt, code = [0] * 16, 0
    for b in range(1, 16):
        code = (code + count[b - 1]) << 1
        nxt[b] = code
    out = []
    for x in lens:
        out.append(int(format(nxt[x], "0%db" % x)[::-1], 2) if x else 0)
        if x:
            nxt[x] += 1
    return out


def _rle(lens):
    """Code-length symbols (sym, extra, extra bits) of lens, taking the longest repeats (across the lit/dist boundary too)."""
    out, i = [], 0
    while i < len(lens):
        v, run = lens[i], 1
        while i + run < len(lens) and lens[i + run] == v:
            run += 1
        if v == 0 and run >= 11:
            r = min(run, 138); out.append((18, r - 11, 7))
        elif v == 0 and run >= 3:
            r = min(run, 10); out.append((17, r - 3, 3))
        else:
            out.append((v, 0, 0)); r = 1
            while v and run - r >= 3:
                k = min(run - r, 6); out.append((16, k - 3, 2)); r += k
        i += r
    return out


_CL_LENS = assign(list(range(19)), 5)


def _len_code(n):
    s = max(k for k, b in enumerate(im.LEN_BASE) if b <= n)
    return 257 + s, n - im.LEN_BASE[s], im.LEN_EXTRA[s]


def _dist_code(d):
    s = max(k for k, b in enumerate(im.DIST_BASE) if b <= d)
    return s, d - im.DIST_BASE[s], im.DIST_EXTRA[s]


def _syms(body):
    lit, dist = {256}, set()
    for t in body:
        if isinstance(t, int):
            lit.add(t)
        else:
            lit.add(284 if t[0] == "m284" else _len_code(t[1])[0])
            dist.add(_dist_code(t[2])[0])
    return lit, dist


def dynamic(w: Writer, body, lit=None, dist=None, hlit=None, hdist=None):
    """A BFINAL-0 dynamic block: body items are literal bytes, ("m", length, distance) and ("m284", 258, distance) (258 as
    284 + 31).  lit / dist: {sym: length} (default: a complete code over the symbols used, or none / one length-1 code)."""
    ls, ds = _syms(body)
    if lit is None:
        lit = assign(sorted(ls), max(1, (len(ls) - 1).bit_length()))
    if dist is None:
        dist = assign(sorted(ds), max(1, (len(ds) - 1).bit_length())) if ds else {}
    hlit = hlit or max(257, max(lit) + 1)
    hdist = hdist or max(1, max(dist, default=0) + 1)
    ll = [lit.get(s, 0) for s in range(hlit)]
    dl = [dist.get(s, 0) for s in range(hdist)]
    cl = [_CL_LENS[s] for s in range(19)]
    clc, lc, dc = _rev_codes(cl), _rev_codes(ll), _rev_codes(dl)
    w.put(0, 1); w.put(2, 2)
    w.put(hlit - 257, 5); w.put(hdist - 1, 5); w.put(19 - 4, 4)
    for s in im.CL_ORDER:
        w.put(cl[s], 3)
    for sym, extra, nb in _rle(ll + dl):
        w.put(clc[sym], cl[sym]); w.put(extra, nb)
    for t in body:
        if isinstance(t, int):
            w.put(lc[t], ll[t])
            continue
        sym, extra, nb = (284, 31, 5) if t[0] == "m284" else _len_code(t[1])
        w.put(lc[sym], ll[sym]); w.put(extra, nb)
        sym, extra, nb = _dist_code(t[2])
        w.put(dc[sym], dl[sym]); w.put(extra, nb)
    w.put(lc[256], ll[256])


def _segment(*parts):
    """A segment from parts: bytes (a stored block) or callables writing blocks; closed by an empty stored block."""
    w = Writer()
    for p in parts:
        if isinstance(p, (bytes, bytearray)):
            w.stored(bytes(p))
        else:
            p(w)
    w.stored(b"")
    return w.bytes()


def _crafted_segments():
    rng = np.random.default_rng(62)
    R = lambda n: _random(n, rng)
    letters = list(b"abcdefghijklmnopqrstuvwxyz")
    segs = []
    segs.append(("eob-only", _segment(b"eob-only block follows", lambda w: dynamic(w, [], lit={256: 1}, dist={}))))
    segs.append(("dist-one-code", _segment(lambda w: dynamic(w, [97, 98, ("m", 5, 1)], dist={0: 1}))))
    segs.append(("dist-empty", _segment(lambda w: dynamic(w, list(b"literals only, no distance code")))))
    # every literal/length and distance symbol coded (HLIT 286, HDIST 30), 15-bit codes used; 258 both ways; distance 32768
    lit15 = assign([s for s in range(286) if s not in (97, 284, 285)] + [97, 284, 285], 15)
    dist15 = assign(list(range(29)) + [29], 15)
    segs.append(("lit15-dist15", _segment(R(40000), lambda w: dynamic(
        w, [97, ("m", 258, 32768), ("m284", 258, 1), 97, ("m", 258, 24577), 97], lit=lit15, dist=dist15, hlit=286, hdist=30))))
    # the longest codes just at and just above the fast-table roots (literal/length 9, distance 8)
    for lmax, dmax in ((9, 8), (10, 9)):
        syms = [256, 257, 258] + letters[:-1] + [ord("z")]
        dsyms = list(range(dmax)) + [dmax]                   # distances 1 .. ; the deepest is the last
        body = letters + [ord("z")] + [("m", 3, im.DIST_BASE[dmax]), ("m", 4, 1), ("m", 3, 2)]
        segs.append(("lit%d-dist%d" % (lmax, dmax), _segment(lambda w, body=body, syms=syms, dsyms=dsyms, lmax=lmax, dmax=dmax: dynamic(
            w, body, lit=assign(syms, lmax), dist=assign(dsyms, dmax)))))
    # 18 x 138, 17 x 10, a literal then 16 x 6, and a 16 that runs from the literal/length lengths into the distance lengths
    rlit = {s: 3 for s in range(148, 155)}
    rlit.update({s: 6 for s in range(280, 286)})
    rlit[256] = 5
    rdist = {0: 6, 1: 6, 2: 6, 3: 6, 4: 1, 5: 2, 6: 3, 7: 4}
    segs.append(("repeats", _segment(lambda w: dynamic(w, list(range(148, 155)) + [("m", 115, 7), ("m", 130, 1)],
                                                       lit=rlit, dist=rdist, hlit=286, hdist=8))))
    segs.append(("dist-eq-out", _segment(lambda w: dynamic(w, [120, 121, 122, ("m", 3, 3), ("m", 12, 6)]))))
    segs.append(("match-end-64k", _segment(R(SEG - 259), lambda w: dynamic(w, [7, ("m", 258, 1)]))))
    segs.append(("stored65535-literal", _segment(R(65535), lambda w: dynamic(w, [42]))))
    segs.append(("blocks100", _segment(*[lambda w, k=k: dynamic(w, [65 + k % 26, 48 + k % 10]) for k in range(100)])))
    segs.append(("mixed", _segment(lambda w: dynamic(w, list(b"huffman first")), R(100),
                                   lambda w: dynamic(w, list(b"then") + [("m", 40, 60), ("m", 13, 113)]))))
    return segs


def _full_segments(k, seed):
    """k zlib-written segments of 64 KiB of text each (raw deflate, full flush)."""
    co = zlib.compressobj(6, zlib.DEFLATED, -15)
    return [co.compress(_text(SEG, seed + i)) + co.flush(zlib.Z_FULL_FLUSH) for i in range(k)]


def wrap(segs) -> bytes:
    """78 9C, the segments, 03 00 and the Adler-32 of what zlib inflates them to."""
    raw = b"".join(segs)
    data = zlib.decompressobj(-15).decompress(raw)
    return b"\x78\x9c" + raw + b"\x03\x00" + zlib.adler32(data).to_bytes(4, "big")


def crafted_streams():
    full = _full_segments(2, 63)
    out = []
    for name, seg in _crafted_segments():
        out.append(("crafted-%s" % name, wrap([seg])))
        out.append(("crafted-%s-behind" % name, wrap(full + [seg])))
    return out


def _pad_segment(size):
    """A segment of exactly `size` bytes that inflates to 64 KiB: a stored block, then a run of 258-byte matches."""
    for m in range(size - 200, size):
        seg = _segment(bytes(range(256)) * (m // 256) + bytes(range(m % 256)),
                       lambda w: dynamic(w, [0] + [("m", 258, 1)] * ((SEG - m - 1) // 258) +
                                         ([("m", (SEG - m - 1) % 258, 1)] if (SEG - m - 1) % 258 >= 3 else
                                          [0] * ((SEG - m - 1) % 258))))
        if len(seg) == size:
            return seg
    raise AssertionError(size)


def split_streams():
    """Streams whose second segment starts at 2 + k * 8192 + d (d in -1, 0, 1): a start on the first position of a scan job,
    on the last position of the job before, and one past."""
    out = []
    for k in (1, 3):
        for d in (-1, 0, 1):
            first = _pad_segment(k * SCAN_CHUNK + d)
            out.append(("split-%d%+d" % (k, d), wrap([first, _segment(b"the next segment")])))
    return out


def cap_stream(n, size=5000, seed=64):
    """One stored segment of `size` random bytes holding n planted 00 00 FF FF markers: n + 1 candidate starts."""
    b = bytearray(_random(size, np.random.default_rng(seed)).replace(im.MARKER, b"\x01\x00\xff\xff"))
    for k in range(n):
        off = 20 + k * 9
        b[off:off + 4] = im.MARKER
    return wrap([_segment(bytes(b))])


def corpus():
    return zlib_streams() + crafted_streams() + split_streams()
