"""A pure-Python RFC 1951 / 1950 inflater (puff-style) and the GPU inflater's layout rules, written from the header of
csrc/rbf_inflate.cuh and from inflate_streams in csrc/rbf_api.cu.

decompress(stream)       zlib.decompress(stream): the bytes, or ZlibError with zlib's own message where zlib raises one.  Code
                         sets are judged as zlib's inflate_table judges them.
segment(stream, start)   the device's view of one segment starting at stream[start]: accepted or not, bytes consumed through the
                         closing 00 00 FF FF, output, Adler-32 parts from (0, 0), and the facts of each block (Block).
verdict(stream, bound)   whether rbf_zlib_decompress_batch inflates the stream on the device (Verdict.on_device), and why not.
features(v)              the edges a device-routed stream reaches (FEATURES), from its blocks.
"""
from __future__ import annotations

import zlib
from dataclasses import dataclass, field
from typing import List, Optional

SEG = 65536
MARKER = b"\x00\x00\xff\xff"
MAX_RATIO = 1032                       # deflate.decompress_routed's default bound per input byte
CL_ORDER = (16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)
LEN_BASE = (3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258)
LEN_EXTRA = (0,) * 8 + (1,) * 4 + (2,) * 4 + (3,) * 4 + (4,) * 4 + (5,) * 4 + (0,)
DIST_BASE = (1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577)
DIST_EXTRA = (0, 0, 0, 0) + tuple(e for e in range(1, 14) for _ in (0, 1))

# Every edge the corpus must reach on the device (features() names).
FEATURES = (
    "multi_huffman",          # a segment with several Huffman blocks
    "stored_then_huffman",    # a Huffman block after a non-empty stored block, in one segment
    "huffman_then_stored",    # a non-empty stored block after a Huffman block, in one segment
    "lit15", "dist15",        # a 15-bit code
    "lit9", "lit10",          # longest literal/length code of exactly 9 (the fast-table root) and 10 bits
    "dist8", "dist9",         # and of the distance code: 8 (its root) and 9 bits
    "lit_eob_only",           # a literal/length code holding only end-of-block (one length-1 code)
    "dist_one_code",          # a distance code of one length-1 code
    "dist_empty",             # a block without distance codes
    "hlit286", "hdist30",
    "rep16x6", "rep17x10", "rep18x138", "rep16_cross",   # maximal repeats; a 16 across the literal/distance boundary
    "len258_285", "len258_284",                          # length 258 as symbol 285 and as 284 + 31
    "dist32768", "dist_eq_out",                          # the longest distance; a distance equal to the segment's output
    "match_end_64k",                                     # a match that ends exactly at 65536
    "stored65535",                                       # a 65535-byte stored block
    "blocks100",                                         # 100 or more blocks in one segment
)


class ZlibError(Exception):
    """zlib.decompress's error, with its message."""


def _err(msg, code=-3):
    return ZlibError("Error %d while decompressing data: %s" % (code, msg))


class _Truncated(ZlibError):
    def __init__(self):
        super().__init__("Error -5 while decompressing data: incomplete or truncated stream")


class _Refused(Exception):
    """The device refuses the segment (a rule zlib does not have)."""


class _Bits:
    """LSB-first bit reader over data[.. end)."""

    def __init__(self, data, byte_pos):
        self.d, self.p, self.end = data, 8 * byte_pos, 8 * len(data)

    def need(self, n):
        if self.p + n > self.end:
            raise _Truncated()

    def peek(self, n):
        i = self.p >> 3
        return (int.from_bytes(self.d[i:i + 4], "little") >> (self.p & 7)) & ((1 << n) - 1)

    def get(self, n):
        self.need(n)
        v = self.peek(n)
        self.p += n
        return v

    def align(self):
        self.p = (self.p + 7) & ~7


class _Code:
    """A canonical code, judged as inflate_table judges it (kind: 'codes', 'lens' or 'dists')."""

    def __init__(self, lens, kind):
        count = [0] * 16
        for n in lens:
            count[n] += 1
        count[0] = 0
        self.max = max([b for b in range(1, 16) if count[b]], default=0)
        self.ncodes = sum(count)
        left = 1
        for b in range(1, 16):
            left = 2 * left - count[b]
            if left < 0:
                raise ValueError("over-subscribed")
        if self.max and left > 0 and (kind == "codes" or self.max != 1):
            raise ValueError("incomplete")
        self.table = [None] * (1 << max(self.max, 1))
        code, nxt = 0, [0] * 16
        for b in range(1, 16):
            code = (code + count[b - 1]) << 1
            nxt[b] = code
        for s, n in enumerate(lens):
            if n:
                c = nxt[n]
                nxt[n] += 1
                r = int(format(c, "0%db" % n)[::-1], 2)
                for f in range(r, len(self.table), 1 << n):
                    self.table[f] = (s, n)

    def decode(self, B, invalid):
        """One symbol.  A pattern that is no code (an empty set, or the unused half of a single length-1 code) is found after
        one bit, as zlib finds it."""
        if self.max == 0:
            B.get(1)
            return None
        e = self.table[B.peek(self.max)]
        if e is None:
            B.need(1)
            raise _err(invalid)
        B.need(e[1])
        B.p += e[1]
        return e[0]


_FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
_FIXED_DIST = [5] * 32


@dataclass
class Block:
    type: str                              # "stored", "fixed" or "dynamic"
    final: int = 0
    stored_len: int = 0
    hlit: int = 0
    hdist: int = 0
    lit_max: int = 0
    lit_n: int = 0
    dist_max: int = 0
    dist_n: int = 0
    lit_eob_only: bool = False
    reps: set = field(default_factory=set)     # ("16", 6), ("17", 10), ("18", 138), ("16x", n) across the boundary
    len258: set = field(default_factory=set)   # {285, 284}
    max_dist: int = 0
    dist_eq_out: bool = False
    match_end_64k: bool = False


def _blocks(data, B, out, seg_start, seg):
    """Inflate blocks from B into out.  seg: the device's segment rules (stop at the first empty stored block, refuse fixed and
    final blocks, distances before seg_start, more than 64 KiB); else zlib's (run through the final block)."""
    blocks: List[Block] = []
    while True:
        B.need(3)
        h = B.get(3)
        final, btype = h & 1, h >> 1
        if seg and final:
            raise _Refused("final")
        if btype == 0:
            B.align()
            B.need(32)
            ln, nln = B.get(16), B.get(16)
            if ln != (~nln & 0xFFFF):
                raise _err("invalid stored block lengths")
            if seg and ln == 0:
                return blocks
            B.need(8 * ln)
            if seg and len(out) - seg_start + ln > SEG:
                raise _Refused("output past 64 KiB")
            i = B.p >> 3
            out += data[i:i + ln]
            B.p += 8 * ln
            blocks.append(Block("stored", final, stored_len=ln))
        elif btype == 3:
            raise _err("invalid block type")
        else:
            blk = Block("fixed" if btype == 1 else "dynamic", final)
            if btype == 1:
                if seg:
                    raise _Refused("fixed")
                lit, dist = _Code(_FIXED_LIT, "lens"), _Code(_FIXED_DIST, "dists")
            else:
                lit, dist = _header(B, blk)
            _body(B, out, lit, dist, blk, seg_start, seg)
            blocks.append(blk)
        if final:
            return blocks


def _header(B, blk):
    hlit, hdist, hclen = B.get(5) + 257, B.get(5) + 1, B.get(4) + 4
    if hlit > 286 or hdist > 30:
        raise _err("too many length or distance symbols")
    cl = [0] * 19
    for i in range(hclen):
        cl[CL_ORDER[i]] = B.get(3)
    try:
        clc = _Code(cl, "codes")
    except ValueError:
        raise _err("invalid code lengths set")
    lens, total = [], hlit + hdist
    while len(lens) < total:
        sym = clc.decode(B, "invalid code lengths set")
        sym = 0 if sym is None else sym                  # an empty code-length code reads every length as 0, one bit each
        if sym < 16:
            lens.append(sym)
            continue
        if sym == 16:
            n = 3 + B.get(2)
            if not lens:
                raise _err("invalid bit length repeat")
            v = lens[-1]
        elif sym == 17:
            n, v = 3 + B.get(3), 0
        else:
            n, v = 11 + B.get(7), 0
        if len(lens) + n > total:
            raise _err("invalid bit length repeat")
        if sym == 16 and len(lens) < hlit < len(lens) + n:
            blk.reps.add(("16x", n))
        blk.reps.add((str(sym), n))
        lens += [v] * n
    if lens[256] == 0:
        raise _err("invalid code -- missing end-of-block")
    try:
        lit = _Code(lens[:hlit], "lens")
    except ValueError:
        raise _err("invalid literal/lengths set")
    try:
        dist = _Code(lens[hlit:], "dists")
    except ValueError:
        raise _err("invalid distances set")
    blk.hlit, blk.hdist = hlit, hdist
    blk.lit_max, blk.lit_n, blk.dist_max, blk.dist_n = lit.max, lit.ncodes, dist.max, dist.ncodes
    blk.lit_eob_only = lit.ncodes == 1 and lens[256] == 1
    return lit, dist


def _body(B, out, lit, dist, blk, seg_start, seg):
    while True:
        sym = lit.decode(B, "invalid literal/length code")
        if sym is None:
            raise _err("invalid literal/length code")
        if sym < 256:
            if seg and len(out) - seg_start >= SEG:
                raise _Refused("output past 64 KiB")
            out.append(sym)
            continue
        if sym == 256:
            return
        if sym > 285:
            raise _err("invalid literal/length code")
        ln = LEN_BASE[sym - 257] + B.get(LEN_EXTRA[sym - 257])
        if ln == 258:
            blk.len258.add(sym)
        ds = dist.decode(B, "invalid distance code")
        if ds is None or ds > 29:
            raise _err("invalid distance code")
        d = DIST_BASE[ds] + B.get(DIST_EXTRA[ds])
        p = len(out) - seg_start
        if d > len(out):
            raise _err("invalid distance too far back")
        if seg and d > p:
            raise _Refused("distance before the segment")
        if seg and ln > SEG - p:
            raise _Refused("output past 64 KiB")
        blk.max_dist = max(blk.max_dist, d)
        blk.dist_eq_out |= d == p
        blk.match_end_64k |= p + ln == SEG
        src = len(out) - d
        if d >= ln:
            out += out[src:src + ln]
        else:
            for k in range(ln):
                out.append(out[src + k])


def decompress(stream) -> bytes:
    """zlib.decompress(stream), or ZlibError with its message."""
    data = bytes(stream)
    if len(data) < 2:
        raise _Truncated()
    cmf, flg = data[0], data[1]
    if (cmf << 8 | flg) % 31:
        raise _err("incorrect header check")
    if cmf & 15 != 8:
        raise _err("unknown compression method")
    if cmf >> 4 > 7:
        raise _err("invalid window size")
    if flg & 0x20:
        raise ZlibError("Error 2 while decompressing data")
    B = _Bits(data, 2)
    out = bytearray()
    _blocks(data, B, out, 0, False)
    B.align()
    B.need(32)
    i = B.p >> 3
    if int.from_bytes(data[i:i + 4], "big") != zlib.adler32(out):
        raise _err("incorrect data check")
    return bytes(out)


@dataclass
class Seg:
    ok: bool
    reason: str = ""
    consumed: int = 0
    out: bytes = b""
    s1: int = 0
    s2: int = 0
    blocks: List[Block] = field(default_factory=list)


def segment(stream, start: int) -> Seg:
    """The device's verdict on the segment at stream[start:] (avail = the rest of the stream)."""
    data = bytes(stream)
    B = _Bits(data, start)
    out = bytearray()
    try:
        blocks = _blocks(data, B, out, 0, True)
    except (ZlibError, _Refused) as e:
        return Seg(False, str(e))
    a = zlib.adler32(bytes(out), 0)
    return Seg(True, "", (B.p >> 3) - start, bytes(out), a & 0xFFFF, a >> 16, blocks)


def candidates(stream) -> List[int]:
    """k_inflate_scan's candidate starts: 2 and every offset after 00 00 FF FF, below the 6-byte trailer."""
    s = bytes(stream)
    end = len(s) - 6
    out = [2] if 2 < end else []
    q = s.find(MARKER, 2)
    while q != -1 and q + 4 < end:
        if q + 4 >= 6:
            out.append(q + 4)
        q = s.find(MARKER, q + 1)
    return out


def cap(n: int, bound: int) -> int:
    return min(2 * -(-bound // SEG) + 8, n // 4 + 2)


@dataclass
class Verdict:
    on_device: bool
    reason: str = ""
    segs: List[Seg] = field(default_factory=list)
    total: int = 0
    ncand: int = 0
    cap: int = 0


def verdict(stream, bound: Optional[int] = None) -> Verdict:
    """Whether the device inflates `stream` under `bound` (default: deflate's largest ratio, as decompress_routed uses)."""
    s = bytes(stream)
    if len(s) < 8 or s[:2] != b"\x78\x9c":
        return Verdict(False, "header or length")
    bound = MAX_RATIO * len(s) if bound is None else bound
    cands = candidates(s)
    v = Verdict(False, "", [], 0, len(cands), cap(len(s), bound))
    if v.ncand > v.cap:
        v.reason = "more candidates than the cap"
        return v
    pos, end = 2, len(s) - 6
    while pos < end:
        if v.segs and len(v.segs[-1].out) != SEG:
            v.reason = "a segment before the last is not 64 KiB"
            return v
        g = segment(s, pos)
        if not g.ok:
            v.reason = "segment at %d: %s" % (pos, g.reason)
            return v
        v.segs.append(g)
        pos += g.consumed
    out = b"".join(g.out for g in v.segs)
    v.total = len(out)
    if pos != end or s[end:end + 2] != b"\x03\x00":
        v.reason = "no 03 00 at the chain's end"
    elif int.from_bytes(s[end + 2:], "big") != zlib.adler32(out):
        v.reason = "Adler-32"
    elif v.total > bound:
        v.reason = "over the bound"
    else:
        v.on_device = True
    return v


def features(v: Verdict) -> set:
    """The FEATURES a stream reaches (of a device-routed verdict)."""
    f = set()
    for g in v.segs:
        kinds = [b.type for b in g.blocks if b.type == "dynamic" or b.stored_len]
        if kinds.count("dynamic") >= 2:
            f.add("multi_huffman")
        for a, b in zip(kinds, kinds[1:]):
            f.add({("stored", "dynamic"): "stored_then_huffman", ("dynamic", "stored"): "huffman_then_stored"}.get((a, b), ""))
        if len(g.blocks) >= 100:
            f.add("blocks100")
        for b in g.blocks:
            if b.stored_len == 65535:
                f.add("stored65535")
            if b.type != "dynamic":
                continue
            f |= {"lit%d" % b.lit_max, "dist%d" % b.dist_max, "hlit%d" % b.hlit, "hdist%d" % b.hdist}
            f |= {"len258_%d" % s for s in b.len258}
            f |= {"rep%sx%d" % r if r[0] != "16x" else "rep16_cross" for r in b.reps}
            if b.lit_eob_only:
                f.add("lit_eob_only")
            if b.dist_n == 1 and b.dist_max == 1:
                f.add("dist_one_code")
            if b.dist_n == 0:
                f.add("dist_empty")
            if b.max_dist == 32768:
                f.add("dist32768")
            if b.dist_eq_out:
                f.add("dist_eq_out")
            if b.match_end_64k:
                f.add("match_end_64k")
    return f & set(FEATURES)
