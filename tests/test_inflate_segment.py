"""CPU tests (-m "not gpu") of the segment inflater the GPU inflate runs (csrc/rbf_inflate.cuh), through its host build
rbf_inflate_segment: every segment of the device coder's streams (modelled on the CPU by tests/deflate_model.compress) inflates
to its bytes with the right length consumed and Adler-32 sums, and a fixed set of malformed segments each comes back as a
non-zero status without a read or write outside its buffers."""
import ctypes as C
import zlib

import numpy as np
import pytest

from tests import deflate_model as dm

SEG = 65536


@pytest.fixture(scope="module")
def cabi():
    from new_bloom_filter_repo_b200 import build, _cabi
    build.build()
    return _cabi


def _text(n, seed):
    rng = np.random.default_rng(seed)
    words = [b"bloom", b"filter", b"frame", b"witness", b"segment", b"the", b"of", b"and", b"\n"]
    out = bytearray()
    while len(out) < n:
        out += words[int(rng.integers(0, len(words)))] + b" "
    return bytes(out[:n])


def _cases():
    rng = np.random.default_rng(20)
    sizes = (0, 1, 65535, 65536, 65537, 3 * 65536 + 1)
    for n in sizes:
        yield "random-%d" % n, rng.integers(0, 256, n, dtype=np.uint8).tobytes()          # stored segments
        yield "text-%d" % n, _text(n, n)
    yield "zeros", bytes(2 * SEG + 7)
    yield "runs", np.repeat(rng.integers(0, 256, 4000, dtype=np.uint8), rng.integers(1, 60, 4000)).tobytes()[:150000]
    yield "u16", (np.cumsum(rng.integers(-3, 4, 100000)) + 30000).astype(np.uint16).tobytes()


def _adler_parts(b: bytes):
    a = zlib.adler32(b, 0)
    return a & 0xFFFF, a >> 16


@pytest.mark.parametrize("name,data", list(_cases()), ids=[c[0] for c in _cases()])
def test_segments_inflate_like_zlib(cabi, name, data):
    stream, segs = dm.compress(data)
    assert zlib.decompress(stream) == data
    d = zlib.decompressobj()
    d.decompress(stream[:2])
    pos = 2
    for k, s in enumerate(segs):
        status, used, out, s1, s2 = cabi.inflate_segment(stream, pos)
        want = data[k * SEG:(k + 1) * SEG]
        assert status == 0, (name, k, status)
        assert used == len(s.out), (name, k)
        assert out == want and d.decompress(stream[pos:pos + used]) == want, (name, k)
        assert (s1, s2) == _adler_parts(want), (name, k)
        pos += used
    assert stream[pos:pos + 2] == b"\x03\x00" and pos + 6 == len(stream)


# ---------------------------------------------------------------- malformed segments
class _Bits:
    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, val, nb):                      # LSB first
        self.v |= (val & ((1 << nb) - 1)) << self.n
        self.n += nb

    def code(self, c, nb):                       # a Huffman code, most significant bit first
        for i in range(nb - 1, -1, -1):
            self.put((c >> i) & 1, 1)

    def bytes(self):
        return self.v.to_bytes((self.n + 7) // 8, "little")


def _dynamic(cl_lens, lens_syms, body, hlit, hdist):
    """A dynamic block (BFINAL 0) from code-length code lengths {sym: len}, the code-length symbols [(sym, extra, nbits)],
    and the body as [(code, nbits)], then an empty stored block."""
    w = _Bits()
    w.put(0, 1); w.put(2, 2)
    w.put(hlit - 257, 5); w.put(hdist - 1, 5); w.put(19 - 4, 4)
    for s in dm.CL_ORDER:
        w.put(cl_lens.get(s, 0), 3)
    lens = [cl_lens.get(s, 0) for s in range(19)]
    codes = [int(format(int(c), "0%db" % l)[::-1], 2) if l else 0 for c, l in zip(dm.canonical(lens), lens)]
    for sym, extra, nb in lens_syms:
        w.code(codes[sym], lens[sym])
        if nb:
            w.put(extra, nb)
    for c, nb in body:
        w.code(c, nb)
    w.put(0, 3)                                  # empty stored block
    return w.bytes() + b"\x00\x00\xff\xff"


_CL = {0: 2, 1: 2, 2: 2, 18: 2}                  # codes 00 01 10 11 for 0, 1, 2, 18
# literal/length lengths: 'A' 2, end-of-block 2, 257 (length 3) 1; distance 0 (distance 1) 1
_LENS = [(18, 54, 7), (2, 0, 0), (18, 127, 7), (18, 41, 7), (2, 0, 0), (1, 0, 0), (1, 0, 0)]
_A, _EOB, _M3, _D1 = (0b10, 2), (0b11, 2), (0b0, 1), (0b0, 1)


def _malformed():
    rng = np.random.default_rng(21)
    text = dm.compress(_text(3000, 5))[0][2:-6]
    rand = dm.compress(rng.integers(0, 256, 300, dtype=np.uint8).tobytes())[0][2:-6]
    assert text[0] & 7 == 4 and rand[0] == 0           # one dynamic and one stored segment
    cases = []
    for cut in range(len(text)):                       # every truncation of the dynamic segment, headers included
        cases.append(("dyn-cut-%d" % cut, text[:cut]))
    for cut in list(range(0, 12)) + [100, 304, len(rand) - 5, len(rand) - 1]:
        cases.append(("stored-cut-%d" % cut, rand[:cut]))
    cases.append(("btype-fixed", bytes([text[0] & ~6 | 2]) + text[1:]))
    cases.append(("btype-reserved", bytes([text[0] | 6]) + text[1:]))
    cases.append(("bfinal", bytes([text[0] | 1]) + text[1:]))
    cases.append(("stored-bfinal", bytes([1]) + rand[1:]))
    cases.append(("nlen", rand[:3] + bytes([rand[3] ^ 1]) + rand[4:]))
    cases.append(("cl-over", _dynamic({s: 1 for s in range(19)}, [], [], 257, 1)))
    cases.append(("cl-incomplete", _dynamic({1: 1}, [], [], 257, 1)))
    cases.append(("lit-over", _dynamic({1: 1, 2: 1}, [(1, 0, 0)] * 258, [], 257, 1)))
    cases.append(("lit-incomplete", _dynamic({0: 1, 2: 1}, [(2, 0, 0)] + [(0, 0, 0)] * 255 + [(2, 0, 0), (0, 0, 0)], [], 257, 1)))
    cases.append(("repeat-past", _dynamic(_CL, [(18, 127, 7), (18, 127, 7)], [], 258, 1)))
    cases.append(("no-eob", _dynamic(_CL, [(2, 0, 0), (2, 0, 0), (18, 127, 7), (18, 108, 7)], [], 258, 1)))
    cases.append(("dist-before-start", _dynamic(_CL, _LENS, [_M3, _D1, _EOB], 258, 1)))
    big = rng.integers(0, 256, SEG, dtype=np.uint8).tobytes()
    st = lambda b: bytes([0, len(b) & 255, len(b) >> 8, ~len(b) & 255, (~len(b) >> 8) & 255]) + b
    cases.append(("output-past-64k", st(big[:65535]) + st(big[:2]) + b"\x00\x00\x00\xff\xff"))
    return cases


def test_crafted_block_is_valid(cabi):
    """The crafting above is sound: 'A', a length-3 match at distance 1 and the end of block inflate (zlib agrees)."""
    seg = _dynamic(_CL, _LENS, [_A, _M3, _D1, _EOB], 258, 1)
    assert zlib.decompressobj(-15).decompress(seg) == b"AAAA"
    status, used, out, s1, s2 = cabi.inflate_segment(seg)
    assert (status, used, out) == (0, len(seg), b"AAAA")


def _run_guarded(cabi, seg, fill):
    """rbf_inflate_segment on seg placed between guard bytes of value `fill`; the output slot also has guards."""
    g = 4096
    inb = np.full(len(seg) + 2 * g, fill, dtype=np.uint8)
    inb[g:g + len(seg)] = np.frombuffer(seg, dtype=np.uint8)
    outb = np.full(SEG + 2 * g, fill ^ 0x5A, dtype=np.uint8)
    st, used, n, s1, s2 = C.c_uint32(), C.c_uint64(), C.c_uint32(), C.c_uint32(), C.c_uint32()
    base_in, base_out = inb.ctypes.data, outb.ctypes.data
    cabi.check(cabi.lib().rbf_inflate_segment(C.c_void_p(base_in + g), len(seg), C.c_void_p(base_out + g), C.byref(st),
                                              C.byref(used), C.byref(n), C.byref(s1), C.byref(s2)))
    assert (inb[:g] == fill).all() and (inb[g + len(seg):] == fill).all()
    assert (outb[:g] == (fill ^ 0x5A)).all() and (outb[g + SEG:] == (fill ^ 0x5A)).all(), "a write crossed the output slot"
    return int(st.value), int(used.value), bytes(outb[g:g + n.value])


@pytest.mark.parametrize("name,seg", _malformed(), ids=[c[0] for c in _malformed()])
def test_malformed_segment_is_a_status(cabi, name, seg):
    results = [_run_guarded(cabi, seg, fill) for fill in (0x00, 0xFF, 0x5A)]
    assert results[0][0] != 0, name
    # the guards after the input differ between the runs: a read past the input would change the result
    assert results[0] == results[1] == results[2], name
