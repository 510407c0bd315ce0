"""CPU tests (-m "not gpu") of the GPU inflater's layout rules and of its segment routine (csrc/rbf_inflate.cuh, through the host
build rbf_inflate_segment) on streams the device coder does not write: zlib-written streams in and out of the segment layout,
hand-built segments of the code shapes zlib never writes, and malformed streams.  The pure-Python inflater in
tests/inflate_model.py is checked against zlib.decompress here, and then serves as the oracle for the routine's results and
for which streams the device takes (tests/test_gpu_inflate_corpus.py)."""
import functools
import zlib

import pytest

from tests import deflate_model as dm
from tests import inflate_corpus as ic
from tests import inflate_model as im
from tests.test_inflate_segment import _malformed, _text


@pytest.fixture(scope="module")
def cabi():
    from new_bloom_filter_repo_b200 import build, _cabi
    build.build()
    return _cabi


@functools.lru_cache(maxsize=None)
def _corpus():
    return dict(ic.corpus())


def _zlib(s):
    try:
        return ("ok", zlib.decompress(s))
    except zlib.error as e:
        return ("error", str(e))


def _model(s):
    try:
        return ("ok", im.decompress(s))
    except im.ZlibError as e:
        return ("error", str(e))


@pytest.mark.parametrize("name", list(_corpus()))
def test_model_inflates_like_zlib(name):
    s = _corpus()[name]
    want = _zlib(s)
    assert want[0] == "ok", name
    assert _model(s) == want, name


def test_routes_and_coverage():
    """Which corpus streams the layout admits, and every FEATURES edge reached by at least one of them."""
    reached, by_zlib, dev = set(), set(), 0
    for name, s in _corpus().items():
        v = im.verdict(s)
        dev += v.on_device
        crafted = name.startswith(("crafted-", "split-"))
        if crafted:
            assert v.on_device, (name, v.reason)
        if "-L0-" in name or "-step" in name or ("-S4-" in name and "-0-" not in name):   # level 0, other flush intervals, Z_FIXED
            assert not v.on_device, name
        if v.on_device:
            reached |= im.features(v)
            if not crafted:
                by_zlib |= im.features(v)
    assert reached == set(im.FEATURES), sorted(set(im.FEATURES) - reached)
    assert {"multi_huffman", "lit9", "dist8", "rep16x6"} <= by_zlib         # zlib's own block splits and code shapes
    assert 0 < dev < len(_corpus())


def _bad_streams():
    """The malformed cases of tests/test_gpu_inflate.py, built on the modelled device coder's stream instead of the GPU's."""
    text = _text(150000, 7)
    s = dm.compress(text)[0]
    wrap = lambda seg: b"\x78\x9c" + seg + b"\x03\x00" + zlib.adler32(b"").to_bytes(4, "big")
    cases = [(n, wrap(seg)) for n, seg in _malformed()]
    cases += [("cut-%d" % k, s[:k]) for k in (0, 1, 2, 3, 7, 8, 10, len(s) // 2, len(s) - 7, len(s) - 6, len(s) - 1)]
    cases += [("bad-adler", s[:-1] + bytes([s[-1] ^ 1])), ("after-trailer", s + b"\x00"), ("after-trailer-2", s + s)]
    cases += [("bad-03", s[:-6] + b"\x03\x01" + s[-4:]), ("flip-mid", s[:5000] + bytes([s[5000] ^ 0x10]) + s[5001:])]
    return cases


def test_model_raises_where_zlib_raises():
    """The model raises zlib's error at the same place (its message), and the layout declines every case but the one that is
    zlib.compress(b"") (an empty segment list), which inflates to nothing on the device too."""
    for name, s in _bad_streams():
        assert _model(s) == _zlib(s), name
        v = im.verdict(s)
        assert v.on_device == (s == zlib.compress(b"")), (name, v.reason)


def test_host_segment_matches_model_on_malformed_streams(cabi):
    for name, s in _bad_streams():
        for q in im.candidates(s):
            status, used, out, s1, s2 = cabi.inflate_segment(s, q)
            g = im.segment(s, q)
            assert (status == 0) == g.ok, (name, q, status, g.reason)
            if g.ok:
                assert (used, out, s1, s2) == (g.consumed, g.out, g.s1, g.s2), (name, q)


@pytest.mark.parametrize("name", list(_corpus()))
def test_host_segment_matches_model_at_every_candidate(cabi, name):
    """rbf_inflate_segment at every candidate start the scan would list: accepted exactly when the model accepts, and then the
    same bytes consumed, output and Adler-32 parts."""
    s = _corpus()[name]
    for q in im.candidates(s):
        g = im.segment(s, q)
        status, used, out, s1, s2 = cabi.inflate_segment(s, q)
        assert (status == 0) == g.ok, (name, q, status, g.reason)
        if g.ok:
            assert (used, out, s1, s2) == (g.consumed, g.out, g.s1, g.s2), (name, q)
