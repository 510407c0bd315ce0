"""GPU inflate (rbf_zlib_decompress_batch, csrc/rbf_inflate.cuh) of streams other producers write: zlib in and out of the
segment layout, hand-built segments of the code shapes zlib never writes, and malformed streams, alone and in one mixed batch.
Every stream returns zlib.decompress's bytes, and goes to the device exactly when tests/inflate_model.py's layout verdict says
so; the bound, output capacity, candidate cap and scan-job edges are pinned; decompress_video takes a group to the host as a
whole when one of its value streams is not the device's or is declined."""
import ctypes as C
import functools
import struct
import zlib

import numpy as np
import pytest

from tests import inflate_corpus as ic
from tests import inflate_model as im
from tests.test_gpu_inflate import _bad_streams, _data, _frames, _gpu_file

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    import new_bloom_filter_repo_b200 as p
    assert p._cabi.device_info()["cc"] == (9, 0)
    return p


@functools.lru_cache(maxsize=None)
def _corpus():
    return dict(ic.corpus())


def _routed(streams, bounds=None):
    from new_bloom_filter_repo_b200 import deflate
    return deflate.decompress_routed(streams, bounds)


def _batch(streams, bounds, capacity):
    """One direct rbf_zlib_decompress_batch call -> (out, offsets, on_device)."""
    from new_bloom_filter_repo_b200 import _cabi
    n = len(streams)
    views = [np.frombuffer(s, dtype=np.uint8) for s in streams]
    srcs = (C.c_void_p * n)(*[v.ctypes.data if v.size else None for v in views])
    lens = np.array([v.size for v in views], dtype=np.uint64)
    bnd = np.array(bounds, dtype=np.uint64)
    out = np.zeros(max(capacity, 1), dtype=np.uint8)
    offs = np.zeros(n + 1, dtype=np.uint64)
    ok = np.zeros(n, dtype=np.uint8)
    _cabi.check(_cabi.lib().rbf_zlib_decompress_batch(_cabi.ctx(), n, srcs, _cabi.ptr(lens), _cabi.ptr(bnd), _cabi.ptr(out),
                                                      capacity, _cabi.ptr(offs), _cabi.ptr(ok)), _cabi.ctx())
    return out, [int(x) for x in offs], [bool(x) for x in ok]


@gpu
@pytest.mark.parametrize("name", list(_corpus()))
def test_single_stream_routes_as_the_layout_says(pkg, name):
    s = _corpus()[name]
    got, dev = _routed([s])
    assert got == [zlib.decompress(s)], name
    v = im.verdict(s)
    assert dev == [v.on_device], (name, v.reason)


@gpu
def test_one_mixed_batch(pkg):
    """The whole corpus with the malformed streams, streams without the 78 9C header (some declined before the scan, among
    accepted ones), 78 9C streams shorter than 8 bytes and zlib.compress(b"") in one call, shuffled, then reversed."""
    text = ic._text(70000, 65)
    others = [zlib.compress(text, 9), zlib.compress(text, 1), zlib.compress(b"x", 9), b"", b"\x78", b"\x08\x1d" + text[:40],
              b"\x78\xda" + ic.layout(text)[2:]]
    short = [b"\x78\x9c", b"\x78\x9c\x03", b"\x78\x9c\x03\x00\x00\x00\x00", b"\x78\x9c\x00\x00\x00\xff\xff"]
    streams = list(_corpus().values()) + [s for _, s in _bad_streams()] + others + short + [zlib.compress(b"")]
    order = np.random.default_rng(66).permutation(len(streams))
    for idx in (list(order), list(order[::-1])):
        batch = [streams[i] for i in idx]
        bounds = [im.MAX_RATIO * len(s) for s in batch]
        want = [im.verdict(s, b).on_device for s, b in zip(batch, bounds)]
        capacity = sum(len(zlib.decompress(s)) for s, w in zip(batch, want) if w)
        out, offs, dev = _batch(batch, bounds, capacity)
        assert dev == want, [k for k, (a, b) in enumerate(zip(dev, want)) if a != b]
        assert offs[-1] == capacity
        for k, s in enumerate(batch):
            got = out[offs[k]:offs[k + 1]].tobytes()
            assert got == (zlib.decompress(s) if want[k] else b""), k
        assert 0 < sum(want) < len(batch)


@gpu
def test_bound_edge(pkg):
    """A bound equal to the inflated size is accepted, one byte less is declined (and zlib.decompress returns the bytes)."""
    for name in ("crafted-lit15-dist15-behind", "crafted-match-end-64k", "text-M8-L6", "split-3+0"):
        s = _corpus()[name]
        data = zlib.decompress(s)
        n = len(data)
        assert im.verdict(s, n).on_device and not im.verdict(s, n - 1).on_device, name
        assert im.cap(len(s), n) == im.cap(len(s), n - 1), name           # only the total decides
        assert _routed([s, s], [n, n - 1]) == ([data, data], [True, False]), name


@gpu
def test_output_capacity_edge(pkg):
    """out_capacity one byte short of the accepted total: the stream that no longer fits is declined, the ones before it keep
    their places, and an empty stream after it still fits."""
    names = ("crafted-dist-eq-out-behind", "crafted-repeats", "crafted-mixed-behind")
    streams = [_corpus()[k] for k in names] + [zlib.compress(b"")]
    datas = [zlib.decompress(s) for s in streams]
    bounds = [im.MAX_RATIO * len(s) for s in streams]
    total = sum(len(d) for d in datas)
    out, offs, dev = _batch(streams, bounds, total)
    assert dev == [True] * 4 and out[:total].tobytes() == b"".join(datas)
    out, offs, dev = _batch(streams, bounds, total - 1)
    assert dev == [True, True, False, True]
    n0, n1 = len(datas[0]), len(datas[1])
    assert offs == [0, n0, n0 + n1, n0 + n1, n0 + n1]
    assert out[:n0].tobytes() == datas[0] and out[n0:n0 + n1].tobytes() == datas[1]


@gpu
def test_candidate_cap_edge(pkg):
    """Under a bound of 5000 bytes the cap is min(2 * 1 + 8, len / 4 + 2) = 10 candidate starts: 9 planted markers (10 starts)
    are accepted, 10 (11 starts) are declined."""
    for n, accepted in ((9, True), (10, False)):
        s = ic.cap_stream(n)
        data = zlib.decompress(s)
        v = im.verdict(s, 5000)
        assert (v.ncand, v.cap, v.on_device) == (n + 1, 10, accepted), v.reason
        assert _routed([s], [5000]) == ([data], [accepted]), n


@gpu
def test_segment_starts_on_scan_job_edges(pkg):
    """Second segments starting at 2 + k * 8192 - 1, + 0 and + 1: the last position of a scan job, the first of the next, and
    one past; every one is found, in a batch of its own and in one together."""
    split = [(k, s) for k, s in _corpus().items() if k.startswith("split-")]
    assert len(split) == 6
    for k, s in split:
        starts = im.candidates(s)
        assert len(starts) == 2 and (starts[1] - 2) % ic.SCAN_CHUNK in (0, 1, ic.SCAN_CHUNK - 1), (k, starts)
    streams = [s for _, s in split]
    got, dev = _routed(streams)
    assert got == [zlib.decompress(s) for s in streams] and all(dev)


# ------------------------------------------------------------------ decompress_video
def _with_vz(payload, vz):
    from new_bloom_filter_repo_b200.improved_video_compressor import ImprovedVideoCompressor
    p = ImprovedVideoCompressor._parse_inter(payload)
    tail = len(payload) - len(p.vz)
    return bytes(payload[:tail - 8]) + struct.pack("<II", len(vz), p.vcount) + vz


def _in_layout(values, bound):
    """values as a zlib-written stream the device takes (the first setting that gives one)."""
    for level, strategy in ((6, zlib.Z_DEFAULT_STRATEGY), (9, zlib.Z_DEFAULT_STRATEGY), (1, zlib.Z_HUFFMAN_ONLY),
                            (6, zlib.Z_RLE), (6, zlib.Z_FILTERED)):
        s = ic.layout(values, level, 8, strategy)
        if im.verdict(s, bound).on_device:
            return s
    raise AssertionError("no zlib setting writes these values in the layout")


@gpu
def test_decompress_video_routes_zlib_layout_groups(pkg, monkeypatch):
    """A GPU-coded file with every inter value stream rewritten by zlib in the segment layout decodes losslessly without
    zlib.decompress seeing a value stream.  With a 78 DA stream in group 0 and a plain level-6 78 9C stream (BFINAL 1, declined)
    in group 1, exactly those two groups go to the host, group 2 stays on the device, and every frame is still lossless."""
    from new_bloom_filter_repo_b200 import deflate, fixed_video_compressor as fvc, improved_video_compressor as ivcmod
    frames = _frames(96, 128, 3, np.uint8, 13, 47, [0.3, 0.15, 0.4])
    comp, pls = _gpu_file(pkg, frames, 30, 4)                      # groups: frames 1-4, 5-8, 9-12
    parsed = [ivcmod.ImprovedVideoCompressor._parse_inter(p) for p in pls[1:]]
    values = [zlib.decompress(p.vz) for p in parsed]
    vz = [_in_layout(v, p.vcount * p.isz) for v, p in zip(values, parsed)]
    seen = []

    class Z:
        error = zlib.error

        @staticmethod
        def decompress(b, *a):
            seen.append(bytes(b))
            return zlib.decompress(b, *a)
    for mod in (ivcmod, fvc, deflate):
        monkeypatch.setattr(mod, "zlib", Z)

    def decode(streams):
        seen.clear()
        dec = comp.decompress_video(compressed_frames=[pls[0]] + [_with_vz(p, z) for p, z in zip(pls[1:], streams)])
        assert len(dec) == len(frames) and all(np.array_equal(_data(a), b) for a, b in zip(dec, frames))
        return {i for i, z in enumerate(streams) if z in seen}

    assert decode(vz) == set()
    mixed = list(vz)
    mixed[1] = zlib.compress(values[1], 9)                          # 78 DA: group 0 (inter frames 1-4)
    mixed[5] = zlib.compress(values[5], 6)                          # 78 9C, one final block: group 1 (frames 5-8)
    assert mixed[1][:2] == b"\x78\xda" and mixed[5][:2] == b"\x78\x9c" and not im.verdict(mixed[5]).on_device
    assert decode(mixed) == set(range(8))
