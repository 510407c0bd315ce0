"""VideoReader decodes a frame range from the last keyframe at or before it, reading, parsing and inflating nothing outside that
span, and downloads only the frames asked for (or copies them into device memory).  Every read is compared with decompress_video
on the same payloads: frames, dtype, shape, YUVFrame-ness and YUV planes, and the error of the first bad frame."""
import ctypes as C
import os
import struct

import numpy as np
import pytest

from tests.util import synth_stream

try:        # at collection, before a test makes the library dlopen libnccl with RTLD_GLOBAL: torch must bind its own NCCL first
    import torch
except ImportError:
    torch = None

gpu = pytest.mark.gpu

P_MIX = [0.05, 0.0, 0.4, 0.01]           # coded, unchanged (raw, empty mask), dense (raw), sparse coded


@pytest.fixture(scope="module")
def pkg():
    import new_bloom_filter_repo_b200 as p
    assert p._cabi.device_info()["cc"] == (9, 0)
    return p


def _ivc():
    from new_bloom_filter_repo_b200 import improved_video_compressor as ivcmod
    return ivcmod


def _counter(pkg, key):
    return pkg._cabi.lib().rbf_get_counter(pkg._cabi.ctx(), key.encode())


def _frames(h, w, ch, dtype, nfr, seed, p_seq=P_MIX):
    f = synth_stream(h, w, nfr, seed, p_seq, dtype)
    return [np.ascontiguousarray(x[..., 0]) if ch == 1 else x for x in f]


def _pan(h, w, ch, dtype, nfr, seed):
    """A random texture panned 3 px right and 2 px up per frame, with the synth_stream changes of P_MIX on top."""
    hi = 256 if dtype == np.uint8 else 65536
    big = np.random.default_rng(seed).integers(0, hi, (h + 2 * nfr, w + 3 * nfr, ch)).astype(dtype)
    out = []
    for t in range(nfr):
        f = big[2 * t:2 * t + h, 3 * (nfr - t):3 * (nfr - t) + w].astype(np.int64)
        r = np.random.default_rng(seed + t)
        f[r.random((h, w)) < P_MIX[t % len(P_MIX)]] += hi // 4
        f = (f % hi).astype(dtype)
        out.append(np.ascontiguousarray(f[..., 0] if ch == 1 else f))
    return out


def _reference_frames(pkg):
    """Reference mode with chroma-only changes in frames 3 and 7: both become keyframes in the middle of the run."""
    f = synth_stream(96, 80, 12, 13, [0.05, 0.02])
    y, x = np.argwhere((f[3, ..., 0] == f[2, ..., 0]) & (f[7, ..., 0] == f[6, ..., 0]))[0]
    f[3:, y, x, 2] ^= 1
    f[7:, y, x, 2] ^= 1
    return [pkg.YUVFrame(a) for a in f]


# name: (frames maker, keyframe_interval, batch_size, entropy coder, value coding, inter_frame_mode, yuv)
CONFIGS = {
    "yuv444-ki30-bs4": (lambda pkg: [pkg.YUVFrame(f) for f in _frames(37, 53, 3, np.uint8, 12, 5)], 30, 4, "zlib", "plain",
                        "lossless", True),                   # one run of 11 in groups of 4, 4, 3
    "bgr-ki6-bs5": (lambda pkg: _frames(64, 64, 3, np.uint8, 12, 6), 6, 5, "gpu", "adaptive", "lossless", False),  # runs of one group
    "gray-bs1": (lambda pkg: _frames(37, 53, 1, np.uint8, 13, 7), 30, 1, "zlib", "adaptive", "lossless", False),
    "gray16-ki5-bs3-motion": (lambda pkg: _pan(64, 64, 1, np.uint16, 12, 8), 5, 3, "gpu", "motion", "lossless", False),
    "bgr-motion-ki30-bs4": (lambda pkg: _pan(48, 64, 3, np.uint8, 12, 9), 30, 4, "zlib", "motion", "lossless", False),
    "ki1": (lambda pkg: _frames(37, 53, 3, np.uint8, 12, 10), 1, 4, "zlib", "plain", "lossless", False),
    "reference-fallbacks": (_reference_frames, 30, 3, "gpu", "plain", "reference", True),
}


def _compress(pkg, name, path=None):
    make, ki, bs, coder, vc, mode, yuv = CONFIGS[name]
    frames = make(pkg)
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=ki, batch_size=bs)
    comp.entropy_coder, comp.value_coding, comp.inter_frame_mode = coder, vc, mode
    if mode == "reference":
        comp.inter_frame_threshold = 3.0
    comp.compress_video(list(frames), output_path=path, input_color_space="YUV" if yuv else "BGR")
    return comp, list(comp._last_compressed_frames)


def _same(got, ref, where=""):
    assert len(got) == len(ref), where
    for i, (g, r) in enumerate(zip(got, ref)):
        gd, rd = (g.data if hasattr(g, "yuv_info") else g), (r.data if hasattr(r, "yuv_info") else r)
        assert hasattr(g, "yuv_info") == hasattr(r, "yuv_info"), (where, i)
        assert gd.dtype == rd.dtype and gd.shape == rd.shape, (where, i)
        assert np.array_equal(gd, rd), (where, i)
        if hasattr(r, "yuv_info"):
            for name in ("y_plane", "u_plane", "v_plane"):
                assert np.array_equal(g.yuv_info[name], r.yuv_info[name]), (where, i, name)


class Recorder:
    """A payload sequence that records the indices it is asked for."""

    def __init__(self, payloads):
        self.payloads, self.asked = payloads, []

    def __len__(self):
        return len(self.payloads)

    def __getitem__(self, i):
        self.asked.append(i)
        return self.payloads[i]


def _key_before(payloads, start):
    keys = [i for i, p in enumerate(payloads) if not _ivc()._is_inter(p)]
    return max([k for k in keys if k <= start], default=0)


# ------------------------------------------------------------------ 1. every range, from the payloads and from the file
@gpu
@pytest.mark.parametrize("name", list(CONFIGS))
def test_every_range(pkg, tmp_path, name):
    path = str(tmp_path / "v.bfvc")
    comp, pls = _compress(pkg, name, path)
    ref = comp.decompress_video(compressed_frames=pls)
    _same(comp.decompress_video(input_path=path), ref, "file")
    F = len(pls)
    vm = [_ivc().ImprovedVideoCompressor._parse_inter(p).vmode for p in pls if _ivc()._is_inter(p)]
    if CONFIGS[name][4] == "motion":
        assert 2 in vm, vm                                 # some pairs are coded against the motion-compensated frame
    if CONFIGS[name][5] == "reference":
        assert not _ivc()._is_inter(pls[3]) and not _ivc()._is_inter(pls[7])
    with pkg.VideoReader(pls, comp) as r1, pkg.VideoReader(path, comp) as r2:
        assert len(r1) == len(r2) == F and r1.keyframes == r2.keyframes
        for start in range(F):
            for stop in range(start + 1, F + 1):
                _same(r1.read(start, stop), ref[start:stop], ("list", start, stop))
                _same(r2.read(start, stop), ref[start:stop], ("file", start, stop))


# ------------------------------------------------------------------ 2. indexing
@pytest.fixture(scope="module")
def gop(pkg):
    comp, pls = _compress(pkg, "bgr-ki6-bs5")
    return comp, pls, comp.decompress_video(compressed_frames=pls)


@gpu
def test_indexing(pkg, gop):
    comp, pls, ref = gop
    F = len(pls)
    r = pkg.VideoReader(pls, comp)
    assert len(r) == F == 12 and r.keyframes == [0, 6]
    for i in range(-F, F):
        _same([r[i]], [ref[i]], i)
    for a, b in [(0, 12), (3, 9), (5, 7), (-4, None), (None, 2), (7, 3), (11, 40)]:
        _same(r[a:b], ref[a:b], (a, b))
    assert r.read(4, 4) == [] and r[4:4] == []
    for bad in (F, -F - 1):
        with pytest.raises(IndexError):
            r[bad]
    for a, b in [(-1, 2), (3, 13), (5, 4)]:
        with pytest.raises(IndexError):
            r.read(a, b)
    with pytest.raises(ValueError, match="step"):
        r[0:6:2]
    r.close()


# ------------------------------------------------------------------ 3. laziness
@gpu
def test_read_touches_exactly_the_span(pkg, gop):
    comp, pls, ref = gop
    rec = Recorder(pls)
    r = pkg.VideoReader(rec, comp)
    for a, b in [(0, 1), (2, 5), (5, 7), (6, 7), (7, 12), (11, 12), (3, 12)]:
        rec.asked = []
        _same(r.read(a, b), ref[a:b], (a, b))
        k = _key_before(pls, a)
        assert sorted(rec.asked) == list(range(k, b)), (a, b, rec.asked)
    r.close()


def _overwrite(path, keep, rng):
    """Every payload of the file outside `keep` replaced by as many random bytes."""
    b = bytearray(open(path, "rb").read())
    pos, i = 8, 0
    while pos < len(b):
        (n,) = struct.unpack_from("<I", b, pos)
        if i not in keep:
            b[pos + 4:pos + 4 + n] = rng.integers(0, 256, n).astype(np.uint8).tobytes()
        pos, i = pos + 4 + n, i + 1
    open(path, "wb").write(bytes(b))


@gpu
@pytest.mark.parametrize("a,b", [(0, 3), (2, 6), (6, 7), (8, 12), (4, 10)])
def test_payloads_outside_the_span_may_be_anything(pkg, tmp_path, a, b):
    path = str(tmp_path / "v.bfvc")
    comp, pls = _compress(pkg, "bgr-ki6-bs5", path)
    ref = comp.decompress_video(compressed_frames=pls)
    _overwrite(path, set(range(_key_before(pls, a), b)), np.random.default_rng(a * 13 + b))
    with pkg.VideoReader(path, comp) as r:
        _same(r.read(a, b), ref[a:b], (a, b))


def _corrupt(pl, kind, ch=3):
    """The corruptions of test_gpu_decode_groups: a popcount that disagrees, a witness cut in half, a wrong shape, no witness."""
    ivcmod = _ivc()
    base, hdr = len(ivcmod._INTER_TAG), struct.calcsize("<IIIBB")
    off = {"h": base, "wlen": base + hdr + 12, "ones": base + hdr + 16}
    b = bytearray(pl)
    if kind == "ones+1":
        import zlib
        struct.pack_into("<Q", b, off["ones"], struct.unpack_from("<Q", b, off["ones"])[0] + 1)
        p = ivcmod.ImprovedVideoCompressor._parse_inter(pl)
        vz = zlib.compress(zlib.decompress(p.vz)[:p.vcount] + bytes(ch), 9)
        tail = len(pl) - len(p.vz) - 8
        return bytes(b[:tail]) + struct.pack("<II", len(vz), p.vcount + ch) + vz
    if kind == "short wlen":
        struct.pack_into("<I", b, off["wlen"], struct.unpack_from("<I", b, off["wlen"])[0] // 2)
    elif kind == "shape":
        struct.pack_into("<I", b, off["h"], struct.unpack_from("<I", b, off["h"])[0] + 1)
    elif kind == "wlen 0":
        struct.pack_into("<I", b, off["wlen"], 0)
    return bytes(b)


@pytest.fixture(scope="module")
def coded_gop(pkg):
    frames = _frames(64, 64, 3, np.uint8, 8, 29, [0.05, 0.02])
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=30, batch_size=7)
    comp.compress_video(list(frames))
    pls = list(comp._last_compressed_frames)
    assert all(_ivc()._is_inter(p) for p in pls[1:])
    return comp, pls


def _exc(fn):
    try:
        fn()
    except Exception as e:
        return type(e), str(e)
    return None


@gpu
@pytest.mark.parametrize("kind", ["ones+1", "short wlen", "shape", "wlen 0"])
@pytest.mark.parametrize("at", [1, 4, 7])
def test_corrupt_frame_in_the_span_raises_as_decompress_video(pkg, tmp_path, coded_gop, kind, at):
    comp, pls = coded_gop
    bad = list(pls)
    bad[at] = _corrupt(pls[at], kind)
    want = _exc(lambda: comp.decompress_video(compressed_frames=bad))
    assert want is not None
    path = str(tmp_path / "bad.bfvc")
    with open(path, "wb") as fh:
        fh.write(b"BFVC" + struct.pack("<I", len(bad)) + b"".join(struct.pack("<I", len(p)) + p for p in bad))
    for src in (bad, path):
        with pkg.VideoReader(src, comp) as r:
            for a, b in [(0, 8), (at, at + 1), (max(1, at - 1), 8)]:
                assert _exc(lambda: r.read(a, b)) == want, (src is path, a, b)
            if at > 1:                                     # frames before it are not affected
                _same(r.read(0, at), comp.decompress_video(compressed_frames=pls)[:at])


@gpu
def test_inter_frame_without_a_keyframe_raises(pkg, coded_gop):
    comp, pls = coded_gop
    with pkg.VideoReader(pls[3:], comp) as r:
        with pytest.raises(ValueError, match="inter frame without a preceding frame"):
            r.read(2, 4)


@gpu
def test_bad_file_fails_at_open_as_decompress_video(pkg, tmp_path, coded_gop):
    comp, pls = coded_gop
    good = b"BFVC" + struct.pack("<I", len(pls)) + b"".join(struct.pack("<I", len(p)) + p for p in pls)
    cases = {"magic": b"BFVD" + good[4:], "table": good[:8 + 4 + len(pls[0]) + 4 + len(pls[1]) + 2], "count": good[:6],
             "empty": b"BFVC" + struct.pack("<I", 0)}
    for name, data in cases.items():
        path = str(tmp_path / (name + ".bfvc"))
        open(path, "wb").write(data)
        want = _exc(lambda: comp.decompress_video(input_path=path))
        assert want is not None and want[0] in (ValueError, struct.error), name
        assert _exc(lambda: pkg.VideoReader(path, comp)) == want, name
    with pytest.raises(ValueError, match="No compressed frames provided"):
        pkg.VideoReader([], comp)
    # a last payload cut short by the end of the file is handed on as short as decompress_video reads it
    path = str(tmp_path / "short.bfvc")
    open(path, "wb").write(good[:-5])
    want = _exc(lambda: comp.decompress_video(input_path=path))
    with pkg.VideoReader(path, comp) as r:
        assert _exc(lambda: r.read(0, len(pls))) == want
        _same(r.read(0, len(pls) - 1), comp.decompress_video(compressed_frames=pls)[:-1])


# ------------------------------------------------------------------ 4. downloads
@pytest.fixture(scope="module")
def hd(pkg):
    frames = [pkg.YUVFrame(f) for f in _frames(1080, 1920, 3, np.uint8, 12, 3)]
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=30, batch_size=5)
    comp.compress_video(list(frames), input_color_space="YUV")
    pls = list(comp._last_compressed_frames)
    return comp, pls, comp.decompress_video(compressed_frames=pls), frames[0].data.nbytes


@gpu
@pytest.mark.parametrize("a", [0, 5, 6, 7, 11])              # groups of 5 from frame 1: frames 1-5, 6-10, 11
def test_read_downloads_the_span_only(pkg, hd, a):
    comp, pls, ref, fb = hd
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    with pkg.VideoReader(pls, comp) as r:
        for b in sorted({a + 1, min(12, a + 3), 12}):
            L.rbf_reset_counters(ctx)
            got = r.read(a, b)
            d2h = _counter(pkg, "d2h_bytes")
            _same(got, ref[a:b], (a, b))
            inter = sum(1 for i in range(a, b) if i)       # the keyframe is built on the host
            assert inter * fb <= d2h < inter * fb + fb, (a, b, d2h)


# ------------------------------------------------------------------ 5. device output
class _CAI:
    """A torch tensor's memory behind a v3 __cuda_array_interface__ that names the stream its pending work runs on."""

    def __init__(self, t, stream):
        self.t = t
        self.__cuda_array_interface__ = dict(t.__cuda_array_interface__, version=3, stream=stream)


def _torch():
    if torch is None or not torch.cuda.is_available():
        pytest.skip("torch with CUDA is needed for device buffers")
    return torch


@gpu
@pytest.mark.parametrize("name", ["yuv444-ki30-bs4", "bgr-ki6-bs5", "gray16-ki5-bs3-motion", "ki1", "reference-fallbacks"])
def test_read_into_device_memory(pkg, name):
    torch = _torch()
    comp, pls = _compress(pkg, name)
    ref = comp.decompress_video(compressed_frames=pls)
    F = len(pls)
    keys = [i for i, p in enumerate(pls) if not _ivc()._is_inter(p)]
    spans = {(0, F), (0, 1), (1, 4), (F - 1, F), (2, F - 1)} | {(k, min(F, k + 3)) for k in keys} | \
            {(max(0, k - 2), min(F, k + 2)) for k in keys if k}
    data = [np.asarray(f.data if hasattr(f, "yuv_info") else f) for f in ref]
    tdt = torch.uint8 if data[0].dtype == np.uint8 else torch.int16
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    fb = data[0].nbytes
    with pkg.VideoReader(pls, comp) as r:
        for a, b in sorted(spans):
            L.rbf_reset_counters(ctx)
            r.read(a, b)
            d2h_host = _counter(pkg, "d2h_bytes")
            out = torch.empty((b - a,) + data[0].shape, dtype=tdt, device="cuda")
            if tdt == torch.int16:                          # torch has no uint16 interface: the same bytes under a u16 typestr
                out = _CAI(out, 1)
                out.__cuda_array_interface__["typestr"] = "<u2"
            L.rbf_reset_counters(ctx)
            assert r.read(a, b, out=out) is out
            d2h, d2d = _counter(pkg, "d2h_bytes"), _counter(pkg, "d2d_bytes")
            t = out.t if isinstance(out, _CAI) else out
            got = t.cpu().numpy().view(data[0].dtype)
            for i in range(a, b):
                assert np.array_equal(got[i - a], data[i]), (a, b, i)
            # the host read's downloads but its inter frames: per-pair counts (< one frame in all) and, for the GPU coder, the
            # keyframe blobs inflated on the device for the host-side keyframe build
            inter = sum(1 for i in range(a, b) if _ivc()._is_inter(pls[i]))
            assert d2h == d2h_host - inter * fb, (a, b, d2h, d2h_host)
            if CONFIGS[name][3] == "zlib":
                assert d2h < fb, (a, b, d2h)
            assert d2d == fb * (b - a), (a, b, d2d)         # keyframes reach out through a slot too


@gpu
def test_device_output_waits_for_the_producer_stream(pkg, gop):
    torch = _torch()
    comp, pls, ref = gop
    side = torch.cuda.Stream()
    shape = (12,) + ref[0].shape
    with pkg.VideoReader(pls, comp) as r:
        for _ in range(2):
            with torch.cuda.stream(side):
                out = torch.empty(shape, dtype=torch.uint8, device="cuda")
                torch.cuda._sleep(50_000_000)               # keep the side stream busy so the fill lands late
                out.fill_(0xFF)
            r.read(0, 12, out=_CAI(out, side.cuda_stream))
            side.synchronize()
            got = out.cpu().numpy()
            for i in range(12):
                assert np.array_equal(got[i], np.asarray(ref[i])), i


@gpu
def test_bad_device_output_raises_before_any_launch(pkg, gop):
    torch = _torch()
    comp, pls, ref = gop
    other = _compress(pkg, "gray-bs1")[1]
    mixed = pls[:6] + [other[0]] + other[1:3]                # a 64x64 BGR GOP, then a 37x53 gray keyframe and its inter frames
    shape = ref[0].shape
    good = torch.empty((3,) + shape, dtype=torch.uint8, device="cuda")
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    r, rm = pkg.VideoReader(pls, comp), pkg.VideoReader(mixed, comp)
    cases = [(r, 2, 5, torch.empty((4,) + shape, dtype=torch.uint8, device="cuda")),
             (r, 2, 5, torch.empty((3,) + shape[:2], dtype=torch.uint8, device="cuda")),
             (r, 2, 5, torch.empty((3,) + shape, dtype=torch.int32, device="cuda")),
             (r, 2, 5, torch.empty((3,) + shape, dtype=torch.float32, device="cuda")),
             (r, 2, 5, torch.empty((3,) + shape[:2] + (6,), dtype=torch.uint8, device="cuda")[..., ::2]),
             (r, 2, 5, torch.empty((3,) + shape, dtype=torch.uint8)),
             (r, 2, 5, np.empty((3,) + shape, np.uint8)),
             (rm, 4, 8, good.new_empty((4,) + shape))]
    for rd, a, b, out in cases:
        L.rbf_reset_counters(ctx)
        with pytest.raises(ValueError):
            rd.read(a, b, out=out)
        assert _counter(pkg, "kernel_launches") == 0 and _counter(pkg, "d2d_bytes") == 0
    r.read(2, 5, out=good)                                  # and the reader still works
    assert np.array_equal(good.cpu().numpy(), np.stack([np.asarray(f) for f in ref[2:5]]))
    r.close()
    rm.close()


# ------------------------------------------------------------------ 6. iteration
@gpu
def test_iteration(pkg, gop, monkeypatch):
    comp, pls, ref = gop
    opened = set()
    orig_init, orig_close = pkg.FrameStream.__init__, pkg.FrameStream.close

    def init(self, *a, **k):
        orig_init(self, *a, **k)
        opened.add(id(self))

    def close(self):
        opened.discard(id(self))
        orig_close(self)
    monkeypatch.setattr(pkg.FrameStream, "__init__", init)
    monkeypatch.setattr(pkg.FrameStream, "close", close)
    rec = Recorder(pls)
    r = pkg.VideoReader(rec, comp)
    _same(list(r), ref)
    for _ in range(2):
        rec.asked = []
        it = iter(r)
        _same([next(it)], ref[:1])
        assert len(set(rec.asked)) <= 2 * comp.batch_size, rec.asked
        _same([next(it) for _ in range(6)], ref[1:7])
        assert opened
        if _ == 0:
            it.close()                                      # the generator closes its streams
            assert not opened
    for f in r:                                             # break out early, then close the reader
        break
    r.read(3, 9)
    r.close()
    assert not opened


# ------------------------------------------------------------------ 7. 4K
@gpu
def test_4k_seek_to_the_end_of_a_gop(pkg):
    frames = [pkg.YUVFrame(f) for f in _frames(2160, 3840, 3, np.uint8, 30, 9, [0.01, 0.05, 0.0, 0.4])]
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=30, batch_size=30)
    comp.compress_video(list(frames), input_color_space="YUV")
    pls = list(comp._last_compressed_frames)
    ref = comp.decompress_video(compressed_frames=pls)[29]
    fb = frames[0].data.nbytes
    with pkg.VideoReader(pls, comp) as r:
        pkg._cabi.lib().rbf_reset_counters(pkg._cabi.ctx())
        got = r.read(29, 30)
        d2h = _counter(pkg, "d2h_bytes")
    _same(got, [ref])
    assert fb <= d2h < 2 * fb, d2h


# ------------------------------------------------------------------ 8. the C ABI
@gpu
def test_copy_frames_c_abi(pkg):
    torch = _torch()
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    h, w, ch = 37, 53, 3
    st = pkg.FrameStream(h, w, ch, np.uint8, max_frames=5, max_pairs=4, k1_only=True)
    try:
        frames = np.random.default_rng(1).integers(0, 256, (5, h, w, ch)).astype(np.uint8)
        st.upload(frames)
        fb = h * w * ch
        for first, count in [(0, 5), (3, 4), (4, 5), (2, 1), (4, 1)]:   # wrap-around when first + count > 5
            out = torch.zeros((count, h, w, ch), dtype=torch.uint8, device="cuda")
            L.rbf_reset_counters(ctx)
            st.copy_frames(first, count, out.data_ptr(), out.numel(), 0)
            assert _counter(pkg, "d2d_bytes") == count * fb
            assert _counter(pkg, "d2h_bytes") == 0 and _counter(pkg, "h2d_bytes") == 0
            assert np.array_equal(out.cpu().numpy(), st.download_batch(first, count)), (first, count)
        dev = torch.zeros((5, h, w, ch), dtype=torch.uint8, device="cuda")
        host = np.zeros((5, h, w, ch), np.uint8)
        pinned = torch.zeros((5, h, w, ch), dtype=torch.uint8).pin_memory()
        bad = [(5, 1, dev.data_ptr(), dev.numel()), (0, 0, dev.data_ptr(), dev.numel()), (0, 6, dev.data_ptr(), 6 * fb),
               (0, 1, 0, dev.numel()), (0, 2, dev.data_ptr(), 2 * fb - 1), (0, 1, host.ctypes.data, host.nbytes),
               (0, 1, pinned.data_ptr(), pinned.numel())]
        for first, count, ptr, cap in bad:
            L.rbf_reset_counters(ctx)
            rc = L.rbf_stream_copy_frames(st._h, first, count, C.c_void_p(ptr or None), cap, 0)
            assert rc == -1, (first, count)                 # RBF_ERR_INVALID
            assert _counter(pkg, "d2d_bytes") == 0 and _counter(pkg, "kernel_launches") == 0
        assert not dev.any().item()
    finally:
        st.close()
