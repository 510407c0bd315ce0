"""GPU inflate of the device coder's zlib streams (csrc/rbf_inflate.cuh, rbf_zlib_decompress_batch, rbf_stream_inflate_values):
deflate.decompress_many returns exactly what zlib.decompress returns (or raises its error) for device streams, other zlib streams
and malformed ones, inflating the device streams on the GPU; decompress_video on files written with the GPU coder is lossless,
never calls zlib.decompress for value streams or keyframe blobs, and raises the host route's error for the first bad frame."""
import zlib

import numpy as np
import pytest

from tests.test_inflate_segment import _malformed, _text
from tests.util import synth_stream

gpu = pytest.mark.gpu
SEG = 65536
SIZES = (0, 1, 65535, 65536, 65537, 3 * 65536 + 1)


@pytest.fixture(scope="module")
def pkg():
    import new_bloom_filter_repo_b200 as p
    assert p._cabi.device_info()["cc"] == (9, 0)
    return p


def _deflate():
    from new_bloom_filter_repo_b200 import deflate
    return deflate


def _bufs():
    rng = np.random.default_rng(30)
    out = []
    for n in SIZES:
        out += [rng.integers(0, 256, n, dtype=np.uint8).tobytes(), _text(n, n),
                (np.cumsum(rng.integers(-3, 4, n // 2)) + 30000).astype(np.uint16).tobytes()]
    return out + [bytes(2 * SEG + 3)]


@gpu
def test_round_trips_alone_and_mixed(pkg):
    d = _deflate()
    bufs = _bufs()
    streams = d.compress_many(bufs)
    for b, s in zip(bufs, streams):
        got, dev = d.decompress_routed([s])
        assert got == [b] and dev == [True], len(b)
    got, dev = d.decompress_routed(streams, [len(b) for b in bufs])
    assert got == bufs and all(dev)
    assert d.decompress(streams[4]) == bufs[4]


@gpu
def test_stored_segments_holding_sync_markers(pkg):
    """Random data with 00 00 FF FF planted at offsets up to what the stream's bound allows (2 ceil(bound / 64 KiB) + 8 candidate
    starts), right before a segment boundary included: the false candidates are inflated and ignored, the chain's slots are
    gathered into place.  Beyond the allowance the stream goes to zlib.decompress."""
    rng = np.random.default_rng(31)
    b = bytearray(rng.integers(0, 256, 3 * SEG + 100, dtype=np.uint8).tobytes())
    plant = [0, 100, 4096, SEG - 5, SEG + 1, 2 * SEG - 5, 2 * SEG + 500, 3 * SEG - 5, 3 * SEG + 90]   # SEG - 5: up to the 2nd block
    for off in plant:
        b[off:off + 4] = b"\x00\x00\xff\xff"
    b = bytes(b)
    s = _deflate().compress(b)
    assert s.count(b"\x00\x00\xff\xff") == 4 + len(plant)        # four segments, each ending in a sync flush
    got, dev = _deflate().decompress_routed([s, s], [len(b), len(b)])
    assert got == [b, b] and dev == [True, True]
    more = bytearray(b)
    for off in rng.integers(0, len(b) - 4, 40):
        more[off:off + 4] = b"\x00\x00\xff\xff"
    s = _deflate().compress(bytes(more))
    got, dev = _deflate().decompress_routed([s], [len(b)])
    assert got == [bytes(more)] and dev == [False]


@gpu
def test_other_zlib_streams(pkg):
    data = _text(200000, 3)
    for level in (0, 1, 6, 9):
        z = zlib.compress(data, level)
        got, dev = _deflate().decompress_routed([z])
        assert got == [data] and dev == [False], level
    assert zlib.compress(data, 6)[:2] == b"\x78\x9c"


def _wrap(seg: bytes, data: bytes = b"") -> bytes:
    return b"\x78\x9c" + seg + b"\x03\x00" + zlib.adler32(data).to_bytes(4, "big")


def _bad_streams():
    text = _text(150000, 7)
    s = _deflate().compress(text)
    cases = [(n, _wrap(seg)) for n, seg in _malformed() if not n.startswith("dyn-cut-") or int(n[8:]) % 37 == 0]
    cases += [("cut-%d" % k, s[:k]) for k in (2, 3, 10, len(s) // 2, len(s) - 7, len(s) - 6, len(s) - 1)]
    cases += [("bad-adler", s[:-1] + bytes([s[-1] ^ 1])), ("after-trailer", s + b"\x00"), ("after-trailer-2", s + s)]
    cases += [("bad-03", s[:-6] + b"\x03\x01" + s[-4:]), ("flip-mid", s[:5000] + bytes([s[5000] ^ 0x10]) + s[5001:])]
    return cases


@gpu
def test_malformed_streams_match_zlib(pkg):
    for name, s in _bad_streams():
        try:
            want = ("ok", zlib.decompress(s))
        except zlib.error as e:
            want = ("error", str(e))
        try:
            got = ("ok", _deflate().decompress(s))
        except zlib.error as e:
            got = ("error", str(e))
        assert got == want, name
        if name.startswith("after-trailer"):                        # zlib.decompress ignores them; the GPU declines the stream
            assert _deflate().decompress_routed([s])[1] == [False], name
    with pytest.raises(zlib.error, match="incorrect data check"):
        _deflate().decompress(dict(_bad_streams())["bad-adler"])


# ------------------------------------------------------------------ FrameStream.apply_chain(inflated=...)
@gpu
def test_apply_chain_reads_inflated_values_once(pkg):
    """The values inflate_values placed serve one apply_chain(inflated=...): asking for more bytes than were placed raises and
    leaves them in place, a valid call reconstructs the frames that values= gives with the same bytes, and a second call raises."""
    from tests.test_gpu_motion import _raw_slots
    h, w, ch, cnt = 48, 40, 3, 4
    n = h * w
    rng = np.random.default_rng(44)
    masks = [(rng.random(n) < p).astype(np.uint8) for p in (0.3, 0.0, 1.0, 0.05)]
    vals = [rng.integers(0, 256, int(m.sum()) * ch).astype(np.uint8) for m in masks]
    nbytes = [v.nbytes for v in vals]
    modes = [0, 1, 0, 1]
    base = rng.integers(0, 256, (h, w, ch)).astype(np.uint8)
    st = pkg.FrameStream(h, w, ch, np.uint8, max_frames=cnt + 1, max_pairs=cnt, k1_only=True)
    try:
        _, ones = st.decode_masks(_raw_slots(masks, n), np.zeros((cnt, 0), np.uint8), [0] * cnt, [0] * cnt, [0.0] * cnt, [1] * cnt)
        lens, ok = st.inflate_values(_deflate().compress_many([v.tobytes() for v in vals]), nbytes)
        assert ok.all() and list(lens) == nbytes
        with pytest.raises(pkg.RbfError):
            st.apply_chain(0, inflated=nbytes[:-1] + [nbytes[-1] + 1], modes=modes)
        st.upload(base, first=0)
        applied = st.apply_chain(0, inflated=nbytes, modes=modes)
        got = st.download_batch(1, cnt)
        with pytest.raises(pkg.RbfError):
            st.apply_chain(0, inflated=nbytes, modes=modes)
        st.upload(base, first=0)
        assert list(applied) == list(st.apply_chain(0, vals, modes=modes)) == list(ones)
        assert np.array_equal(got, st.download_batch(1, cnt))
        with pytest.raises(ValueError):
            st.apply_chain(0, vals, inflated=nbytes)
    finally:
        st.close()


# ------------------------------------------------------------------ decompress_video
def _frames(h, w, ch, dtype, nfr, seed, p_seq):
    f = synth_stream(h, w, nfr, seed, p_seq, dtype)
    return [np.ascontiguousarray(x[..., 0]) if ch == 1 else x for x in f]


def _gpu_file(pkg, frames, ki, bs, coding="plain", yuv=False):
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=ki, batch_size=bs, use_direct_yuv=yuv)
    comp.entropy_coder = "gpu"
    comp.value_coding = coding
    src = [pkg.YUVFrame(f) for f in frames] if yuv else list(frames)
    comp.compress_video(src, input_color_space="YUV" if yuv else "BGR")
    return comp, list(comp._last_compressed_frames)


def _data(f):
    return np.asarray(f.data if hasattr(f, "yuv_info") else f)


@gpu
@pytest.mark.parametrize("coding", ["plain", "adaptive", "motion"])
@pytest.mark.parametrize("h,w,ch,dtype,yuv,nfr,ki,bs", [
    (72, 88, 3, np.uint8, True, 9, 30, 4),      # YUV444, groups of 4 (longer than, and a last one shorter)
    (64, 96, 3, np.uint16, False, 7, 30, 6),    # BGR 16-bit, one group equal to the run
    (80, 64, 1, np.uint8, False, 6, 3, 1),      # 1-channel, groups of one frame, two keyframes
    (48, 40, 1, np.uint16, False, 5, 30, 8),
])
def test_gpu_coded_files_round_trip(pkg, coding, h, w, ch, dtype, yuv, nfr, ki, bs):
    frames = _frames(h, w, ch, dtype, nfr, 41, [0.04, 0.2, 0.01])
    comp, pls = _gpu_file(pkg, frames, ki, bs, coding, yuv)
    dec = comp.decompress_video(compressed_frames=pls)
    assert len(dec) == nfr
    for a, b in zip(dec, frames):
        assert np.array_equal(_data(a), b)
    if yuv:
        ref = comp.compressor.decompress_frame(pls[0])
        assert type(dec[0]) is type(ref) and ref.yuv_info["format"] == dec[0].yuv_info["format"]
        for k in ("y_plane", "u_plane", "v_plane"):
            assert np.array_equal(ref.yuv_info[k], dec[0].yuv_info[k])


@gpu
def test_4k_gop_of_30(pkg):
    frames = _frames(2160, 3840, 3, np.uint8, 30, 42, [0.01, 0.05, 0.15, 0.30])
    comp, pls = _gpu_file(pkg, frames, 30, 30, yuv=True)
    dec = comp.decompress_video(compressed_frames=pls)
    assert all(np.array_equal(_data(a), b) for a, b in zip(dec, frames))


@gpu
def test_values_and_keyframes_never_reach_zlib(pkg, monkeypatch):
    """Per group the values go up compressed: h2d differs from the host route's by exactly the inflated minus the compressed value
    bytes.  zlib.decompress never sees a value stream or a keyframe blob."""
    from new_bloom_filter_repo_b200 import _cabi, deflate, fixed_video_compressor as fvc, improved_video_compressor as ivcmod
    frames = _frames(256, 320, 3, np.uint8, 8, 43, [0.3, 0.2])
    comp, pls = _gpu_file(pkg, frames, 30, 7, yuv=True)
    inter = [ivcmod.ImprovedVideoCompressor._parse_inter(p) for p in pls[1:]]
    watched = {bytes(p.vz) for p in inter} | {bytes(b) for b, _ in fvc.FixedVideoCompressor.keyframe_blobs(pls[0])}
    seen = []

    class Z:
        error = zlib.error

        @staticmethod
        def decompress(b, *a):
            seen.append(bytes(b) in watched)
            return zlib.decompress(b, *a)
    for mod in (ivcmod, fvc, deflate):
        monkeypatch.setattr(mod, "zlib", Z)
    L, ctx = _cabi.lib(), _cabi.ctx()

    def h2d_of_decode():
        L.rbf_reset_counters(ctx)
        dec = comp.decompress_video(compressed_frames=pls)
        assert all(np.array_equal(_data(a), b) for a, b in zip(dec, frames))
        return L.rbf_get_counter(ctx, b"h2d_bytes")
    h2d = h2d_of_decode()
    assert not any(seen)
    with monkeypatch.context() as m:
        _host_route(m)
        h2d_host = h2d_of_decode()
    vz = sum(len(p.vz) for p in inter)
    inflated = sum(p.vcount * p.isz for p in inter)
    assert inflated != vz and h2d_host - h2d == inflated - vz, (h2d, h2d_host, vz, inflated)


def _host_route(monkeypatch):
    """The route files of the default coder take: every value stream inflated with zlib.decompress on the host."""
    from new_bloom_filter_repo_b200 import improved_video_compressor as ivcmod

    def host(st, jobs, pool):
        for j in jobs:
            if j.p is not None and j.values is None:
                j.values = pool.submit(zlib.decompress, j.p.vz)
    monkeypatch.setattr(ivcmod.ImprovedVideoCompressor, "_inflate_group", staticmethod(host))


def _outcome(comp, pls):
    try:
        return ("ok", [_data(f).tobytes() for f in comp.decompress_video(compressed_frames=pls)])
    except Exception as e:
        return (type(e), str(e))


@gpu
def test_error_order_matches_host_route(pkg, monkeypatch):
    from tests.test_gpu_decode_groups import _corrupt
    frames = _frames(64, 64, 3, np.uint8, 8, 29, [0.05, 0.02])
    comp, pls = _gpu_file(pkg, frames, 30, 7)
    from new_bloom_filter_repo_b200 import improved_video_compressor as ivcmod
    p4 = ivcmod.ImprovedVideoCompressor._parse_inter(pls[4])
    tail = len(pls[4]) - len(p4.vz)
    bad_vz = pls[4][:tail + 40] + bytes([pls[4][tail + 40] ^ 0x55]) + pls[4][tail + 41:]
    cases = [[(at, kind)] for kind in ("ones+1", "short wlen", "shape", "wlen 0") for at in (1, 4, 7)]
    cases += [[(3, "short wlen"), (5, "shape")], [(3, "shape"), (5, "short wlen")], [(3, "ones+1"), (5, "short wlen")],
              [(3, "short wlen"), (5, "ones+1")], [(4, "vz")], [(2, "shape"), (4, "vz")], [(4, "vz"), (6, "shape")]]
    runs = []
    for case in cases:
        bad = list(pls)
        for at, kind in case:
            bad[at] = bad_vz if kind == "vz" else _corrupt(pls[at], kind)
        runs.append(bad)
    device = [_outcome(comp, bad) for bad in runs]
    with monkeypatch.context() as m:
        _host_route(m)
        host = [_outcome(comp, bad) for bad in runs]
    for case, a, b in zip(cases, device, host):
        assert a[0] != "ok" and a == b, case
