"""decompress_video decodes each run of inter frames in groups: one batched mask decode (rbf_stream_decode_masks), one chained
reconstruction sweep (rbf_stream_apply_chain, K4c) and one batched download per group.  The frames are compared with an
independent route -- the C oracle's BloomFilterCompressor.decompress of every mask and the Python oracle's _apply_frame_diff on
the previously decoded frame -- and the error of the first bad frame of a file must be the one a frame-by-frame decode raises."""
import struct
import zlib

import numpy as np
import pytest

from tests.util import synth_stream

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    import new_bloom_filter_repo_b200 as p
    assert p._cabi.device_info()["cc"] == (9, 0)
    return p


@pytest.fixture(scope="module")
def co():
    from oracle import c_oracle
    c_oracle.build()
    return c_oracle


def _ivc():
    from new_bloom_filter_repo_b200 import improved_video_compressor as ivcmod
    return ivcmod


def _independent_decode(co, payloads):
    """Frame by frame: keyframes with the CPU keyframe codec; inter frames with the C oracle's mask decode and the Python oracle's
    scatter on the previously decoded frame."""
    from new_bloom_filter_repo_b200.fixed_video_compressor import FixedVideoCompressor
    from oracle import rbf_oracle as po
    ivcmod = _ivc()
    out = []
    for c in payloads:
        if not c.startswith((ivcmod._INTER_TAG, ivcmod._INTER_TAG_V1)):
            f = FixedVideoCompressor(verbose=False).decompress_frame(c)
            out.append(np.asarray(f.data if hasattr(f, "yuv_info") else f))
            continue
        p = ivcmod.ImprovedVideoCompressor._parse_inter(c)
        n = p.h * p.w
        vals = np.frombuffer(zlib.decompress(p.vz), dtype=np.uint8 if p.isz == 1 else np.uint16)[:p.vcount]
        if p.raw:
            bits = bytes(p.mask_bytes) if p.v1 else zlib.decompress(p.mask_bytes)
            mask = np.unpackbits(np.frombuffer(bits, dtype=np.uint8))[:n]
        else:
            bm = np.unpackbits(np.frombuffer(p.mask_bytes, dtype=np.uint8))[:p.l]
            wt = np.unpackbits(np.frombuffer(p.witness_bytes, dtype=np.uint8))[:p.wlen]
            mask = co.decompress(bm, wt, n, p.k)
        prev = out[-1]
        m2 = mask.reshape(p.h, p.w)
        out.append(po.apply_frame_diff(prev, m2, vals) if prev.ndim == 3 else po.apply_frame_diff(prev[..., None], m2, vals)[..., 0])
    return out


def _frames(h, w, ch, dtype, nfr, seed, p_seq):
    f = synth_stream(h, w, nfr, seed, p_seq, dtype)
    if ch == 1:
        f = np.ascontiguousarray(f[..., 0])
    return [x for x in f]


def _compress(pkg, frames, ki, bs, coder="zlib", yuv=False, num_threads=None):
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=ki, batch_size=bs, num_threads=num_threads, use_direct_yuv=yuv)
    comp.entropy_coder = coder
    comp.compress_video(list(frames), input_color_space="YUV" if yuv else "BGR")
    return comp, list(comp._last_compressed_frames)


def _check_round_trip(pkg, co, comp, frames, payloads, yuv):
    dec = comp.decompress_video(compressed_frames=payloads)
    ref = _independent_decode(co, payloads)
    assert len(dec) == len(frames) == len(ref)
    for i, (d, r, f) in enumerate(zip(dec, ref, frames)):
        dd = d.data if hasattr(d, "yuv_info") else d
        assert hasattr(d, "yuv_info") == yuv, i
        assert dd.dtype == r.dtype and dd.shape == r.shape, i
        assert np.array_equal(dd, r), i
        assert np.array_equal(dd, np.asarray(f.data if hasattr(f, "yuv_info") else f)), i
        if yuv:
            for q, name in enumerate(("y_plane", "u_plane", "v_plane")):
                assert np.array_equal(d.yuv_info[name], dd[:, :, q]), (i, name)
    return dec


P_MIX = [0.05, 0.0, 0.4, 0.01]           # coded, unchanged (raw, empty mask), dense (raw), sparse coded


# (h, w, channels, dtype, yuv, frames, keyframe_interval, batch_size, coder): runs longer than a group, exactly one group, groups of 1
@gpu
@pytest.mark.parametrize("h,w,ch,dtype,yuv,nfr,ki,bs,coder", [
    (37, 53, 3, np.uint8, True, 12, 30, 4, "zlib"),        # YUV444: one run of 11 in groups of 4, 4, 3
    (64, 64, 3, np.uint8, False, 12, 6, 5, "gpu"),         # BGR: runs of 5 = exactly one group each
    (37, 53, 1, np.uint8, False, 7, 30, 1, "zlib"),        # groups of one
    (64, 64, 1, np.uint16, False, 11, 5, 3, "gpu"),
    (37, 53, 3, np.uint16, False, 10, 30, 7, "zlib"),
    (1080, 1920, 3, np.uint8, True, 8, 30, 3, "gpu"),
    (1080, 1920, 1, np.uint16, False, 6, 30, 30, "zlib"),
])
def test_round_trip_matches_independent_route(pkg, co, h, w, ch, dtype, yuv, nfr, ki, bs, coder):
    frames = _frames(h, w, ch, dtype, nfr, 5, P_MIX)
    if yuv:
        frames = [pkg.YUVFrame(f) for f in frames]
    comp, payloads = _compress(pkg, frames, ki, bs, coder, yuv)
    assert sum(p.startswith(_ivc()._INTER_TAG) for p in payloads) == nfr - (nfr + ki - 1) // ki
    _check_round_trip(pkg, co, comp, frames, payloads, yuv)


@gpu
def test_round_trip_4k_gop_of_30(pkg, co):
    frames = [pkg.YUVFrame(f) for f in _frames(2160, 3840, 3, np.uint8, 30, 9, [0.01, 0.05, 0.0, 0.4])]
    comp, payloads = _compress(pkg, frames, 30, 30, "zlib", True)
    _check_round_trip(pkg, co, comp, frames, payloads, True)


@gpu
def test_static_scene(pkg, co):
    f0 = _frames(64, 64, 3, np.uint8, 1, 3, [0.0])[0]
    frames = [f0.copy() for _ in range(9)]
    comp, payloads = _compress(pkg, frames, 30, 4)
    _check_round_trip(pkg, co, comp, frames, payloads, False)


@gpu
def test_rbf1_payload_inside_a_group(pkg, co):
    ivcmod = _ivc()
    frames = _frames(64, 64, 3, np.uint8, 7, 71, [0.05, 0.4, 0.05])
    comp, pls = _compress(pkg, frames, 30, 6)
    pos = len(ivcmod._INTER_TAG)
    p2 = pos + struct.calcsize("<IIIBB") + struct.calcsize("<dIIQ")
    raw_at = [i for i, pl in enumerate(pls) if i and struct.unpack_from("<IIIBB", pl, pos)[4] == 1]
    assert raw_at and 1 < raw_at[0] < 6
    i = raw_at[0]
    (bl,) = struct.unpack_from("<I", pls[i], p2)
    bits = zlib.decompress(pls[i][p2 + 4:p2 + 4 + bl])
    pls[i] = ivcmod._INTER_TAG_V1 + pls[i][pos:p2] + struct.pack("<I", len(bits)) + bits + pls[i][p2 + 4 + bl:]
    _check_round_trip(pkg, co, comp, frames, pls, False)


@gpu
def test_reference_mode_keyframe_fallbacks_inside_a_run(pkg, co):
    f = synth_stream(96, 80, 11, 13, [0.05, 0.02])
    y, x = np.argwhere((f[3, ..., 0] == f[2, ..., 0]) & (f[7, ..., 0] == f[6, ..., 0]))[0]
    f[3:, y, x, 2] ^= 1                                    # chroma-only changes in frames 3 and 7: the Y mask cannot carry them,
    f[7:, y, x, 2] ^= 1                                    # so both become keyframes in the middle of the run
    frames = [pkg.YUVFrame(a) for a in f]
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=30, batch_size=3)
    comp.inter_frame_mode = "reference"
    comp.inter_frame_threshold = 3.0
    stats = comp.compress_video(list(frames), input_color_space="YUV")
    pls = list(comp._last_compressed_frames)
    assert stats["keyframes"] == 3 and not pls[3].startswith(_ivc()._INTER_TAG) and not pls[7].startswith(_ivc()._INTER_TAG)
    _check_round_trip(pkg, co, comp, frames, pls, True)


# ------------------------------------------------------------------ errors: the first bad frame decides
_HDR = struct.calcsize("<IIIBB")


def _field_off(name):
    base = len(_ivc()._INTER_TAG)
    return {"h": base, "wlen": base + _HDR + 8 + 4, "ones": base + _HDR + 8 + 8}[name]


def _corrupt(pl, kind, ch=3):
    b = bytearray(pl)
    if kind == "ones+1":                                   # value count kept consistent: only the decoded mask's popcount disagrees
        struct.pack_into("<Q", b, _field_off("ones"), struct.unpack_from("<Q", b, _field_off("ones"))[0] + 1)
        p = _ivc().ImprovedVideoCompressor._parse_inter(pl)
        vals = zlib.decompress(p.vz)[:p.vcount] + bytes(ch)
        vz = zlib.compress(vals, 9)
        tail = len(pl) - len(p.vz) - 8
        return bytes(b[:tail]) + struct.pack("<II", len(vz), p.vcount + ch) + vz
    if kind == "short wlen":
        (wlen,) = struct.unpack_from("<I", b, _field_off("wlen"))
        assert wlen >= 2
        struct.pack_into("<I", b, _field_off("wlen"), wlen // 2)
    elif kind == "shape":
        struct.pack_into("<I", b, _field_off("h"), struct.unpack_from("<I", b, _field_off("h"))[0] + 1)
    elif kind == "wlen 0":
        struct.pack_into("<I", b, _field_off("wlen"), 0)
    return bytes(b)


@pytest.fixture(scope="module")
def coded_gop(pkg):
    frames = _frames(64, 64, 3, np.uint8, 8, 29, [0.05, 0.02])
    comp, pls = _compress(pkg, frames, 30, 7)               # frames 1..7: one group of 7
    assert all(pl.startswith(_ivc()._INTER_TAG) for pl in pls[1:])
    return comp, pls


_EXC = {"ones+1": ValueError, "short wlen": IndexError, "shape": ValueError, "wlen 0": ValueError}


@gpu
@pytest.mark.parametrize("kind", ["ones+1", "short wlen", "shape", "wlen 0"])
@pytest.mark.parametrize("at", [1, 4, 7])                   # first, middle and last frame of the group
def test_corrupt_frame_raises(pkg, coded_gop, kind, at):
    comp, pls = coded_gop
    bad = list(pls)
    bad[at] = _corrupt(pls[at], kind)
    with pytest.raises(_EXC[kind]) as ei:
        comp.decompress_video(compressed_frames=bad)
    assert ei.type is _EXC[kind]
    assert len(comp.decompress_video(compressed_frames=pls)) == 8       # nothing of the failed call sticks


@gpu
@pytest.mark.parametrize("at", [1, 4, 7])
def test_inter_payload_first_raises(pkg, coded_gop, at):
    comp, pls = coded_gop
    with pytest.raises(ValueError, match="without a preceding frame"):
        comp.decompress_video(compressed_frames=pls[at:])


@gpu
@pytest.mark.parametrize("first,later", [("short wlen", "shape"), ("shape", "short wlen"), ("ones+1", "short wlen"),
                                         ("short wlen", "ones+1")])
def test_first_bad_frame_decides(pkg, coded_gop, first, later):
    comp, pls = coded_gop
    bad = list(pls)
    bad[3], bad[5] = _corrupt(pls[3], first), _corrupt(pls[5], later)
    with pytest.raises(_EXC[first]) as ei:
        comp.decompress_video(compressed_frames=bad)
    assert ei.type is _EXC[first]


# ------------------------------------------------------------------ rbf_stream_apply_chain edges
def _raw_slots(masks, n):
    nb = (n + 7) // 8
    bms = np.zeros((len(masks), (nb + 15) // 16 * 16), dtype=np.uint8)
    for i, m in enumerate(masks):
        bms[i, :nb] = np.packbits(m)
    return bms


# n not a multiple of 32, of the 4096-px tile, or of 16 bytes; one and several tiles; 1, 2, 3 and 6 bytes per pixel
@gpu
@pytest.mark.parametrize("h,w,ch,dtype", [(37, 53, 1, np.uint8), (61, 70, 3, np.uint8), (67, 129, 3, np.uint16),
                                          (45, 91, 1, np.uint16), (1, 4096, 3, np.uint8), (3, 5, 1, np.uint8)])
def test_apply_chain_edges(pkg, h, w, ch, dtype):
    rng = np.random.default_rng(h * w)
    n = h * w
    hi = 256 if dtype == np.uint8 else 65536
    shape = (h, w, ch) if ch > 1 else (h, w)
    masks = [np.zeros(n, np.uint8), np.ones(n, np.uint8), (rng.random(n) < 0.3).astype(np.uint8),
             (rng.random(n) < 0.01).astype(np.uint8)]
    st = pkg.FrameStream(h, w, ch, dtype, max_frames=5, max_pairs=4, k1_only=True)
    try:
        cnt = len(masks)
        consumed, ones = st.decode_masks(_raw_slots(masks, n), np.zeros((cnt, 0), np.uint8), [0] * cnt, [0] * cnt, [0.0] * cnt,
                                         [1] * cnt)
        assert list(ones) == [int(m.sum()) for m in masks] and not consumed.any()
        base = rng.integers(0, hi, shape).astype(dtype)
        vals = [rng.integers(0, hi, int(m.sum()) * ch).astype(dtype) for m in masks]
        exp, cur = [], base.copy()
        for m, v in zip(masks, vals):
            cur = cur.copy()
            cur.reshape(n, ch)[m.astype(bool)] = v.reshape(-1, ch)
            exp.append(cur)
        # base in slot 3: the chain writes slots 4, 0, 1, 2 (slots wrap), and the download wraps with it
        st.upload(base, first=3)
        applied = st.apply_chain(3, vals)
        assert list(applied) == list(ones)
        got = st.download_batch(4, cnt)
        for t in range(cnt):
            assert np.array_equal(got[t], exp[t]), t
        assert np.array_equal(st.download(3), base)
        # one value too few at pair 2: pairs 0 and 1 are applied, frames of pairs 2 and 3 are not written
        sentinel = np.full((2,) + shape, 7, dtype=dtype)
        st.upload(base, first=0)
        st.upload(sentinel, first=3)
        short = vals[:2] + [vals[2][:-ch]] + vals[3:]
        applied = st.apply_chain(0, short)
        assert list(applied) == [ones[0], ones[1], 0, 0]
        got = st.download_batch(1, 4)
        assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])
        assert (got[2] == 7).all() and (got[3] == 7).all()
    finally:
        st.close()


# ------------------------------------------------------------------ batching is real
@gpu
def test_launches_and_copies_per_group(pkg):
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    frames = _frames(120, 160, 3, np.uint8, 30, 37, [0.05, 0.02, 0.08])
    fb = frames[0].nbytes
    stats = {}
    for bs in (29, 10, 5):
        comp, pls = _compress(pkg, frames, 30, bs)
        assert all(pl.startswith(_ivc()._INTER_TAG) for pl in pls[1:])
        L.rbf_reset_counters(ctx)
        dec = comp.decompress_video(compressed_frames=pls)
        assert np.array_equal(np.asarray(dec[-1]), frames[-1])
        groups = (29 + bs - 1) // bs
        launches, d2h = L.rbf_get_counter(ctx, b"kernel_launches"), L.rbf_get_counter(ctx, b"d2h_bytes")
        stats[bs] = (groups, launches)
        extra = d2h - 29 * fb                               # the frames, plus per-pair counters: no mask crosses PCIe
        assert 0 <= extra <= 16 * 29 + 16 * groups, (bs, d2h)
    (g1, l1), (g2, l2), (g3, l3) = stats[29], stats[10], stats[5]
    per_group = (l2 - l1) // (g2 - g1)
    assert per_group * (g2 - g1) == l2 - l1 and per_group * (g3 - g1) == l3 - l1, stats
    assert l1 - per_group * g1 == 0 and per_group <= 12, stats


# ------------------------------------------------------------------ CPU: the payload layout round trips
class _R:
    def __init__(self, raw, k, l, wlen, ones):
        self.raw, self.k, self.l, self.wlen, self.ones = raw, k, l, wlen, ones


@pytest.mark.parametrize("tag", ["RBF1", "RBF2"])
@pytest.mark.parametrize("raw", [False, True])
def test_parse_inter_round_trips_the_layout(tag, raw):
    ivcmod = _ivc()
    I = ivcmod.ImprovedVideoCompressor
    rng = np.random.default_rng(7)
    bm, wt = rng.integers(0, 256, 300).astype(np.uint8), rng.integers(0, 256, 300).astype(np.uint8)
    r = _R(raw, 0.0 if raw else 2.718281828459045, 0 if raw else 1001, 0 if raw else 517, 123)
    rz = rng.integers(0, 256, 77).astype(np.uint8).tobytes() if raw else None
    vz = b"values-stream"
    pl = I._inter_layout((31, 45), 2, 3, r, bm, wt, rz, vz, 369)
    if tag == "RBF1":
        pl = ivcmod._INTER_TAG_V1 + pl[len(ivcmod._INTER_TAG):]
    p = I._parse_inter(pl)
    assert p.v1 == (tag == "RBF1")
    assert (p.h, p.w, p.isz, p.ch, bool(p.raw)) == (31, 45, 2, 3, raw)
    assert (p.k, p.l, p.wlen, p.ones, p.vcount) == (r.k, r.l, r.wlen, 123, 369)
    assert bytes(p.vz) == vz
    if raw:
        assert bytes(p.mask_bytes) == rz and bytes(p.witness_bytes) == b""
    else:
        assert bytes(p.mask_bytes) == bm[:(1001 + 7) // 8].tobytes() and bytes(p.witness_bytes) == wt[:(517 + 7) // 8].tobytes()
