"""The device zlib coder (csrc/rbf_deflate.cuh, deflate.py, FrameStream.zlib_changed, entropy_coder="gpu").
CPU tests check the shared code-length builder and the bound; GPU tests decode every stream with stock zlib."""
import heapq
import struct
import zlib

import numpy as np
import pytest

from tests.util import synth_stream


@pytest.fixture(scope="module")
def cabi():
    from new_bloom_filter_repo_b200 import build, _cabi
    build.build()
    return _cabi


def _huffman_cost(freqs):
    """Total bits and depth of an unconstrained Huffman code (heapq), for the used symbols."""
    h = [(f, i, 0) for i, f in enumerate(freqs) if f]
    if len(h) < 2:
        return None, None
    heapq.heapify(h)
    cost, uid = 0, len(freqs)
    depth = {}
    nodes = {i: [i] for _, i, _ in h}
    while len(h) > 1:
        f1, i1, d1 = heapq.heappop(h)
        f2, i2, d2 = heapq.heappop(h)
        cost += f1 + f2
        nodes[uid] = nodes.pop(i1) + nodes.pop(i2)
        for s in nodes[uid]:
            depth[s] = depth.get(s, 0) + 1
        heapq.heappush(h, (f1 + f2, uid, max(d1, d2) + 1))
        uid += 1
    return cost, max(depth.values())


def _check_lengths(cabi, freqs, max_bits):
    freqs = [int(x) for x in freqs]
    lens = [int(x) for x in cabi.deflate_code_lengths(freqs, max_bits)]
    used = [i for i, f in enumerate(freqs) if f]
    assert max(lens) <= max_bits
    assert sum(1 for x in lens if x) >= 2
    if len(used) >= 2:
        assert all(lens[i] == 0 for i, f in enumerate(freqs) if not f)
        assert sum(2.0 ** -x for x in lens if x) == 1.0
        cost, depth = _huffman_cost(freqs)
        if depth <= max_bits:
            assert sum(f * l for f, l in zip(freqs, lens)) == cost
    else:
        assert sum(1 for x in lens if x) == 2 and all(lens[i] == 1 for i in used)
    return lens


def test_code_lengths_random(cabi):
    rng = np.random.default_rng(5)
    for trial in range(300):
        nsym = int(rng.choice([19, 30, 286, 288, int(rng.integers(2, 289))]))
        max_bits = 7 if nsym == 19 else int(rng.choice([15, 15, 9, 12]))
        f = rng.integers(0, 1000, nsym) * (rng.random(nsym) < rng.random())
        if rng.random() < 0.3:
            f = (rng.pareto(1.0, nsym) * 10).astype(np.int64) * (rng.random(nsym) < 0.7)
        if np.count_nonzero(f) > 2 ** max_bits:
            continue
        _check_lengths(cabi, f, max_bits)


def test_code_lengths_fibonacci_forces_the_limit(cabi):
    fib = [1, 1]
    while len(fib) < 40:
        fib.append(fib[-1] + fib[-2])
    for n, max_bits in ((40, 15), (30, 15), (25, 7), (19, 7), (286, 15)):
        f = (fib * 8)[:n]
        assert _huffman_cost(f)[1] > max_bits
        lens = _check_lengths(cabi, f, max_bits)
        assert max(lens) == max_bits


def test_code_lengths_single_and_no_symbol(cabi):
    for nsym, max_bits in ((286, 15), (30, 15), (19, 7)):
        _check_lengths(cabi, [0] * nsym, max_bits)
        for s in (0, 1, nsym - 1):
            f = [0] * nsym
            f[s] = 77
            _check_lengths(cabi, f, max_bits)


def test_zlib_bound(cabi):
    last = 0
    for n in list(range(0, 300)) + [65534, 65535, 65536, 65537, 131071, 131072, 131073, 3 * 65536 + 1, 10 ** 7, 10 ** 8 + 3]:
        b = cabi.zlib_bound(n)
        assert b >= n + 6 and b >= last
        last = b
    assert cabi.zlib_bound(0) == 8


# ------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def pkg():
    import new_bloom_filter_repo_b200 as p
    assert p._cabi.device_info()["cc"] == (9, 0)
    return p


def _inflate(z, data):
    d = zlib.decompressobj()
    out = d.decompress(z) + d.flush()
    assert d.eof and d.unused_data == b""
    assert out == bytes(data)
    from new_bloom_filter_repo_b200 import _cabi
    assert len(z) <= _cabi.zlib_bound(len(data))


def _periodic(period, n, seed):
    rng = np.random.default_rng(seed)
    return np.resize(rng.integers(0, 256, period, dtype=np.uint8), n).tobytes()


def _inputs():
    rng = np.random.default_rng(9)
    rnd = lambda n: rng.integers(0, 256, n, dtype=np.uint8).tobytes()      # noqa: E731
    ins = {"empty": b""}
    for n in (1, 2, 3, 258, 259, 65535, 65536, 65537, 3 * 65536 + 1):
        ins["text%d" % n] = (b"the quick brown fox jumps over the lazy dog %d " % n * (n // 40 + 1))[:n]
        ins["rand%d" % n] = rnd(n)
    ins["zeros1M"] = bytes(1 << 20)
    ins["random1M"] = np.random.default_rng(1).integers(0, 256, 1 << 20, dtype=np.uint8).tobytes()
    ins["two_symbol"] = (rng.random(300000) < 0.3).astype(np.uint8).tobytes()
    ins["period32768"] = _periodic(32768, 200000, 2)
    ins["period32769"] = _periodic(32769, 200000, 3)
    ins["frame_u8"] = synth_stream(1080, 1920, 2, 4, [0.05])[1].tobytes()
    ins["frame_u16"] = synth_stream(1080, 1920, 1, 6, [0.05], dtype=np.uint16)[0].tobytes()
    return ins


@pytest.mark.gpu
def test_streams_decode_with_stock_zlib(pkg):
    ins = _inputs()
    names = list(ins)
    zs = pkg.deflate.compress_many([ins[k] for k in names])
    for k, z in zip(names, zs):
        _inflate(z, ins[k])
    assert zs[names.index("empty")] == bytes.fromhex("789c030000000001")
    for k in ("zeros1M",):
        assert len(zs[names.index(k)]) < len(ins[k]) // 100
    assert len(zs[names.index("random1M")]) == len(ins["random1M"]) + 16 * 15 + 8     # stored: 2 blocks + sync flush per segment


@pytest.mark.gpu
def test_buffer_kinds_and_determinism(pkg):
    a = np.arange(300000, dtype=np.uint16).reshape(300, 1000) % 777
    z1 = pkg.deflate.compress(a)
    _inflate(z1, a.tobytes())
    assert pkg.deflate.compress(a) == z1
    assert pkg.deflate.compress(bytearray(a.tobytes())) == z1
    assert pkg.deflate.compress(memoryview(a.tobytes())) == z1
    batch = pkg.deflate.compress_many([b"x" * 1000, a, b"", a.tobytes()])
    assert batch[1] == z1 and batch[3] == z1
    with pytest.raises(ValueError):
        pkg.deflate.compress(a[:, ::2])


@pytest.mark.gpu
def test_ratio_floor_on_keyframe(pkg):
    x = synth_stream(1080, 1920, 3, 2, [0.05])[0].tobytes()
    z = pkg.deflate.compress(x)
    _inflate(z, x)
    assert len(z) <= 1.10 * len(zlib.compress(x, 1)), (len(z), len(zlib.compress(x, 1)))


@pytest.mark.gpu
def test_zlib_changed_matches_gather(pkg):
    frames = synth_stream(270, 480, 6, 8, [0.05, 0.0, 0.3, 0.01, 0.5])
    st = pkg.FrameStream(270, 480, 3, np.uint8, max_frames=6)
    st.upload(frames)
    res = st.encode_consecutive(6, 3.0)
    assert any(r.ones == 0 for r in res)
    gathered = st.gather_changed()
    zs = st.zlib_changed()
    assert len(zs) == len(gathered) == 5
    for g, z in zip(gathered, zs):
        _inflate(z, g.tobytes())
    assert st.zlib_changed() == zs
    st.close()


def _clip(kind, n, seed):
    """yuv8: YUV444 frames with plane info; yuv16: 16-bit YUV444 samples as plain 3-channel frames (the keyframe decoder,
    fvc:76-181, reads plane info as 8-bit planes); bgr8; gray8 / gray16: 1-channel frames."""
    dt = np.uint16 if kind.endswith("16") else np.uint8
    fr = synth_stream(72, 120, n, seed, [0.05, 0.4, 0.0, 0.2], dtype=dt)
    if kind.startswith("gray"):
        return [np.ascontiguousarray(f[:, :, 0]) for f in fr], "BGR"
    return [f for f in fr], ("YUV" if kind == "yuv8" else "BGR")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["yuv8", "yuv16", "bgr8", "gray8", "gray16"])
@pytest.mark.parametrize("mode", ["lossless", "reference"])
@pytest.mark.parametrize("ki", [1, 5])
def test_compress_video_gpu_coder_roundtrip(pkg, kind, mode, ki):
    frames, cs = _clip(kind, 7, 3)
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=ki)
    comp.entropy_coder = "gpu"
    comp.inter_frame_mode = mode
    comp.inter_frame_threshold = 3.0
    comp.compress_video(list(frames), input_color_space=cs)
    gpu_payloads = list(comp._last_compressed_frames)
    dec = comp.decompress_video(compressed_frames=gpu_payloads)
    assert comp.verify_lossless(frames, dec)["lossless"]
    if ki == 1:
        ref = pkg.ImprovedVideoCompressor(keyframe_interval=1)
        ref.compress_video(list(frames), input_color_space=cs)
        fvc = pkg.FixedVideoCompressor(verbose=False)
        for g, z in zip(gpu_payloads, ref._last_compressed_frames):
            dg, dz = fvc.decompress_frame(g), fvc.decompress_frame(z)
            assert np.array_equal(np.asarray(dg), np.asarray(dz))
            if hasattr(dz, "yuv_info"):
                for name in ("y_plane", "u_plane", "v_plane"):
                    assert np.array_equal(dg.yuv_info[name], dz.yuv_info[name])
                assert dg.yuv_info["format"] == dz.yuv_info["format"]


@pytest.mark.gpu
def test_compress_video_rejects_unknown_coder(pkg):
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=1)
    comp.entropy_coder = "brotli"
    with pytest.raises(ValueError):
        comp.compress_video([np.zeros((8, 8, 3), np.uint8)])


@pytest.mark.gpu
def test_gpu_inter_payload_layout(pkg):
    """The inter payload keeps _inter_layout's fields: value count and stream length agree with the gather."""
    frames, cs = _clip("yuv8", 4, 11)
    comp = pkg.ImprovedVideoCompressor(keyframe_interval=4)
    comp.entropy_coder = "gpu"
    comp.compress_video(list(frames), input_color_space=cs)
    p = comp._last_compressed_frames[1]
    pos = 8 + struct.calcsize("<IIIBB") + struct.calcsize("<dIIQ")
    (bl,) = struct.unpack_from("<I", p, pos)
    pos += 4 + bl
    (wl,) = struct.unpack_from("<I", p, pos)
    pos += 4 + wl
    vlen, vcount = struct.unpack_from("<II", p, pos)
    vals = zlib.decompress(p[pos + 8:pos + 8 + vlen])
    assert len(vals) == vcount and pos + 8 + vlen == len(p)
