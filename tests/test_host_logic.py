"""CPU tests of host-side glue: keyframe codec wire format (byte-identical to the reference's
FixedVideoCompressor), YUVFrame wrapper, shard partitioning."""
import hashlib

import numpy as np

from tests.util import golden_json, golden_npz


def test_keyframe_payload_bytes_match_reference():
    from new_bloom_filter_repo_b200.fixed_video_compressor import FixedVideoCompressor
    g = golden_json("keyframe_kat.json")
    arr = golden_npz("keyframe_arrays.npz")
    comp = FixedVideoCompressor(verbose=False)
    for rec in g["cases"]:
        f = arr[rec["name"] + "/frame"]
        fr = comp.add_yuv_info_to_frame(f) if rec["yuv"] else f
        payload = comp.compress_frame(fr)
        assert hashlib.sha256(payload).hexdigest() == rec["payload_sha256"]
        assert payload == arr[rec["name"] + "/payload"].tobytes()
        back = comp.decompress_frame(payload)
        data = back.data if hasattr(back, "yuv_info") else back
        assert np.array_equal(data, f) and data.dtype == f.dtype
        assert hasattr(back, "yuv_info") == rec["yuv"]
        res = comp.verify_lossless([fr], [back])
        assert res["lossless"] and res["exact_frame_matches"] == 1


def test_verify_lossless_detects_difference():
    from new_bloom_filter_repo_b200.fixed_video_compressor import FixedVideoCompressor
    comp = FixedVideoCompressor(verbose=False)
    a = np.zeros((4, 4, 3), np.uint8)
    b = a.copy(); b[1, 1, 1] = 9
    r = comp.verify_lossless([a, a], [a, b])
    assert not r["lossless"] and r["diff_frames"] == [1] and r["max_diff_frame"] == 1
    assert comp.verify_lossless([a], [a, a])["lossless"] is False


def test_shard_partition():
    from new_bloom_filter_repo_b200.distributed import shard_pairs
    for pairs in (1, 7, 8, 29, 290, 299):
        for world in (1, 2, 3, 4, 8):
            seen = []
            for r in range(world):
                lo, hi = shard_pairs(pairs, r, world)
                assert 0 <= lo <= hi <= pairs
                seen += list(range(lo, hi))
            assert seen == list(range(pairs))
            sizes = [shard_pairs(pairs, r, world)[1] - shard_pairs(pairs, r, world)[0] for r in range(world)]
            assert max(sizes) - min(sizes) <= 1


def test_keyframe_job_equals_compress_frame():
    """The GOP loop compresses a keyframe's zlib blobs as separate pool jobs (ImprovedVideoCompressor._keyframe_job with the
    "zlib" coder): the assembled payload is byte-identical to compress_frame's."""
    from concurrent.futures import ThreadPoolExecutor
    from new_bloom_filter_repo_b200.fixed_video_compressor import FixedVideoCompressor
    from new_bloom_filter_repo_b200.improved_video_compressor import ImprovedVideoCompressor
    c = FixedVideoCompressor(verbose=False)
    comp = object.__new__(ImprovedVideoCompressor)         # the "zlib" coder's keyframe job needs no device
    comp.entropy_coder = "zlib"
    rng = np.random.default_rng(0)
    with ThreadPoolExecutor(3) as pool:
        for shape, dt in (((48, 64, 3), np.uint8), ((32, 40), np.uint8), ((20, 24, 3), np.uint16)):
            f = rng.integers(0, 200, shape).astype(dt)
            assert comp._keyframe_job(f, pool)() == c.compress_frame(f)
            if f.ndim == 3:
                y = c.add_yuv_info_to_frame(f)
                assert comp._keyframe_job(y, pool)() == c.compress_frame(y)


def test_bench_counters_go_stale_with_the_sources(tmp_path, monkeypatch):
    """bench.py reports roofline.traffic / issue_frac only while the kernel sources still hash to what was profiled
    (scripts/ncu_summary.py --json records that hash), and reports nothing when no counters file exists."""
    import hashlib
    import json
    import os
    import bench
    sources = ["new_bloom_filter_repo_b200/csrc/" + f for f in ("rbf_k3_query.cuh", "rbf_hash.cuh", "rbf_k2_insert.cuh", "rbf_kernels.cu")]
    h = hashlib.sha256()
    for name in sources:                                       # a copy of the current sources under a fake ROOT
        data = open(os.path.join(bench.ROOT, name), "rb").read()
        os.makedirs(os.path.dirname(tmp_path / name), exist_ok=True)
        (tmp_path / name).write_bytes(data)
        h.update(data)
    monkeypatch.setattr(bench, "ROOT", str(tmp_path))
    assert bench.kernel_counters("k_query4") is None           # no counters file: the fields stay null
    (tmp_path / "profiles").mkdir()
    rec = {"kernel": "k_query4", "pairs_in_launch": 29, "dram_bytes_per_pair": 1.5e6, "thread_inst_per_px": 100.0,
           "issue_active_frac": 0.6, "sources": sources, "sources_sha16": h.hexdigest()[:16]}
    counters = tmp_path / "profiles" / "r02_k_query4_counters.json"
    counters.write_text(json.dumps(rec))
    c = bench.kernel_counters("k_query4")
    assert c is not None and c["stale"] is False and c["dram_bytes_per_pair"] == 1.5e6 and c["thread_inst_per_px"] == 100.0
    counters.write_text(json.dumps(dict(rec, sources_sha16="0" * 16)))       # same sources, different recorded hash
    assert bench.kernel_counters("k_query4")["stale"] is True
    counters.write_text(json.dumps(rec))
    (tmp_path / sources[0]).write_bytes(b"// edited\n" + (tmp_path / sources[0]).read_bytes())   # the sources change
    assert bench.kernel_counters("k_query4")["stale"] is True
    assert bench.kernel_counters("k_no_such_kernel") is None


def test_bench_stream_frames_equals_fill_stream_slices():
    """Strong scaling: a rank builds only frames lo..hi of the shared stream; they must equal the full stream's slice."""
    import bench
    for dt in (np.uint8, np.uint16):
        full = np.empty((9, 24, 40, 3), dt)
        bench.fill_stream(full, seed=3)
        for lo, hi in ((0, 3), (3, 8), (7, 8)):
            out = np.empty((hi - lo + 1, 24, 40, 3), dt)
            bench.stream_frames(9, 24, 40, 3, lo, hi, out)
            assert np.array_equal(out, full[lo:hi + 1])


def test_bench_dump_outputs_files(tmp_path, monkeypatch):
    """--dump-outputs: float64 per-pair results and CRC-32s, float32 byte samples capped at DUMP_SAMPLE, all reloadable."""
    import zlib
    from types import SimpleNamespace
    import bench
    monkeypatch.setattr(bench, "DUMP_SAMPLE", 4000)
    rng = np.random.default_rng(0)
    bms, wts, mks = (rng.integers(0, 256, (3, w), dtype=np.uint8) for w in (3000, 1000, 5000))
    st = SimpleNamespace(fetch_batch=lambda first, count, want_masks=False: (bms, wts, mks))
    res = [SimpleNamespace(ones=100 + t, resid=t, p=0.05, k=3.3, l=l, wlen=w, raw=l == 0)
           for t, (l, w) in enumerate([(20000, 7000), (0, 0), (23999, 7999)])]
    bench.dump_outputs(str(tmp_path), st, res, 3)
    out = {p.stem: np.load(p) for p in tmp_path.glob("*.npy")}
    assert sum(p.stat().st_size for p in tmp_path.glob("*.npy")) < 64 << 20
    assert out["l"].dtype == np.float64 and list(out["l"]) == [20000, 0, 23999] and list(out["raw"]) == [0, 1, 0]
    assert out["bitmap_crc32"][0] == zlib.crc32(bms[0, :2500].tobytes()) and out["bitmap_crc32"][1] == zlib.crc32(b"")
    assert out["mask_crc32"][2] == zlib.crc32(mks[2].tobytes())
    assert out["witness_bytes_sample"].dtype == np.float32 and out["witness_bytes_sample"].size == 1875
    assert out["mask_bytes_sample"].size == 4000 and set(np.unique(out["mask_bytes_sample"])) <= set(range(256))


def test_bench_host_cores_is_positive_and_bounded():
    import os
    import bench
    n = bench.host_cores()
    assert 1 <= n <= (os.cpu_count() or 1)
