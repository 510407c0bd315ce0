"""The host orchestration of rbf_api.cu: the kernel_launches counter equals the kernels each entry point actually ran (torch.profiler's
CUDA activity trace is the independent count), decode_verify decodes the last encode whichever encode path produced it, and
stage_ms refuses once an encode without stage events (encode_host) has replaced the timed one."""
import json
import os
import tempfile

import numpy as np
import pytest

from tests.util import synth_stream

gpu = pytest.mark.gpu

THR = 3.0
P_SEQ = [0.05, 0.5, 0.0, 0.02, 0.1]      # coded, raw (p >= p*), raw (no change), coded, coded
NFR = 33                                  # 32 pairs: enough for encode_ranges = 4 and kq_ranges = 4 to split the encode


@pytest.fixture(scope="module")
def pkg():
    import new_bloom_filter_repo_b200 as p
    assert p._cabi.device_info()["cc"] == (9, 0)
    return p


def _set(pkg, **opts):
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    for k, v in opts.items():
        pkg._cabi.check(L.rbf_set_option(ctx, k.encode(), int(v)), ctx)


DEFAULTS = dict(encode_ranges=1, kq_ranges=1, host_chunk_frames=32)


def counted_run(pkg, fn, name, counts):
    """fn() inside the range "entry <name>" of the open profiler session -> fn's result; counts[name] = its kernel_launches delta."""
    import torch
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    torch.cuda.synchronize()
    before = L.rbf_get_counter(ctx, b"kernel_launches")
    with torch.profiler.record_function("entry " + name):
        out = fn()
        torch.cuda.synchronize()
    counts[name] = L.rbf_get_counter(ctx, b"kernel_launches") - before
    return out


def profiled_kernels(run):
    """run(counts) under ONE torch.profiler session with CPU and CUDA activities -> {name: (counts[name], [(kernel name, grid, block)]
    of the library's kernels launched inside the range "entry <name>", in start order)}.  A kernel belongs to the range that holds
    its launch call (the trace links the two by correlation id).  Memcpy and memset activities are not kernels and are left out.
    One session, opened by a synchronised torch kernel: in a process that had already run other tests, a trace of one short session
    per entry point lost kernels, sometimes a whole session's."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    counts = {}
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device="cuda").add_(1)
        torch.cuda.synchronize()
        run(counts)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    ranges = {e["name"][len("entry "):]: (e["ts"], e["ts"] + e["dur"]) for e in events
              if e.get("cat") == "user_annotation" and e["name"].startswith("entry ")}
    assert sorted(ranges) == sorted(counts), (sorted(ranges), sorted(counts))
    launched = {e["args"]["correlation"]: e["ts"] for e in events if e.get("cat") == "cuda_runtime" and "correlation" in e.get("args", {})}
    ks = sorted((e for e in events if e.get("cat") == "kernel" and "rbf::" in e["name"]), key=lambda e: e["ts"])
    out = {}
    for name, (t0, t1) in ranges.items():
        mine = [e for e in ks if t0 <= launched.get(e["args"].get("correlation"), -1) <= t1]
        out[name] = (counts[name], [(e["name"], tuple(e["args"].get("grid", ())), tuple(e["args"].get("block", ()))) for e in mine])
    return out


def _decode_inputs(st, res, n):
    """What decode_masks takes for the pairs of the last encode: packbits bitmaps (the packbits mask for a raw pair) and witnesses."""
    P = len(res)
    bm, wt, mk = st.fetch_batch(0, P, want_masks=True)
    nb = (n + 7) // 8
    bslot = max(bm.shape[1], (nb + 15) // 16 * 16)
    bitmaps = np.zeros((P, bslot), dtype=np.uint8)
    bitmaps[:, :bm.shape[1]] = bm
    for i, r in enumerate(res):
        if r.raw:
            bitmaps[i, :nb] = np.packbits(np.unpackbits(mk[i], bitorder="little")[:n])
    return (bitmaps, wt, [r.l for r in res], [r.wlen for r in res], [r.k for r in res], [int(r.raw) for r in res])


def entry_points(pkg, h, w, counts):
    """Every host path under test, each through counted_run."""
    frames = synth_stream(h, w, NFR, 11, P_SEQ)
    st = pkg.FrameStream(h, w, 3, np.uint8, max_frames=NFR, max_pairs=NFR - 1)
    try:
        for name, opts in (("encode", {}), ("encode_ranges4", dict(encode_ranges=4)), ("encode_kq4", dict(kq_ranges=4))):
            st.upload(frames)
            _set(pkg, **dict(DEFAULTS, **opts))
            try:
                res = counted_run(pkg, lambda: st.encode_consecutive(NFR, THR), name, counts)
            finally:
                _set(pkg, **DEFAULTS)
        assert any(r.raw for r in res) and not all(r.raw for r in res)
        _set(pkg, host_chunk_frames=3)
        try:
            res = counted_run(pkg, lambda: st.encode_host(frames, THR), "encode_host", counts)
        finally:
            _set(pkg, **DEFAULTS)
        mism = counted_run(pkg, st.decode_verify, "decode_verify", counts)
        assert not mism.any()
        vals = counted_run(pkg, st.gather_changed, "gather_changed", counts)
        counted_run(pkg, st.zlib_changed, "zlib_changed", counts)
        args = _decode_inputs(st, res, h * w)
        counted_run(pkg, lambda: (st.decode_masks(*args), st.apply_chain(0, vals)), "decode_masks+apply_chain", counts)
        assert np.array_equal(st.download(NFR - 1), frames[-1])
    finally:
        _set(pkg, **DEFAULTS)
        st.close()
    mask = (frames[1] != frames[0]).any(-1).reshape(-1).astype(np.uint8)
    bfc = pkg.BloomFilterCompressor()
    bm, wt, _, n_, _ = counted_run(pkg, lambda: bfc.compress(mask), "compress", counts)
    dec = counted_run(pkg, lambda: bfc.decompress(bm, wt, n_, bfc.last_info.k), "decompress", counts)
    assert np.array_equal(dec, mask)


@gpu
@pytest.mark.parametrize("h,w", [(120, 160), (1080, 1920)])
def test_launch_counter_equals_kernels_run(pkg, h, w):
    """120x160 has one witness chunk (K3b and K4b skip the pass-count kernel); 1080p has several."""
    for name, (n, ks) in profiled_kernels(lambda counts: entry_points(pkg, h, w, counts)).items():
        assert ks, (name, "the profiler recorded no kernel")
        assert n == len(ks), (name, n, [k[0][:60] for k in ks])


@gpu
def test_decode_verify_follows_the_last_encode(pkg):
    h, w = 120, 160
    frames = synth_stream(h, w, NFR, 5, P_SEQ)
    other = synth_stream(h, w, NFR, 6, P_SEQ[::-1])
    st = pkg.FrameStream(h, w, 3, np.uint8, max_frames=NFR, max_pairs=NFR - 1)
    try:
        # K2 beside K3 (per-range K3 work lists), then a chunked encode_host of fewer pairs
        st.upload(frames)
        _set(pkg, kq_ranges=4)
        try:
            st.encode_consecutive(NFR, THR)
        finally:
            _set(pkg, **DEFAULTS)
        _set(pkg, host_chunk_frames=2)
        try:
            res = st.encode_host(other[:17], THR)
        finally:
            _set(pkg, **DEFAULTS)
        assert any(r.raw for r in res) and not all(r.raw for r in res)
        mism = st.decode_verify()
        assert mism.shape == (16,) and not mism.any(), mism
        # encode_host, then a pipelined encode over other frames
        st.encode_host(other, THR)
        st.upload(frames)
        _set(pkg, encode_ranges=4)
        try:
            st.encode_consecutive(NFR, THR)
        finally:
            _set(pkg, **DEFAULTS)
        mism = st.decode_verify()
        assert mism.shape == (NFR - 1,) and not mism.any(), mism
        # a group decode leaves no encode to verify, until the next encode
        res = st.encode_consecutive(NFR, THR)
        args = _decode_inputs(st, res, h * w)
        st.decode_masks(*args)
        with pytest.raises(pkg._cabi.RbfError):
            st.decode_verify(NFR - 1)
        st.upload(other)
        st.encode_consecutive(NFR, THR)
        mism = st.decode_verify()
        assert not mism.any(), mism
    finally:
        _set(pkg, **DEFAULTS)
        st.close()


@gpu
def test_stage_ms_refuses_after_encode_host(pkg):
    frames = synth_stream(120, 160, 9, 3, P_SEQ)
    st = pkg.FrameStream(120, 160, 3, np.uint8, max_frames=9)
    try:
        st.upload(frames)
        st.encode_consecutive(9, THR)
        ms = st.stage_ms()
        assert ms["encode_total"] > 0.0
        st.encode_host(frames, THR)
        with pytest.raises(pkg._cabi.RbfError):
            st.stage_ms()
    finally:
        st.close()
