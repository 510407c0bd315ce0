"""Every way rbf_api.cu splits one encode -- pipelined ranges (encode_ranges), K2 beside K3 (kq_ranges), host chunks (encode_host,
host_chunk_frames) -- against the C oracle, pair by pair, at the range, chunk and override edges where the host code goes wrong:
per-pair k / l overrides at the first and last pair of a range, ranges and chunks in which every pair is raw (on a stream whose
slots were last written by a bigger encode, by decode_verify or by decode_masks), pair lists that are not one chain, and the pair
counts at which a split starts.

The reference of a pair is independent of the library: the mask from oracle.frame_diff_mask, (bitmap, witness, p, k, l) from
oracle.compress.  After any encode, with any schedule, a raw pair's bitmap and witness rows read as zero, and a coded pair's rows
are zero past its payload."""
import contextlib
import json
import math
import os
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from tests.util import synth_stream

pytestmark = pytest.mark.gpu

THR = 3.0
P_RAW = 0.45                                  # p >= p* = 0.32453: raw, whatever the override
CODED_P = (0.05, 0.02, 0.1, 0.2, 0.01, 0.15, 0.03)
KS = (0.5, 1.0, 1.25, 2.0, 2.7, 3.0, 3.5, 4.0, 4.2, 5.0, 5.9, 1.6, 2.35, 4.75, 0.85)   # floor 0..5, fractional and integral
H, W = 120, 160
DEFAULT_SCHEDULE = dict(encode_ranges=1, kq_ranges=1, host_chunk_frames=32)


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


@contextlib.contextmanager
def schedule(pkg, **opts):
    """Context options are process-wide: every schedule option is set explicitly (an RBF_* environment knob must not leak in),
    and the defaults come back whatever happens inside."""
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    try:
        for k, v in dict(DEFAULT_SCHEDULE, **opts).items():
            pkg._cabi.check(L.rbf_set_option(ctx, k.encode(), int(v)), ctx)
        yield
    finally:
        for k, v in DEFAULT_SCHEDULE.items():
            L.rbf_set_option(ctx, k.encode(), v)


def launches(pkg):
    return pkg._cabi.lib().rbf_get_counter(pkg._cabi.ctx(), b"kernel_launches")


# ------------------------------------------------------------------ inputs and the oracle
def coded_p(i):
    return CODED_P[i % len(CODED_P)]


def raw_p(i):
    return P_RAW if i % 2 == 0 else 0.0


def make_frames(p_list, seed, h=H, w=W, channels=3, dtype=np.uint8):
    """synth_stream with pair t changing a p_list[t] share of its pixels, plus the low bit of one sample (not the one the mask reads
    for 3 channels) flipped in 1% of each frame's pixels: those differ without crossing the threshold, so resid is not zero."""
    fr = synth_stream(h, w, len(p_list) + 1, seed, list(p_list), dtype)
    if channels == 1:
        fr = np.ascontiguousarray(fr[..., 0])
    for t in range(1, len(fr)):
        flip = np.random.default_rng(seed * 7919 + t).random((h, w)) < 0.01
        if channels == 1:
            fr[t][flip] ^= 1
        else:
            fr[t, :, :, 2][flip] ^= 1
    return fr


class Ref:
    __slots__ = ("mask", "ones", "resid", "p", "k", "l", "wlen", "raw", "floor_k", "act_T", "bitmap", "witness")


def oracle_pair(co, prev, curr, ko=0.0, lo=0):
    m, ones = co.frame_diff_mask(prev, curr, THR)
    r = Ref()
    r.mask = m.reshape(-1)
    r.ones = ones
    changed = (prev != curr).reshape(r.mask.size, -1).any(axis=1)
    r.resid = int((changed & (r.mask == 0)).sum())
    ob, ow, r.p, _, _, k, l = co.compress(r.mask, k_l_override=(float(ko), int(lo)) if ko > 0 else None)
    r.raw = l == 0
    r.k, r.l = float(k), int(l)
    r.wlen = 0 if r.raw else len(ow)
    r.floor_k = 0 if r.raw else int(math.floor(k))
    r.act_T = 0 if r.raw else co.activation_threshold(k - math.floor(k))
    r.bitmap = b"" if r.raw else np.packbits(ob).tobytes()
    r.witness = b"" if r.raw else np.packbits(ow).tobytes()
    return r


def oracle_refs(co, frames, prev=None, curr=None, ko=None, lo=None):
    """The oracle of every pair, on a few threads: the C oracle keeps no state and ctypes releases the GIL around its calls."""
    P = len(frames) - 1 if prev is None else len(prev)
    prev = range(P) if prev is None else prev
    curr = range(1, P + 1) if curr is None else curr
    args = [(frames[a], frames[b], ko[i] if ko else 0.0, lo[i] if lo else 0) for i, (a, b) in enumerate(zip(prev, curr))]
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        return list(ex.map(lambda a: oracle_pair(co, *a), args))


# ------------------------------------------------------------------ running a schedule and checking its outputs
def chunk_bounds(nframes, ch):
    """Pair boundaries of encode_host's chunks of ch frames: chunk k encodes the pairs whose current frame it holds."""
    b = [0]
    for f0 in range(0, nframes, ch):
        p1 = min(f0 + ch, nframes) - 1
        if p1 > b[-1]:
            b.append(p1)
    return b


def range_bounds(sched, P):
    """Pair boundaries of the pieces a schedule splits P pairs into (four nominal pieces for the serial encode)."""
    if "host_chunk_frames" in sched:
        return chunk_bounds(P + 1, sched["host_chunk_frames"])
    R = sched.get("encode_ranges", sched.get("kq_ranges", 4))
    return [P * r // R for r in range(R + 1)]


def run(pkg, st, sched, frames, ko=None, lo=None, prev=None, curr=None):
    """One encode of frames under sched -> (results, encode_host's bitmap rows, witness rows) (rows None for the resident encode)."""
    with schedule(pkg, **sched):
        if "host_chunk_frames" in sched:
            assert ko is None and prev is None
            P, slot = len(frames) - 1, (st.npix + 7) // 8 + 16
            ob = np.full((P, slot), 0xAB, np.uint8)            # every row is written: bytes past a payload must come back zero
            ow = np.full((P, slot), 0xAB, np.uint8)
            res = st.encode_host(frames, THR, bitmap_slot=slot, witness_slot=slot, out_bitmaps=ob, out_witness=ow)
            return res, ob, ow
        st.upload(frames)
        kw = {} if ko is None else dict(k_override=ko, l_override=lo)
        if prev is None:
            return st.encode_consecutive(len(frames), THR, **kw), None, None
        return st.encode(prev, curr, THR, **kw), None, None


def fields(r):
    return (r.n, r.ones, r.resid, r.raw, r.l, r.wlen, r.k.hex(), r.p.hex(), r.floor_k, r.act_T)


def assert_rows(bms, wts, refs, what):
    for i, o in enumerate(refs):
        nb, nw = len(o.bitmap), len(o.witness)
        assert bms[i, :nb].tobytes() == o.bitmap, (what, "bitmap", i)
        assert not bms[i, nb:].any(), (what, "bitmap row not zero past the payload", i, o.raw)
        assert wts[i, :nw].tobytes() == o.witness, (what, "witness", i)
        assert not wts[i, nw:].any(), (what, "witness row not zero past the payload", i, o.raw)


def assert_encode(st, res, refs, ob=None, ow=None):
    """Every PairResult field first (a wrong pair fails here, before anything decodes it), then the bytes through encode_host's rows,
    fetch and fetch_batch, then the GPU round trip."""
    assert len(res) == len(refs)
    for i, (r, o) in enumerate(zip(res, refs)):
        want = (st.npix, o.ones, o.resid, o.raw, o.l, o.wlen, o.k.hex(), float(o.p).hex(), o.floor_k, o.act_T)
        assert fields(r) == want, (i, fields(r), want)
    if ob is not None:
        assert_rows(ob, ow, refs, "encode_host")
    for i, o in enumerate(refs):
        bm, wt, mk = st.fetch(i)
        assert bm.tobytes() == o.bitmap and wt.tobytes() == o.witness, ("fetch", i)
        assert np.array_equal(mk, o.mask), ("mask", i)
    bms, wts, _ = st.fetch_batch(0, len(refs))
    assert_rows(bms, wts, refs, "fetch_batch")
    assert not st.decode_verify().any()


# ------------------------------------------------------------------ A. per-pair overrides
SPECIAL = ("optimal", "l_zero", "pstar", "override", "l_n", "p_zero")


def override_plan(bounds, n, raw_ranges=()):
    """(p per pair, k_override, l_override): distinct (k, l) per pair, so that coding a pair with another pair's override changes
    its bytes; the first and last pair of every range (and every seventh pair) take one of the SPECIAL kinds in turn.  Pairs of
    raw_ranges change by p = 0 (no override) or p >= p* (override kept, to be ignored)."""
    P = bounds[-1]
    ends = sorted({b for r in range(len(bounds) - 1) for b in (bounds[r], bounds[r + 1] - 1)} | set(range(3, P, 7)))
    kind = {i: SPECIAL[j % len(SPECIAL)] for j, i in enumerate(ends)}
    raw = {i for r in raw_ranges for i in range(bounds[r], bounds[r + 1])}
    p, ko, lo = [], [], []
    for i in range(P):
        k, l = KS[i % len(KS)], int(n * (1500 + (977 * i) % 4500) / 19200)    # l from 0.08 n to 0.31 n
        kd, pi = kind.get(i, "override"), coded_p(i)
        if kd == "optimal":
            k, l = 0.0, 1234                                  # k <= 0: no override, l ignored
        elif kd == "l_zero":
            l = 0                                             # forces raw
        elif kd == "l_n":
            l = n + 7 * (i % 2)                               # l >= n forces raw
        elif kd == "pstar":
            pi = P_RAW                                        # p >= p*: the override is ignored
        elif kd == "p_zero":
            pi, k = 0.0, 0.0                                  # no change, no override: raw
        if i in raw:
            pi = raw_p(i)
            if pi == 0.0:
                k = 0.0                                       # an override would code the empty mask
        p.append(pi); ko.append(k); lo.append(l)
    return p, ko, lo


A_CASES = [(dict(encode_ranges=R), P) for R in (2, 3, 5, 8) for P in (8 * R, 8 * R + 3)] + \
          [(dict(kq_ranges=Q), P) for Q in (2, 8) for P in (8 * Q, 8 * Q + 3)]


def _sid(sched):
    return ",".join("%s=%d" % kv for kv in sched.items()) or "serial"


def check_overrides(pkg, co, sched, P, seed, h=H, w=W, channels=3, dtype=np.uint8, raw_ranges=()):
    p, ko, lo = override_plan(range_bounds(sched, P), h * w, raw_ranges)
    frames = make_frames(p, seed, h, w, channels, dtype)
    refs = oracle_refs(co, frames, ko=ko, lo=lo)
    assert any(r.raw for r in refs) and sum(not r.raw for r in refs) > P // 2
    st = pkg.FrameStream(h, w, channels, dtype, max_frames=P + 1)
    try:
        for s in (sched, {}):                                 # the split, then the serial encode over the same slots
            res, _, _ = run(pkg, st, s, frames, ko, lo)
            assert_encode(st, res, refs)
    finally:
        st.close()


@pytest.mark.parametrize("sched,P", A_CASES, ids=["%s-P%d" % (_sid(s), P) for s, P in A_CASES])
def test_overrides_follow_their_pair(pkg, co, sched, P):
    check_overrides(pkg, co, sched, P, seed=100 + P)


@pytest.mark.parametrize("channels,dtype", [(1, np.uint8), (3, np.uint16)], ids=["1ch-u8", "3ch-u16"])
def test_overrides_follow_their_pair_formats(pkg, co, channels, dtype):
    check_overrides(pkg, co, dict(encode_ranges=3), 27, seed=7, channels=channels, dtype=dtype)


# ------------------------------------------------------------------ B. all-raw ranges and chunks, after any earlier call
LAYOUTS = ("first", "middle", "last", "every", "only_last_coded")
PRIORS = ("coded_bigger", "decode_verify", "decode_masks")
B_SCHEDULES = [(dict(encode_ranges=R), 8 * R) for R in (2, 4, 8)] + [(dict(kq_ranges=Q), 8 * Q) for Q in (2, 4)] + \
              [({}, 12)] + [(dict(host_chunk_frames=ch), P) for ch, P in ((2, 8), (3, 12), (7, 28))]


def layout_p(bounds, layout):
    P, m = bounds[-1], len(bounds) - 1
    raw_r = {"first": {0}, "middle": {m // 2}, "last": {m - 1}, "every": set(range(m)), "only_last_coded": set(range(m))}[layout]
    raw = {i for r in raw_r for i in range(bounds[r], bounds[r + 1])}
    p = [raw_p(i) if i in raw or i % 6 == 5 else coded_p(i) for i in range(P)]
    if layout == "only_last_coded":
        p[-1] = coded_p(0)
    return p


def decode_inputs(st, res, n):
    """What decode_masks takes for the pairs of the last encode: packbits bitmaps (the packbits mask for a raw pair) and witnesses."""
    P = len(res)
    bm, wt, mk = st.fetch_batch(0, P, want_masks=True)
    nb = (n + 7) // 8
    bitmaps = np.zeros((P, max(bm.shape[1], (nb + 15) // 16 * 16)), dtype=np.uint8)
    bitmaps[:, :bm.shape[1]] = bm
    for i, r in enumerate(res):
        if r.raw:
            bitmaps[i, :nb] = np.packbits(np.unpackbits(mk[i], bitorder="little")[:n])
    return bitmaps, wt, [r.l for r in res], [r.wlen for r in res], [r.k for r in res], [int(r.raw) for r in res]


def leave_slots(pkg, st, prior, P, seed):
    """Leave the stream's first P slots as the named kind of call wrote them."""
    n = st.npix
    with schedule(pkg):
        if prior == "coded_bigger":                           # every slot: l = n - 1 and a witness of most of the n positions
            fr = make_frames([0.1] * P, seed)
            st.upload(fr)
            res = st.encode_consecutive(P + 1, THR, k_override=[0.3] * P, l_override=[n - 1] * P)
            assert all(not r.raw and r.l == n - 1 and r.wlen > n // 2 for r in res)
            return
        fr = make_frames([0.45 if i % 4 == 3 else 0.1 for i in range(P)], seed)
        st.upload(fr)
        res = st.encode_consecutive(P + 1, THR)
        assert sum(not r.raw for r in res) >= P // 2
        if prior == "decode_verify":
            assert not st.decode_verify().any()
        else:
            _, ones = st.decode_masks(*decode_inputs(st, res, n))
            assert [int(o) for o in ones] == [r.ones for r in res]


@pytest.mark.parametrize("sched,P", B_SCHEDULES, ids=["%s-P%d" % (_sid(s), P) for s, P in B_SCHEDULES])
def test_all_raw_ranges_after_any_earlier_call(pkg, co, sched, P):
    bounds = range_bounds(sched, P)
    follow = make_frames([coded_p(i) for i in range(P)], 500 + P)
    follow_refs = oracle_refs(co, follow)
    st = pkg.FrameStream(H, W, 3, np.uint8, max_frames=P + 1)
    try:
        for li, layout in enumerate(LAYOUTS):
            frames = make_frames(layout_p(bounds, layout), 200 + 10 * li + P)
            refs = oracle_refs(co, frames)
            raw = [r.raw for r in refs]
            if layout == "every":
                assert all(raw)
            elif layout == "only_last_coded":
                assert raw == [True] * (P - 1) + [False]
            else:
                assert not all(raw)
            for prior in PRIORS:
                leave_slots(pkg, st, prior, P, seed=300 + P)
                res, ob, ow = run(pkg, st, sched, frames)
                assert_encode(st, res, refs, ob, ow)
                res, ob, ow = run(pkg, st, sched, follow)        # a fully coded encode afterwards
                assert_encode(st, res, follow_refs, ob, ow)
    finally:
        st.close()


# ------------------------------------------------------------------ C. pair lists that are not one chain
def _walk(P):
    w = [(i // 6) * 2 + (0, 1, 2, 3, 2, 1)[i % 6] for i in range(P + 1)]
    return w[:-1], w[1:]


C_P = 32
PAIR_LISTS = {
    "swapped": lambda P: ([t + 1 for t in range(P)], list(range(P))),
    "reversed_chain": lambda P: ([P - t for t in range(P)], [P - t - 1 for t in range(P)]),
    "revisit": _walk,
    "duplicates": lambda P: ([t // 3 for t in range(P)], [t // 3 + 1 for t in range(P)]),
    # one chain per range of encode_ranges = 4 and 2 (lo[2] = P/2), broken exactly there: not a chain as a whole
    "broken_at_range_boundary": lambda P: ([t if t < P // 2 else t + 5 for t in range(P)], [t + 1 if t < P // 2 else t + 6 for t in range(P)]),
}


@pytest.mark.parametrize("name", list(PAIR_LISTS))
def test_non_chain_pair_lists(pkg, co, name):
    prev, curr = PAIR_LISTS[name](C_P)
    nfr = max(prev + curr) + 1
    frames = make_frames([(0.05, P_RAW, 0.02, 0.0, 0.1, 0.2, 0.01)[t % 7] for t in range(nfr - 1)], 41)
    refs = oracle_refs(co, frames, prev, curr)
    assert any(r.raw for r in refs) and not all(r.raw for r in refs)
    st = pkg.FrameStream(H, W, 3, np.uint8, max_frames=nfr, max_pairs=C_P)
    try:
        for sched in ({}, dict(encode_ranges=2), dict(encode_ranges=4), dict(kq_ranges=4)):
            res, _, _ = run(pkg, st, sched, frames, prev=prev, curr=curr)
            assert_encode(st, res, refs)
    finally:
        st.close()


# ------------------------------------------------------------------ D. which schedule ran
@pytest.mark.parametrize("opt", ["encode_ranges", "kq_ranges"])
def test_split_starts_at_eight_pairs_per_range(pkg, opt):
    """Below 8 pairs per range the encode falls back to the serial one (the same kernel launches); from 8 on it splits (more)."""
    st = pkg.FrameStream(H, W, 3, np.uint8, max_frames=66)
    try:
        for R in (2, 4, 8):
            for P in (8 * R - 1, 8 * R, 8 * R + 1):
                frames = make_frames([coded_p(i) for i in range(P)], 600 + P)
                delta, outs = {}, {}
                for name, sched in (("serial", {}), ("split", {opt: R})):
                    before = launches(pkg)
                    res, _, _ = run(pkg, st, sched, frames)
                    delta[name] = launches(pkg) - before
                    bms, wts, _ = st.fetch_batch(0, P)
                    outs[name] = ([fields(r) for r in res], bms.tobytes(), wts.tobytes())
                assert outs["split"] == outs["serial"], (opt, R, P)
                if P < 8 * R:
                    assert delta["split"] == delta["serial"], (opt, R, P, delta)
                else:
                    assert delta["split"] > delta["serial"], (opt, R, P, delta)
    finally:
        st.close()


def profiled_kernels(fn):
    """Runs fn() under torch.profiler with CUDA activities -> (fn's result, names of the library's kernels in start order).  A torch
    kernel opens the window, synchronised before fn runs: the trace has been seen to lose the first kernels of a window."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device="cuda").add_(1)
        torch.cuda.synchronize()
        out = fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    ks = sorted((e for e in events if e.get("cat") == "kernel" and "rbf::" in e["name"]), key=lambda e: e["ts"])
    return out, [e["name"] for e in ks]


def test_launch_counter_with_all_raw_pieces(pkg):
    """Staging an all-raw range or chunk launches no kernel: the counter still equals the kernels the profiler recorded."""
    st = pkg.FrameStream(H, W, 3, np.uint8, max_frames=65)
    try:
        for sched, P, raw_piece in ((dict(encode_ranges=8), 64, 3), (dict(host_chunk_frames=3), 12, 2)):
            bounds = range_bounds(sched, P)
            raw = range(bounds[raw_piece], bounds[raw_piece + 1])
            frames = make_frames([raw_p(i) if i in raw else coded_p(i) for i in range(P)], 700 + P)
            before = launches(pkg)
            res, ks = profiled_kernels(lambda: run(pkg, st, sched, frames)[0])
            assert all(res[i].raw for i in raw) and not all(r.raw for r in res)
            assert ks and launches(pkg) - before == len(ks), (sched, launches(pkg) - before, ks)
    finally:
        st.close()


# ------------------------------------------------------------------ E. encode_host chunks
E_NFR = 20


def host_layout_p(nframes, ch, seed_shift=0):
    """Chunk 1 codes only its boundary pair p0 = f0 - 1, chunk 2 is all raw, the others mix coded and raw pairs."""
    b = chunk_bounds(nframes, ch)
    p = [raw_p(i) if (i + seed_shift) % 6 == 5 else coded_p(i + seed_shift) for i in range(nframes - 1)]
    for k in (1, 2):
        if k < len(b) - 1:
            for i in range(b[k], b[k + 1]):
                p[i] = raw_p(i)
    if len(b) > 2:
        p[b[1]] = coded_p(1)
    return p


@pytest.mark.parametrize("ch", [2, 3, 7, E_NFR - 1, E_NFR, E_NFR + 5])
def test_encode_host_chunks(pkg, co, ch):
    frames = make_frames(host_layout_p(E_NFR, ch), 800 + ch)
    fewer = make_frames(host_layout_p(13, ch, 3), 900 + ch)           # the next call has fewer frames
    ref_st = pkg.FrameStream(H, W, 3, np.uint8, max_frames=E_NFR)
    st = pkg.FrameStream(H, W, 3, np.uint8, max_frames=E_NFR)
    try:
        for fr in (frames, fewer):
            refs = oracle_refs(co, fr)
            assert any(r.raw for r in refs) and not all(r.raw for r in refs)
            resident, _, _ = run(pkg, ref_st, {}, fr)
            assert_encode(ref_st, resident, refs)
            if fr is frames:
                leave_slots(pkg, st, "coded_bigger", E_NFR - 1, seed=31)
            res, ob, ow = run(pkg, st, dict(host_chunk_frames=ch), fr)
            assert len(res) == len(resident)
            for i, (r, want) in enumerate(zip(res, resident)):
                assert fields(r) == fields(want), (ch, i, fields(r), fields(want))
            assert_encode(st, res, refs, ob, ow)
    finally:
        st.close()
        ref_st.close()


# ------------------------------------------------------------------ F. size
def test_1080p_overrides_all_raw_middle_range(pkg, co):
    """Several witness chunks per pair."""
    check_overrides(pkg, co, dict(encode_ranges=4), 32, seed=13, h=1080, w=1920, raw_ranges=(2,))


def test_4k_overrides_two_ranges(pkg, co):
    check_overrides(pkg, co, dict(encode_ranges=2), 16, seed=17, h=2160, w=3840)
