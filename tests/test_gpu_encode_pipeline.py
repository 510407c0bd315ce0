"""The default pipelined encode (encode_ranges, pipe_k1_sms) against the references at the launch edges it brought in: K1 of
ranges 1.. as wide CTAs of G sweeps on pipe_k1_sms SMs, and K2 of the ranges before the last sized for the SMs K1 leaves free.

A. Wide K1 against the numpy reference mask of test_gpu_k1_edges, every bit of every pair of every range, at tile counts around
   G, G*S and 2*G*S (S = pipe_k1_sms) and chains of every length mod SW_STAGES; both mask modes, gray, every threshold branch.
B. The whole encode against the C oracle fed the numpy reference mask, with S chosen so that range 0's K2 has one frame in its
   partial wave, none, every frame, and several copies of each, and with K2 on one SM.
C. The launches of A and B as torch.profiler saw them: each wide K1 has the block and grid predicted from the kernel headers,
   each K2 the grid predicted for its SM share; and the option clamps.  Without C, an encode that quietly ran the serial
   schedule would pass A and B.

Every schedule runs on a context of its own, created here, so no option set on the process-wide context decides it and none
leaks into it."""
import contextlib
import ctypes as C
import math
import os
import re
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np
import pytest

from tests.test_gpu_encode_schedules import Ref, assert_encode, make_frames
from tests.test_gpu_host_paths import counted_run, profiled_kernels
from tests.test_gpu_k1_edges import EDGE_THRESHOLDS, FORMATS, probe_chain, ref_diff, ref_mask

gpu = pytest.mark.gpu

CSRC = Path(__file__).resolve().parents[1] / "new_bloom_filter_repo_b200" / "csrc"


# ------------------------------------------------------------------ launch geometry, from the sources
def _src(name):
    return (CSRC / name).read_text()


def _int(src, pattern):
    return int(re.search(pattern, src).group(1))


def _geometry():
    k1, kc, k2, api = _src("rbf_k1_threshold.cuh"), _src("rbf_kernels.cu"), _src("rbf_k2_insert.cuh"), _src("rbf_api.cu")
    g = dict(
        SW_THREADS=_int(k1, r"constexpr int SW_THREADS = (\d+);"),
        SW_STAGES=_int(k1, r"constexpr int SW_STAGES = (\d+);"),
        SW_MAX_SWEEPS=_int(k1, r"constexpr int SW_MAX_SWEEPS = (\d+);"),
        MAX_SMEM=_int(kc, r"constexpr int max_smem = (\d+);"),
        K2_CTAS_PER_SM=_int(k2, r"#define RBF_K2_CTAS_PER_SM (\d+)"),
        K2_MAX_CS=_int(k2, r"#define RBF_K2_MAX_CS (\d+)"),
        I2_CAP=_int(k2, r"constexpr int I2_CAP = (\d+);"),
        DEFAULT_R=_int(api, r"int encode_ranges = (\d+);"),
        DEFAULT_S=_int(api, r"int pipe_k1_sms = (\d+);"),
    )
    g["SW_TILE_PX"] = 32 * g["SW_THREADS"]
    g["K2_WARPS"] = 32 // g["K2_CTAS_PER_SM"]
    g["K2_WORDS"] = ((233472 // g["K2_CTAS_PER_SM"] - 1024 - g["K2_WARPS"] * g["I2_CAP"] * 2) // 4) & ~15
    return g


GEO = _geometry()
TILE = GEO["SW_TILE_PX"]


def test_geometry_matches_sources():
    """The formulas below restate these lines; if one of them changes, so must this file."""
    k1, kc, k2, api = _src("rbf_k1_threshold.cuh"), _src("rbf_kernels.cu"), _src("rbf_k2_insert.cuh"), _src("rbf_api.cu")
    for src, line in [
        (k1, "constexpr uint32_t SW_TILE_PX = 32u * SW_THREADS;"),
        (k1, "return (uint32_t)SW_STAGES * SW_TILE_PX * PB + 128u;"),
        (k1, "const uint32_t sweep = blockIdx.x * G + g, nsweeps = gridDim.x * G;"),
        (kc, "constexpr int wide = max_smem / sweep_smem < SW_MAX_SWEEPS ? max_smem / sweep_smem : SW_MAX_SWEEPS;"),
        (kc, "grid = (ntiles + sweeps - 1u) / sweeps;"),
        (kc, "if (grid > (uint32_t)sms) grid = (uint32_t)sms;"),
        (kc, "k_threshold_sweep<PB, S, GRAY><<<grid, SW_THREADS * sweeps, smem, st>>>"),
        (k2, "#define RBF_K2_WARPS (32 / RBF_K2_CTAS_PER_SM)"),
        (k2, "constexpr uint32_t K2_WORDS = ((233472u / K2_CTAS_PER_SM - 1024u - K2_LIST_BYTES) / 4u) & ~15u;"),
        (k2, "constexpr uint32_t K2_LIST_BYTES = (uint32_t)K2_WARPS * I2_CAP * 2u;"),
        (kc, "uint32_t slots = (uint32_t)((int64_t)L.k2_clusters[cs] * (sms < L.sm_count ? sms : L.sm_count) / L.sm_count);"),
        (kc, "const uint32_t full = (uint32_t)F / slots * slots, rem = (uint32_t)F - full;"),
        (kc, "const uint32_t useful = (nslab + cs * K2_WARPS - 1u) / (cs * K2_WARPS);"),
        (kc, "uint32_t copies = rem ? slots / rem : 1u;"),
        (kc, "insert_cluster_config(cs, full + rem * copies, st, &attr);"),
        (api, "if (!strcmp(key, \"encode_ranges\")) { c->encode_ranges = (int)(v < 1 ? 1 : (v > 8 ? 8 : v)); return RBF_OK; }"),
        (api, "if (!strcmp(key, \"pipe_k1_sms\")) { c->pipe_k1_sms = (int)(v < 1 ? 1 : (v > 1024 ? 1024 : v)); return RBF_OK; }"),
        (api, "const int k1_sms = c->pipe_k1_sms < c->L.sm_count ? c->pipe_k1_sms : c->L.sm_count - 1;"),
        (api, "if (pairs < 8u * R) R = 1u;"),
        (api, "r > 0 ? k1_sms : 0, c->st_k1"),
        (api, "r + 1 < R ? c->L.sm_count - k1_sms : c->L.sm_count, c->st"),
    ]:
        assert line in src, line
    assert [G(pb) for pb in (1, 2, 3, 6)] == [4, 4, 4, 2]
    assert GEO["K2_WORDS"] == 49920 and GEO["K2_MAX_CS"] == 1 and (GEO["DEFAULT_R"], GEO["DEFAULT_S"]) == (2, 66)


def G(pb):
    """Sweeps per wide K1 CTA: as many rings of SW_STAGES tiles as fit the opt-in shared memory, SW_MAX_SWEEPS at most."""
    return min(GEO["MAX_SMEM"] // (GEO["SW_STAGES"] * TILE * pb + 128), GEO["SW_MAX_SWEEPS"])


def pb_of(fmt):
    c, dt = FORMATS[fmt]
    return c * np.dtype(dt).itemsize


def ranges_of(opt_r, P):
    """encode_ranges as set (clamped to 1..8) -> the ranges an encode of P pairs runs, as [lo, hi) pair bounds."""
    R = min(max(opt_r, 1), 8)
    if P < 8 * R:
        R = 1
    lo = [P * r // R for r in range(R + 1)]
    return list(zip(lo[:-1], lo[1:]))


def k1_sms(opt_s, sm):
    """pipe_k1_sms as set (clamped to 1..1024) -> the SMs K1 of ranges 1.. runs on: never all of them."""
    s = min(max(opt_s, 1), 1024)
    return s if s < sm else sm - 1


def ntiles(npix):
    return -(-npix // TILE)


def wide_k1(pb, npix, sms):
    """(grid, block) of a wide K1 launch."""
    return (min(-(-ntiles(npix) // G(pb)), sms), 1, 1), (GEO["SW_THREADS"] * G(pb), 1, 1)


def k2_plan(F, sms, sm, npix, max_l):
    """launch_insert of F frames on `sms` of the `sm` SMs -> (slots, full, rem, copies, units).  One K2 CTA per SM (its shared
    memory), clusters of one CTA: sm * K2_CTAS_PER_SM resident clusters."""
    words = -(-max_l // 32)
    assert words <= 2 * GEO["K2_MAX_CS"] * GEO["K2_WORDS"], "the arrays go to k_insert2, not the cluster kernel"
    cs = min(max(-(-words // GEO["K2_WORDS"]), 1), GEO["K2_MAX_CS"])
    assert cs == 1, "the resident clusters of cs > 1 are measured, not predicted"
    slots = max(sm * GEO["K2_CTAS_PER_SM"] * min(sms, sm) // sm, 1)
    full = F // slots * slots
    rem = F - full
    nslab = -(-(-(-npix // 100)) // 32)
    useful = -(-nslab // (cs * GEO["K2_WARPS"]))
    copies = max(min(slots // rem if rem else 1, useful), 1)
    return slots, full, rem, copies, full + rem * copies


# ------------------------------------------------------------------ contexts
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


@pytest.fixture(scope="module")
def contexts(pkg):
    """contexts(R, S) -> a fresh context with encode_ranges = R and pipe_k1_sms = S, one per (R, S), destroyed at the end."""
    L = pkg._cabi.lib()
    dev = int(os.environ.get("RBF_DEVICE", os.environ.get("LOCAL_RANK", "0")))   # the device of _cabi.ctx()
    made = {}

    def get(R, S):
        if (R, S) not in made:
            h = C.c_void_p()
            pkg._cabi.check(L.rbf_ctx_create(dev, C.byref(h)))
            made[(R, S)] = h
            pkg._cabi.check(L.rbf_set_option(h, b"encode_ranges", int(R)), h)
            pkg._cabi.check(L.rbf_set_option(h, b"pipe_k1_sms", int(S)), h)
        return made[(R, S)]
    try:
        yield get
    finally:
        for h in made.values():
            L.rbf_ctx_destroy(h)


@contextlib.contextmanager
def on_ctx(pkg, h):
    """FrameStreams created and used inside take their context (and their error messages) from h."""
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(pkg._cabi, "ctx", lambda: h)
        yield


@pytest.fixture(scope="module")
def sm_count(pkg):
    return pkg._cabi.device_info()["sm_count"]


# ------------------------------------------------------------------ A. wide K1 against the numpy reference
def chain_frames(fmt, npix, nfr):
    """probe_chain [nfr, 1, npix(, C)], with frame t >= 1 also changed at every 61st pixel from (13 t) mod 61 on: the Y sample's
    top and bottom bits flipped.  probe_chain alone repeats with period 2 (every pair is the probe pair, either way round, but
    for its last pixel), so a sweep that compared frames two apart in its ring would still write the right masks; with the
    marks every pair's mask is its own."""
    c, dt = FORMATS[fmt]
    fr = probe_chain(fmt, npix, nfr)
    flat = fr.reshape(nfr, npix, c)
    mark = dt(np.iinfo(dt).max // 2 + 2)
    for t in range(1, nfr):
        flat[t, (13 * t) % 61::61, 0] ^= mark
    return fr.reshape((nfr, 1, npix, c) if c == 3 else (nfr, 1, npix))


def ragged_npix(T):
    """A frame of T tiles whose last tile and last mask word are both partial, and whose last tile's bulk copy ends at a
    different 16 B remainder for different T."""
    return T * TILE - 45 - 2 * T


def tile_edges(g, s):
    return sorted({max(1, x) for x in (1, g - 1, g, g + 1, g * s - 1, g * s, g * s + 1, 2 * g * s + 1)})


def modes(fmt):
    return [(0, False), (1, False)] + ([(0, True), (1, True)] if FORMATS[fmt][0] == 3 else [])


P_R2 = (16, 17, 19, 21)       # range 1 holds 8, 9, 10, 11 pairs: chains of 9, 10, 11, 12 frames, every length mod SW_STAGES
P_R8 = (67,)                  # eight ranges of 8 or 9 pairs: seven wide launches back to back on the K1 stream
A_CASES = ([(fmt, s, 2, P_R2, tuple(tile_edges(G(pb_of(fmt)), s))) for fmt in FORMATS for s in (1, 3)]
           + [(fmt, GEO["DEFAULT_S"], 2, P_R2, (G(pb_of(fmt)) * 66 - 1, G(pb_of(fmt)) * 66 + 1)) for fmt in ("u8x3", "u16x3")]
           + [(fmt, 3, 8, P_R8, (1, 2 * G(pb_of(fmt)) * 3 + 1)) for fmt in FORMATS])


def _aid(case):
    fmt, s, r, ps, tiles = case
    return "%s-S%d-R%d" % (fmt, s, r)


def test_a_cases_reach_every_edge():
    for fmt in FORMATS:
        g = G(pb_of(fmt))
        for s in (1, 3):
            tiles = {t for f, ss, r, _, ts in A_CASES if f == fmt and ss == s and r == 2 for t in ts}
            assert tiles == {max(1, x) for x in (1, g - 1, g, g + 1, g * s - 1, g * s, g * s + 1, 2 * g * s + 1)}
        assert any(f == fmt and r == 8 for f, _, r, _, _ in A_CASES)
    for fmt in ("u8x3", "u16x3"):
        g = G(pb_of(fmt))
        assert {g * 66 - 1, g * 66 + 1} <= {t for f, s, _, _, ts in A_CASES if f == fmt and s == 66 for t in ts}
    for _, _, r, ps, tiles in A_CASES:
        for T in tiles:
            n = ragged_npix(T)
            assert ntiles(n) == T and n % TILE and n % 32
        for P in ps:
            assert len(ranges_of(r, P)) == r                       # the encode splits
    frames_r1 = {(hi - lo + 1) % GEO["SW_STAGES"] for P in P_R2 for lo, hi in ranges_of(2, P)[1:]}
    assert frames_r1 == set(range(GEO["SW_STAGES"]))


def test_chain_frames_make_every_pair_distinct():
    for fmt in FORMATS:
        npix = 3 * TILE + 77
        fr = chain_frames(fmt, npix, 23)
        diff = [ref_diff(fr[t], fr[t + 1])[0] for t in range(22)]
        for t in range(22):
            for u in range(t + 1, 22):
                assert (diff[t] != diff[u]).sum() > npix // 100, (fmt, t, u)


def chain_diffs(frames, npairs, gray):
    return [ref_diff(frames[t], frames[t + 1], gray) for t in range(npairs)]


def k1_expected(diffs, thr, mask_mode):
    """[(mask bool [npix], ones, resid) per pair] at one threshold."""
    return [ref_mask(d, a, thr, mask_mode) for d, a in diffs]


def check_k1_out(st, res, exp, npix, where):
    """Every mask bit, the padding bits past npix, ones and resid of each pair of the last encode."""
    P = len(res)
    _, _, mk = st.fetch_batch(0, P, want_masks=True)
    bits = np.unpackbits(mk, axis=1, bitorder="little")
    for t in range(P):
        em, eones, eresid = exp[t]
        bad = np.flatnonzero(bits[t, :npix] != em.reshape(-1))
        assert bad.size == 0, (where, "pair", t, "first wrong mask bits", bad[:8].tolist())
        assert not bits[t, npix:].any(), (where, "pair", t, "padding bits past npix are set")
        assert (res[t].ones, res[t].resid) == (eones, eresid), (where, "pair", t)


def k1_stream(pkg, fmt, npix, nfr):
    c, dt = FORMATS[fmt]
    return pkg.FrameStream(1, npix, c, dt, max_frames=nfr, max_pairs=nfr - 1, k1_only=True)


@gpu
@pytest.mark.parametrize("case", A_CASES, ids=[_aid(c) for c in A_CASES])
def test_wide_k1_matches_reference(pkg, contexts, case):
    fmt, s, r, ps, tiles = case
    h = contexts(r, s)
    pmax = max(ps)
    for T in tiles:
        npix = ragged_npix(T)
        frames = chain_frames(fmt, npix, pmax + 1)
        with on_ctx(pkg, h):
            st = k1_stream(pkg, fmt, npix, pmax + 1)
            try:
                st.upload(frames)
                for mask_mode, gray in modes(fmt):
                    st.set_option("mask_mode", mask_mode)
                    st.set_option("gray_mode", int(gray))
                    diffs = chain_diffs(frames, pmax, gray)
                    for thr in EDGE_THRESHOLDS:
                        exp = k1_expected(diffs, thr, mask_mode)
                        for P in ps:
                            res = st.encode_consecutive(P + 1, thr)
                            check_k1_out(st, res, exp[:P], npix, (fmt, T, npix, s, r, P, mask_mode, gray, thr))
            finally:
                st.close()


# ------------------------------------------------------------------ B. the whole encode against the C oracle
B_H, B_W = 540, 960           # 518 400 px: 162 slabs of 32 centuries, so K2 can use up to 6 copies of a frame
B_P, B_R = 32, 2
B_F0 = B_P // B_R             # range 0's pairs: the F of its K2
THR = 3.0
B_PMIX = (0.05, 0.02, 0.45, 0.1, 0.0, 0.2, 0.01, 0.03)       # coded, plus raw pairs: p >= p* (0.45) and no change (0.0)
B_MODES = {"u8x3": [(0, False), (1, False), (0, True), (1, True)], "u16x3": [(0, False), (1, True)]}
B_TARGETS = ("rem1", "whole_waves", "all_partial", "third", "one_sm")
B_CASES = [("u8x3", t) for t in B_TARGETS] + [("u16x3", "rem1"), ("u16x3", "one_sm")]


def b_pipe_sms(target, sm):
    """pipe_k1_sms that gives range 0's K2 (F0 frames on sm - S SMs) the named wave shape."""
    if target == "one_sm":
        return sm - 1
    if target == "third":                      # about F0 / 3 slots, with a partial wave of several copies per frame
        ok = [x for x in range(2, B_F0) if k2_plan(B_F0, x, sm, B_H * B_W, 1)[3] > 1]
        return sm - min(ok, key=lambda x: abs(3 * x - B_F0))
    return sm - {"rem1": B_F0 - 1, "whole_waves": B_F0, "all_partial": B_F0 + 1}[target]


def test_b_targets_reach_every_wave_shape():
    """On the 132 SMs of an H100 SXM (the test itself uses the device's count)."""
    sm, n = 132, B_H * B_W
    plan = {t: k2_plan(B_F0, sm - b_pipe_sms(t, sm), sm, n, 1) for t in B_TARGETS}
    assert plan["rem1"][2] == 1 and plan["rem1"][3] > 1
    assert plan["whole_waves"][2] == 0 and plan["whole_waves"][4] == B_F0
    assert plan["all_partial"][1] == 0 and plan["all_partial"][2] == B_F0
    assert plan["third"][3] > 1 and abs(3 * plan["third"][0] - B_F0) <= 3
    assert plan["one_sm"][0] == 1
    last = k2_plan(B_P - B_F0, sm, sm, n, 1)                    # the last range: every SM, copies capped by `useful`
    assert last[1] == 0 and last[3] == 6
    assert ranges_of(B_R, B_P)[0] == (0, B_F0)


def oracle_from_mask(co, m, ones, resid):
    """Ref (as test_gpu_encode_schedules builds it) of a pair whose mask is m: co.compress decides (p, k, l, bitmap, witness)."""
    flat = m.reshape(-1).astype(np.uint8)
    ob, ow, p, _, _, k, l = co.compress(flat)
    r = Ref()
    r.mask, r.ones, r.resid, r.p = flat, ones, resid, p
    r.raw = l == 0
    r.k, r.l = float(k), int(l)
    r.wlen = 0 if r.raw else len(ow)
    r.floor_k = 0 if r.raw else int(math.floor(k))
    r.act_T = 0 if r.raw else co.activation_threshold(k - math.floor(k))
    r.bitmap = b"" if r.raw else np.packbits(ob).tobytes()
    r.witness = b"" if r.raw else np.packbits(ow).tobytes()
    return r


class BRefs:
    """The frames of B per format and their oracle per (format, mask_mode, gray), computed once for the module."""

    def __init__(self, co):
        self.co, self._frames, self._refs = co, {}, {}

    def frames(self, fmt):
        if fmt not in self._frames:
            c, dt = FORMATS[fmt]
            p = [B_PMIX[i % len(B_PMIX)] for i in range(B_P)]
            self._frames[fmt] = make_frames(p, 61 + len(self._frames), B_H, B_W, c, dt)
        return self._frames[fmt]

    def refs(self, fmt, mask_mode, gray):
        key = (fmt, mask_mode, gray)
        if key not in self._refs:
            fr = self.frames(fmt)

            def one(t):
                return oracle_from_mask(self.co, *ref_mask(*ref_diff(fr[t], fr[t + 1], gray), THR, mask_mode))
            with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
                refs = list(ex.map(one, range(B_P)))
            for lo, hi in ranges_of(B_R, B_P):                 # every range launches K2
                assert not all(r.raw for r in refs[lo:hi]), key
            assert any(r.raw for r in refs), key
            self._refs[key] = refs
        return self._refs[key]


@pytest.fixture(scope="module")
def brefs(co):
    return BRefs(co)


def check_b_encode(st, res, refs, npix, where):
    assert_encode(st, res, refs)
    _, _, mk = st.fetch_batch(0, len(refs), want_masks=True)
    bits = np.unpackbits(mk, axis=1, bitorder="little")
    for t, o in enumerate(refs):
        assert np.array_equal(bits[t, :npix], o.mask), (where, "mask row", t)
        assert not bits[t, npix:].any(), (where, "padding bits past npix are set", t)


@gpu
@pytest.mark.parametrize("fmt,target", B_CASES, ids=["%s-%s" % c for c in B_CASES])
def test_encode_matches_oracle_at_k2_wave_edges(pkg, contexts, brefs, sm_count, fmt, target):
    c, dt = FORMATS[fmt]
    s = b_pipe_sms(target, sm_count)
    frames = brefs.frames(fmt)
    with on_ctx(pkg, contexts(B_R, s)):
        st = pkg.FrameStream(B_H, B_W, c, dt, max_frames=B_P + 1)
        try:
            st.upload(frames)
            for mask_mode, gray in B_MODES[fmt]:
                refs = brefs.refs(fmt, mask_mode, gray)
                st.set_option("mask_mode", mask_mode)
                st.set_option("gray_mode", int(gray))
                res = st.encode_consecutive(B_P + 1, THR)
                check_b_encode(st, res, refs, B_H * B_W, (fmt, target, s, mask_mode, gray))
        finally:
            st.close()


# ------------------------------------------------------------------ C. what was launched
K1_RE = re.compile(r"k_threshold_sweep<\s*(?:\(int\))?(\d+)\s*,\s*(?:\(int\))?(\d+)\s*,\s*(true|false|\(bool\)[01])\s*>")


def check_launches(name, launched, ks, pb, gray, npix, rngs, S, sm, k2=None):
    """ks: (kernel, grid, block) of one encode in start order.  rngs: its ranges; S: pipe_k1_sms as set; k2: (max_l per range)
    of a coded encode."""
    assert ks and launched == len(ks), (name, "kernel_launches", launched, "kernels traced", len(ks))
    k1 = [k for k in ks if "k_threshold" in k[0]]
    assert len(k1) == len(rngs), (name, [k[0][:60] for k in k1])
    sms = k1_sms(S, sm)
    for r, (kname, grid, block) in enumerate(k1):
        m = K1_RE.search(kname)
        assert m, (name, "not the sweep", kname)
        assert (int(m.group(1)), m.group(3) in ("true", "(bool)1")) == (pb, gray), (name, kname)
        if r == 0:
            assert block == (GEO["SW_THREADS"], 1, 1) and grid[0] <= ntiles(npix), (name, "range 0 is one sweep per CTA", grid, block)
        else:
            assert (grid, block) == wide_k1(pb, npix, sms), (name, "range", r, grid, block, wide_k1(pb, npix, sms))
    k2s = [k for k in ks if "k_insert" in k[0]]
    if k2 is None:
        assert not k2s, (name, k2s)
        return
    assert len(k2s) == len(rngs) and all("k_insert_cluster" in k[0] for k in k2s), (name, [k[0][:60] for k in k2s])
    for r, ((lo, hi), (kname, grid, block)) in enumerate(zip(rngs, k2s)):
        share = sm - sms if r + 1 < len(rngs) else sm
        units = k2_plan(hi - lo, share, sm, npix, k2[r])[4]
        assert (grid, block) == ((1, units, 1), (32 * GEO["K2_WARPS"], 1, 1)), (name, "K2 of range", r, grid, block, units)


@gpu
def test_launch_shapes(pkg, contexts, brefs, sm_count):
    sm = sm_count
    c_cases = []                    # (name, R, S, fmt, T, P, mask_mode, gray)
    for fmt, s, r, ps, tiles in A_CASES:
        for T in tiles:
            for gray in (False, True) if FORMATS[fmt][0] == 3 else (False,):
                c_cases.append(("A %s T%d S%d R%d gray%d" % (fmt, T, s, r, gray), r, s, fmt, T, ps[0], 0, gray))
    g16 = G(pb_of("u16x3"))
    c_cases += [("clamp pipe_k1_sms 0", 2, 0, "u8x3", 2 * G(3) + 1, 16, 0, False),
                ("clamp pipe_k1_sms sm", 2, sm, "u16x3", g16 * (sm - 1) + 1, 16, 0, False),
                ("clamp pipe_k1_sms 5000", 2, 5000, "u16x3", g16 * (sm - 1) + 1, 16, 1, True),
                ("clamp encode_ranges 0", 0, 66, "u8x1", 5, 16, 0, False),
                ("clamp encode_ranges 9", 9, 3, "u16x1", 5, 64, 1, False)]
    expect = {}

    def run(counts):
        for name, r, s, fmt, T, P, mask_mode, gray in c_cases:
            npix = ragged_npix(T)
            frames = chain_frames(fmt, npix, P + 1)
            with on_ctx(pkg, contexts(r, s)):
                st = k1_stream(pkg, fmt, npix, P + 1)
                try:
                    st.upload(frames)
                    st.set_option("mask_mode", mask_mode)
                    st.set_option("gray_mode", int(gray))
                    res = counted_run(pkg, lambda: st.encode_consecutive(P + 1, 0.0), name, counts)
                    check_k1_out(st, res, k1_expected(chain_diffs(frames, P, gray), 0.0, mask_mode), npix, name)
                finally:
                    st.close()
            expect[name] = (pb_of(fmt), gray, npix, ranges_of(r, P), s, None)
        for fmt, target in B_CASES:
            c, dt = FORMATS[fmt]
            s = b_pipe_sms(target, sm)
            mask_mode, gray = B_MODES[fmt][-1]
            refs = brefs.refs(fmt, mask_mode, gray)
            name = "B %s %s S%d" % (fmt, target, s)
            with on_ctx(pkg, contexts(B_R, s)):
                st = pkg.FrameStream(B_H, B_W, c, dt, max_frames=B_P + 1)
                try:
                    st.upload(brefs.frames(fmt))
                    st.set_option("mask_mode", mask_mode)
                    st.set_option("gray_mode", int(gray))
                    res = counted_run(pkg, lambda: st.encode_consecutive(B_P + 1, THR), name, counts)
                    check_b_encode(st, res, refs, B_H * B_W, name)
                finally:
                    st.close()
            rngs = ranges_of(B_R, B_P)
            max_l = [max(o.l for o in refs[lo:hi]) for lo, hi in rngs]
            expect[name] = (pb_of(fmt), gray, B_H * B_W, rngs, s, max_l)

    seen = profiled_kernels(run)
    assert sorted(seen) == sorted(expect)
    for name, (pb, gray, npix, rngs, s, k2) in expect.items():
        launched, ks = seen[name]
        check_launches(name, launched, ks, pb, gray, npix, rngs, s, sm, k2)
    assert len(ranges_of(0, 16)) == 1 and len(ranges_of(9, 64)) == 8
    assert wide_k1(3, ragged_npix(2 * G(3) + 1), k1_sms(0, sm))[0] == (1, 1, 1)
    assert wide_k1(6, ragged_npix(g16 * (sm - 1) + 1), k1_sms(sm, sm))[0] == (sm - 1, 1, 1)
