"""FrameStream.decode_verify against an oracle decode of altered bit arrays: exact mismatch counts at every query kernel, witness
chunk and encode path, and the encode's outputs intact afterwards.

decode_verify (rbf_stream_decode_verify) decodes every pair of the last encode from its own bitmap and witness on the device (K3
query, K3b pass counts, K4b k_expand) and counts the 32-bit mask words in which the decode differs from the encoded mask
(k_count_diff).  After an unaltered encode every count is 0, so a verifier that always says 0 would pass every other test.  Here
the bitmaps are altered in place on the device, through rbf_stream_bitmap_region, and each count is compared with a model that
shares nothing with the library:
  * pass = the C oracle's pass mask of the altered bit array (orc_decompress_kl with an all-ones witness of n bits),
  * decoded[i] = w[rank(i)] where pass[i] and rank(i) < wlen, else 0 (witness bits at or past wlen read as 0, as k_expand does),
  * count = the ceil(n/32) little-endian words in which decoded differs from the encoded mask M.
M, w, wlen and (k, l) are the library's own outputs (fetch_batch, the pair results).  Raw pairs report 0.  Edits stay inside
pair slots [0, pairs) and inside each slot's first ceil(l/8) bytes: only bytes the library reads are touched."""
import contextlib
import ctypes as C
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

THR = 3.0
VARIANTS = (0, 1, 5, 6)
# the context's defaults (rbf_api.cu); every test here sets what it needs and puts these back
CTX_DEFAULTS = dict(query_variant=5, query_warps=0, query_smem_bytes=0, encode_ranges=2, kq_ranges=1, host_chunk_frames=32)


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
def options(pkg, **opts):
    L, ctx = pkg._cabi.lib(), pkg._cabi.ctx()
    try:
        for k, v in opts.items():
            pkg._cabi.check(L.rbf_set_option(ctx, k.encode(), int(v)), ctx)
        yield
    finally:
        for k in opts:
            L.rbf_set_option(ctx, k.encode(), CTX_DEFAULTS[k])


# ------------------------------------------------------------------ the device bit arrays
class _DeviceBytes:
    """A device byte range torch can wrap without a copy."""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": "|u1", "data": (ptr, False), "version": 3, "strides": None}


def bitmap_region(pkg, st, pairs):
    """-> uint8 CUDA tensor [pairs, stride] over the stream's bitmap slots (pair i's packbits-order bitmap starts at row i)."""
    import torch
    ptr, stride = C.c_void_p(), C.c_uint64()
    pkg._cabi.check(pkg._cabi.lib().rbf_stream_bitmap_region(st._h, C.byref(ptr), C.byref(stride)), pkg._cabi.ctx())
    assert ptr.value and stride.value % 128 == 0 and stride.value >= (st.npix + 7) // 8
    t = torch.as_tensor(_DeviceBytes(ptr.value, (int(pairs), int(stride.value))), device="cuda")
    assert t.data_ptr() == ptr.value
    return t


def read_region(region):
    import torch
    torch.cuda.synchronize()
    return region.cpu().numpy()


def write_bitmaps(region, edits, ls):
    """edits: {pair: packed bitmap}; each write covers the pair's first ceil(l/8) bytes only."""
    import torch
    for i, bm in edits.items():
        nb = (ls[i] + 7) // 8
        assert bm.shape == (nb,), (i, bm.shape, nb)
        region[i, :nb] = torch.from_numpy(np.ascontiguousarray(bm)).to(region.device)
    torch.cuda.synchronize()


# ------------------------------------------------------------------ the model
def oracle_pass(co, bits, n, k):
    """The oracle's pass mask of a bit array (one byte per bit): orc_decompress_kl with an all-ones witness of n bits."""
    bits = np.ascontiguousarray(bits, dtype=np.uint8)
    wit = np.ones(n, dtype=np.uint8)
    out = np.empty(n, dtype=np.uint8)
    co.lib().orc_decompress_kl(co._ptr(bits), bits.size, co._ptr(wit), n, n, float(k), *[int(s) for s in co.IVC_SEEDS], co._ptr(out))
    return out


def diff_words(a, b):
    """Number of 32-bit little-endian words of two n-bit masks (one byte per bit) that differ; bits past n are zero in both."""
    n = a.size
    nw = -(-n // 32)
    d = np.zeros(32 * nw, dtype=bool)
    d[:n] = a != b
    return int(d.reshape(nw, 32).any(axis=1).sum())


def model_count(co, bm_packed, l, n, k, mask, wit_packed, wlen):
    """Mismatch words of the decode of bit array bm_packed (np.packbits order, l bits) with witness wit_packed (wlen bits)."""
    pas = oracle_pass(co, np.unpackbits(bm_packed)[:l], n, k).astype(bool)
    rank = np.cumsum(pas, dtype=np.int64) - 1
    w = np.unpackbits(wit_packed)[:wlen]
    dec = np.zeros(n, dtype=np.uint8)
    sel = pas & (rank < wlen)
    dec[sel] = w[rank[sel]]
    return diff_words(dec, mask)


def model_counts(co, edits, infos, masks, wts):
    """{pair: expected count} of every edited pair, the oracle runs side by side (ctypes releases the GIL)."""
    co.lib()
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        fut = {i: ex.submit(model_count, co, bm, infos[i].l, infos[i].n, infos[i].k, masks[i], wts[i], infos[i].wlen)
               for i, bm in edits.items()}
        return {i: f.result() for i, f in fut.items()}


# ------------------------------------------------------------------ edits of a packed bit array
def get_bit(bm, b):
    return (int(bm[b >> 3]) >> (7 - (b & 7))) & 1


def with_bit(bm, b, v):
    out = bm.copy()
    if v:
        out[b >> 3] |= 0x80 >> (b & 7)
    else:
        out[b >> 3] &= ~(0x80 >> (b & 7)) & 0xFF
    return out


def h1(co, i, l):
    """The first probe of position i (with k = 1.0 its only one: floor_k 1, no activation)."""
    return co.xxh64(str(int(i)).encode(), co.IVC_SEEDS[0]) % l


def clear_set_bit(bm, l, rng):
    """Clear one set bit.  Only members set bits, so some member probes it: that member fails and the later ranks shift."""
    ones = np.flatnonzero(np.unpackbits(bm)[:l])
    return with_bit(bm, int(ones[rng.integers(ones.size)]), 0)


def set_clear_bit_k1(co, bm, l, mask, start):
    """k = 1.0: set the clear bit of the first non-member at or after `start` whose bit is clear; it passes from now on."""
    for j in range(start, mask.size):
        if not mask[j]:
            b = h1(co, j, l)
            if not get_bit(bm, b):
                return with_bit(bm, b, 1), j
    raise AssertionError("no non-member with a clear bit")


def all_bits(l, v):
    return np.packbits(np.full(l, v, dtype=np.uint8))


def flip_padding(bm, l):
    """Flip the bits [l, 8*ceil(l/8)) of the last byte, which no probe reads."""
    assert l % 8
    out = bm.copy()
    out[-1] ^= (1 << (8 - l % 8)) - 1
    return out


def last_century_edit_k1(co, bm, l, n, mask):
    """k = 1.0: clear the bit of a member in the last (ragged) century that no earlier position probes, so the first position
    the edit affects lies in that century.  The earlier probers of the candidate bits come from one oracle pass over an array
    holding only those bits."""
    s0 = 100 * ((n - 1) // 100)
    cand = {}
    for j in range(s0, n):
        if mask[j]:
            cand.setdefault(h1(co, j, l), j)
    only = np.zeros(l, dtype=np.uint8)
    only[list(cand)] = 1
    probers = np.flatnonzero(oracle_pass(co, only, n, 1.0))
    for i in probers[probers < s0]:
        cand.pop(h1(co, i, l), None)
    assert cand, "no member bit of the last century is free of earlier probers"
    b = min(cand)
    assert get_bit(bm, b)
    return with_bit(bm, b, 0), cand[b]


# ------------------------------------------------------------------ streams
def chain_frames(masks, H, W):
    """Frames whose pair t changes by |dY| = 128 exactly where masks[t] is set (one channel, threshold 3)."""
    frames = np.zeros((len(masks) + 1, H, W), dtype=np.uint8)
    for t, m in enumerate(masks):
        frames[t + 1] = frames[t] ^ (m.reshape(H, W) << 7)
    return frames


def fetch_all(st, F):
    bms, wts, mks = st.fetch_batch(0, F, want_masks=True)
    masks = [np.unpackbits(mks[i], bitorder="little")[:st.npix] for i in range(F)]
    return bms, wts, masks


def check_region_contract(region, bms, res):
    """Before any edit, the region is fetch_batch's bitmaps byte for byte at the reported stride, and zero past each payload."""
    got = read_region(region)
    for i, r in enumerate(res):
        nb = 0 if r.raw else (r.l + 7) // 8
        assert np.array_equal(got[i, :bms.shape[1]], bms[i]), i
        assert not got[i, nb:].any(), (i, nb)


def coded_bitmaps(bms, res):
    return {i: bms[i, :(r.l + 7) // 8].copy() for i, r in enumerate(res) if not r.raw}


def check_intact(st, res, bms_want, wts_want, F):
    """fetch_batch returns the given bitmaps (edits included) and the encode's witnesses."""
    bms, wts, _ = st.fetch_batch(0, F)
    for i, r in enumerate(res):
        if r.raw:
            assert not bms[i].any() and not wts[i].any(), i
            continue
        nb, nw = (r.l + 7) // 8, (r.wlen + 7) // 8
        assert np.array_equal(bms[i, :nb], bms_want[i]), i
        assert np.array_equal(wts[i, :nw], wts_want[i, :nw]), i
        assert not bms[i, nb:].any() and not wts[i, nw:].any(), i


# ------------------------------------------------------------------ A + B. kinds of edit at every query kernel and regime
# (H, W, l, query_smem_bytes): a few words; the whole array in shared memory; most of it in L2; half-decade tiles
# (2^23 < l <= 2^24); rings (l > 2^24).  Every n is ragged (n % 100 and n % 32 non-zero) and l is not a multiple of 8.
REGIMES = {
    "words": (9, 13, 77, 0),
    "smem": (270, 483, 100_003, 0),
    "l2": (270, 483, 100_003, 16),
    "half": (2901, 3001, 8_400_007, 0),
    "rings": (4099, 4111, 16_784_217, 0),
}
# pair: (role, k); raw pairs have p >= p* whatever the override
A_PAIRS = [("control", 3.0), ("clear", 3.19), ("set", 1.0), ("raw", 0.0), ("zeros", 2.5), ("ones", 4.71), ("padding", 2.0),
           ("last", 1.0), ("control", 0.37)]


def regime_masks(n, seed):
    rng = np.random.default_rng(seed)
    s0 = 100 * ((n - 1) // 100)
    masks = []
    for role, _ in A_PAIRS:
        m = (rng.random(n) < (0.45 if role == "raw" else 0.05)).astype(np.uint8)
        if role != "raw":
            m[s0::3] = 1                                    # members in the last century
        masks.append(m)
    return masks


def plan_edits(co, bms, res, masks, rng):
    """The edit of every role in A_PAIRS -> {pair: packed bitmap}, and the position the last-century edit is for."""
    edits, note = {}, {}
    for i, (role, _) in enumerate(A_PAIRS):
        r = res[i]
        if role in ("control", "raw"):
            continue
        bm = bms[i, :(r.l + 7) // 8].copy()
        if role == "clear":
            edits[i] = clear_set_bit(bm, r.l, rng)
        elif role == "set":
            edits[i], note["set"] = set_clear_bit_k1(co, bm, r.l, masks[i], r.n // 4)
        elif role == "zeros":
            edits[i] = all_bits(r.l, 0)
        elif role == "ones":
            edits[i] = all_bits(r.l, 1)
        elif role == "padding":
            edits[i] = flip_padding(bm, r.l)
        elif role == "last":
            edits[i], note["last"] = last_century_edit_k1(co, bm, r.l, r.n, masks[i])
    return edits, note


@pytest.mark.parametrize("regime", list(REGIMES))
def test_edit_kinds_at_every_query_kernel(pkg, co, regime):
    H, W, l, smem = REGIMES[regime]
    n, F = H * W, len(A_PAIRS)
    assert n % 32 and n % 100 and l % 8 and l < n
    masks = regime_masks(n, 1000 + l)
    st = pkg.FrameStream(H, W, 1, np.uint8, max_frames=F + 1, max_pairs=F)
    try:
        st.upload(chain_frames(masks, H, W))
        res = st.encode(list(range(F)), list(range(1, F + 1)), THR, k_override=[k for _, k in A_PAIRS],
                        l_override=[0 if role == "raw" else l for role, _ in A_PAIRS])
        assert [r.raw for r in res] == [role == "raw" for role, _ in A_PAIRS]
        assert all(r.l == l and r.k == k for r, (role, k) in zip(res, A_PAIRS) if role != "raw")
        bms, wts, got_masks = fetch_all(st, F)
        for i in range(F):
            assert np.array_equal(got_masks[i], masks[i]), i
        region = bitmap_region(pkg, st, F)
        check_region_contract(region, bms, res)
        for v in VARIANTS:
            with options(pkg, query_variant=v, query_smem_bytes=smem):
                assert not st.decode_verify().any(), v
        edits, note = plan_edits(co, bms, res, got_masks, np.random.default_rng(l))
        exp = model_counts(co, edits, res, got_masks, wts)
        want = [exp.get(i, 0) for i in range(F)]
        role = {r: i for i, (r, _) in enumerate(A_PAIRS) if r not in ("control", "raw")}
        # the model itself: an edit that drops a member or adds a pass changes the decode; an all-zero array (floor k >= 1) decodes
        # to the zero mask; padding is never read
        for r in ("clear", "set", "zeros", "ones", "last"):
            assert want[role[r]] > 0, (r, want)
        assert want[role["zeros"]] == diff_words(np.zeros(n, np.uint8), got_masks[role["zeros"]])
        assert want[role["padding"]] == 0
        assert note["last"] >= 100 * ((n - 1) // 100) and note["set"] >= n // 4
        write_bitmaps(region, edits, [r.l for r in res])
        for v in VARIANTS:
            with options(pkg, query_variant=v, query_smem_bytes=smem):
                got = st.decode_verify()
            assert got.tolist() == want, (v, got.tolist(), want)
        after = coded_bitmaps(bms, res)
        after.update(edits)
        check_intact(st, res, after, wts, F)
    finally:
        st.close()


# ------------------------------------------------------------------ C. K4b witness chunks
def witness_chunks(F, ncent, sm):
    """Chunks per frame of K3b / K4b (witness_chunks in rbf_kernels.cu): >= 8 waves of the GPU, >= 4096 centuries a chunk, <= 32."""
    return max(1, min(-(-16 * sm // F), ncent // 4096, 32))


def chunk_starts(ncent, chunks):
    """First century of every chunk but the first."""
    return [ncent * x // chunks for x in range(1, chunks)]


def boundary_edit_k1(co, bm, l, mask, c_last, c_first):
    """k = 1.0: clear the bit of a member in century c_last (the last of a chunk) and set the clear bit of a non-member in century
    c_first (the first of the next): the pass counts of both chunks change."""
    n = mask.size
    j = next(j for j in range(min(100 * c_last + 99, n - 1), 100 * c_last - 1, -1) if mask[j])
    cleared = h1(co, j, l)
    bm = with_bit(bm, cleared, 0)
    for j in range(100 * c_first, min(100 * c_first + 100, n)):
        b = h1(co, j, l)
        if not mask[j] and b != cleared and not get_bit(bm, b):
            return with_bit(bm, b, 1)
    raise AssertionError("century %d: no non-member with a clear bit" % c_first)


# (name, H, W, pairs, decode_verify pair counts whose chunk layout the edits sit on)
CHUNK_CASES = [("one chunk", 120, 160, 4, (4,)), ("1080p", 1080, 1920, 4, (4,)), ("32 chunks", 3201, 4096, 1, (1,)),
               ("96 pairs", 3201, 4096, 96, (96, 2))]


@pytest.mark.parametrize("case", CHUNK_CASES, ids=[c[0] for c in CHUNK_CASES])
def test_witness_chunk_boundaries(pkg, co, case):
    """Edits on each side of every chunk boundary of K4b, at the chunk counts a decode of 1, 2, 4 or 96 pairs takes: a chunk base
    taken from the encode's pass counts (or from the wrong chunk) gives a count the model does not."""
    name, H, W, F, decode_pairs = case
    n = H * W
    ncent = (n + 99) // 100
    sm = pkg._cabi.device_info()["sm_count"]
    chunks = {P: witness_chunks(P, ncent, sm) for P in decode_pairs}
    assert chunks[decode_pairs[0]] == {"one chunk": 1, "1080p": 5, "32 chunks": 32}.get(name, chunks[decode_pairs[0]])
    if name == "96 pairs":
        assert chunks[96] < chunks[2] == 32
    l = n // 3 | 1
    rng = np.random.default_rng(n + F)
    base = [(rng.random(n) < 0.05).astype(np.uint8) for _ in range(min(F, 2))]
    bounds = sorted({c for P in decode_pairs for c in chunk_starts(ncent, chunks[P])})
    for m in base:
        for c in bounds or [ncent - 1]:
            m[100 * c - 1] = 1                             # a member in the last century of every chunk
    masks = [base[t % len(base)] for t in range(F)]
    st = pkg.FrameStream(H, W, 1, np.uint8, max_frames=len(base) + 1, max_pairs=F)
    try:
        st.upload(chain_frames(base, H, W))
        prev, curr = [t % len(base) for t in range(F)], [t % len(base) + 1 for t in range(F)]
        ks = [1.0 if t < 2 else 3.0 for t in range(F)]
        res = st.encode(prev, curr, THR, k_override=ks, l_override=[l] * F)
        assert not any(r.raw for r in res) and all(r.l == l for r in res)
        bms, wts, _ = st.fetch_batch(0, F)
        _, _, got_masks = fetch_all(st, len(base))
        assert all(np.array_equal(got_masks[i], base[i]) for i in range(len(base)))
        region = bitmap_region(pkg, st, F)
        check_region_contract(region, bms, res)
        edits = {}
        for i in range(min(F, 2)):                          # pair 0: every boundary; pair 1 (96 pairs): the first one only
            bm = bms[i, :(l + 7) // 8].copy()
            for c in (bounds if i == 0 else bounds[:1]) or [None]:
                bm = boundary_edit_k1(co, bm, l, masks[i], c - 1 if c else 0, c if c else ncent - 1)
            edits[i] = bm
        want_map = model_counts(co, edits, res, masks, wts)
        assert all(c > 0 for c in want_map.values()), want_map
        write_bitmaps(region, edits, [r.l for r in res])
        for P in decode_pairs:
            got = st.decode_verify(P)
            assert got.tolist() == [want_map.get(i, 0) for i in range(P)], (P, chunks[P], got[:4].tolist(), want_map)
        after = coded_bitmaps(bms, res)
        after.update(edits)
        check_intact(st, res, after, wts, F)
    finally:
        st.close()


# ------------------------------------------------------------------ D + E. encode paths, and the state decode_verify leaves
DH, DW, DP = 120, 161, 20
D_RAW = (9, 10)                                             # raw pairs in the middle (one on each side of the ranged split)
PATHS = {"pipelined ranges": dict(encode_ranges=2), "serial": dict(encode_ranges=1), "kq_ranges": dict(encode_ranges=1, kq_ranges=2),
         "encode_host": dict(host_chunk_frames=6)}


def d_masks():
    rng = np.random.default_rng(77)
    return [(rng.random(DH * DW) < (0.45 if t in D_RAW else (0.02, 0.05, 0.1)[t % 3])).astype(np.uint8) for t in range(DP)]


def d_encode(pkg, st, path, frames):
    with options(pkg, **PATHS[path]):
        if path == "encode_host":
            slot = (st.npix + 7) // 8 + 16
            ob = np.full((DP, slot), 0xAB, np.uint8)
            ow = np.full((DP, slot), 0xAB, np.uint8)
            res = st.encode_host(frames, THR, bitmap_slot=slot, witness_slot=slot, out_bitmaps=ob, out_witness=ow)
            for i, r in enumerate(res):
                nb, nw = (0, 0) if r.raw else ((r.l + 7) // 8, (r.wlen + 7) // 8)
                assert not ob[i, nb:].any() and not ow[i, nw:].any(), i
            return res
        st.upload(frames)
        return st.encode(list(range(DP)), list(range(1, DP + 1)), THR)


def check_against_oracle(co, st, res, masks, oracle):
    bms, wts, got = fetch_all(st, DP)
    for i, r in enumerate(res):
        ob, ow, _, _, _, ok, ol = oracle[i]
        assert np.array_equal(got[i], masks[i]), i
        assert r.raw == (ol == 0), i
        if r.raw:
            assert not bms[i].any() and not wts[i].any(), i
            continue
        assert (r.l, r.k, r.wlen) == (ol, ok, len(ow)), (i, r)
        nb, nw = (r.l + 7) // 8, (r.wlen + 7) // 8
        assert np.array_equal(bms[i, :nb], np.packbits(ob)) and not bms[i, nb:].any(), i
        assert np.array_equal(wts[i, :nw], np.packbits(ow)) and not wts[i, nw:].any(), i
    return bms, wts, got


@pytest.mark.parametrize("path", list(PATHS))
def test_encode_paths_and_state_afterwards(pkg, co, path):
    """decode_verify follows whichever path made the last encode; a shorter decode_verify returns the first counts; afterwards
    the bitmaps (edits included), witnesses and changed values are as before, a second decode_verify repeats its counts, and the
    next encode of the same frames is the oracle's again."""
    masks = d_masks()
    frames = chain_frames(masks, DH, DW)
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        oracle = list(ex.map(co.compress, masks))
    st = pkg.FrameStream(DH, DW, 1, np.uint8, max_frames=DP + 1, max_pairs=DP)
    try:
        res = d_encode(pkg, st, path, frames)
        assert [r.raw for r in res] == [t in D_RAW for t in range(DP)]
        bms, wts, got = check_against_oracle(co, st, res, masks, oracle)
        region = bitmap_region(pkg, st, DP)
        check_region_contract(region, bms, res)
        values = st.gather_changed()
        for i in range(DP):
            assert np.array_equal(values[i], frames[i + 1].reshape(-1)[masks[i] == 1]), i
        # E, without edits: all zero, nothing moved
        assert not st.decode_verify().any()
        check_intact(st, res, coded_bitmaps(bms, res), wts, DP)
        # D: edits on coded pairs of both ranges, at the first and last pair, beside the raw pairs
        rng = np.random.default_rng(5)
        edits = {0: clear_set_bit(bms[0, :(res[0].l + 7) // 8], res[0].l, rng), 8: all_bits(res[8].l, 0),
                 11: clear_set_bit(bms[11, :(res[11].l + 7) // 8], res[11].l, rng), DP - 1: all_bits(res[DP - 1].l, 1)}
        want_map = model_counts(co, edits, res, got, wts)
        assert all(c > 0 for c in want_map.values()), want_map
        want = [want_map.get(i, 0) for i in range(DP)]
        write_bitmaps(region, edits, [r.l for r in res])
        first = st.decode_verify()
        assert first.tolist() == want, (path, first.tolist(), want)
        for P in (1, 9, 12, DP - 1):
            assert st.decode_verify(P).tolist() == want[:P], P
        # E, with edits
        after = coded_bitmaps(bms, res)
        after.update(edits)
        check_intact(st, res, after, wts, DP)
        assert st.decode_verify().tolist() == want
        again = st.gather_changed()
        assert all(np.array_equal(a, b) for a, b in zip(again, values))
        res2 = d_encode(pkg, st, path, frames)
        check_against_oracle(co, st, res2, masks, oracle)
        assert not st.decode_verify().any()
    finally:
        st.close()
