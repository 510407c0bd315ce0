"""The multi-rank exchange of the packed bit arrays over peer memory, with N ranks on ONE GPU.

Several library contexts in one process play ranks 0..N-1.  A context's peer state is a table of device pointers
(rbf_peer_gather_init), and inside one process every device pointer is valid in every context, so handing every context the same
tables runs the real k_push_slots / k_peer_signal / k_peer_wait and the real host protocol of rbf_stream_allgather_bitmaps
between N receive buffers.  Only CUDA IPC is left out (rbf_peer_export / rbf_peer_open wrap cudaIpcGetMemHandle /
cudaIpcOpenMemHandle); NCCL cannot put two ranks on one GPU, so its path keeps test_nccl_allgather_single_rank and bench.py.

A. The C ABI, one host thread: every rank encodes its block of the stream and pushes, then every rank reads.
B. ShardedStreamEncoder end to end, one thread per rank, with a thread-local context, a threading fake of torch.distributed
   and the raw device pointer in place of the IPC handle; and, under B, contexts encoding from several threads at once.

Every received row is compared with a single-stream encode of the whole stream on the process-wide context, whose bit arrays
are checked against the C oracle.  No test lets a wait run into its time-out: every wait is satisfiable within milliseconds.
"""
import contextlib
import ctypes as C
import os
import threading
import time

import numpy as np
import pytest

from tests.util import synth_stream

pytestmark = pytest.mark.gpu

THR = 3.0
RBF_ERR_INVALID, RBF_ERR_STATE = -1, -6
H, W = 54, 97                                       # 5238 pixels: not a multiple of 32
# densities of the successive pairs: coded pairs of different l, an empty and a dense mask (both raw, their rows are zero)
P_SEQ = [0.05, 0.0, 0.15, 0.01, 0.4, 0.3, 0.02]
PAIRS = {2: 7, 3: 11, 5: 13, 8: 21, 16: 39}         # total pairs per world size, none divisible by it


@pytest.fixture(scope="module")
def pkg():
    import new_bloom_filter_repo_b200 as p
    info = p._cabi.device_info()
    assert info["cc"] == (9, 0), info
    return p


@pytest.fixture(scope="module")
def co():
    from oracle import c_oracle
    c_oracle.build()
    return c_oracle


def _device():
    return int(os.environ.get("RBF_DEVICE", os.environ.get("LOCAL_RANK", "0")))


@pytest.fixture(scope="module")
def ctxs(pkg, request):
    """request.param contexts on the device, one per rank."""
    L = pkg._cabi.lib()
    hs = []
    try:
        for _ in range(request.param):
            h = C.c_void_p()
            pkg._cabi.check(L.rbf_ctx_create(_device(), C.byref(h)))
            hs.append(h)
        yield hs
    finally:
        for h in hs:
            L.rbf_peer_gather_shutdown(h)
            L.rbf_ctx_destroy(h)


@contextlib.contextmanager
def on_ctx(pkg, h):
    """_cabi.ctx() returns h inside (a FrameStream takes its context from it in rbf_stream_create only)."""
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(pkg._cabi, "ctx", lambda: h)
        yield


def launches(pkg, h):
    return pkg._cabi.lib().rbf_get_counter(h, b"kernel_launches")


def make_stream(h, w, total_pairs, seed, p_seq, shift=0):
    return synth_stream(h, w, total_pairs + 1, seed, p_seq[shift:] + p_seq[:shift])


class Reference:
    """The single-stream encode of a whole stream on the process-wide context: every pair's PairResult and packbits bit array
    (empty for a raw pair).  The bit arrays of `oracle_pairs` are checked against the C oracle's compress of the fetched mask,
    and the fetched mask against the oracle's frame difference."""

    def __init__(self, pkg, co, frames, oracle_pairs=None):
        n = len(frames)
        st = pkg.FrameStream(frames.shape[1], frames.shape[2], 3, frames.dtype, max_frames=n)
        try:
            st.upload(frames)
            self.results = st.encode_consecutive(n, THR)
            self.bitmaps = [st.fetch(t, want_mask=False)[0] for t in range(n - 1)]
            for j in (range(n - 1) if oracle_pairs is None else sorted(set(oracle_pairs))):
                mask = st.fetch(j)[2]
                omask = co.frame_diff_mask(frames[j], frames[j + 1], THR)[0].reshape(-1)
                assert np.array_equal(mask, omask), j
                ob, ow, op, on, ratio, ok, ol = co.compress(mask)
                r = self.results[j]
                if ok == 0:
                    assert r.raw and r.l == 0 and self.bitmaps[j].size == 0, (j, r)
                else:
                    assert not r.raw and (r.l, r.k, r.wlen) == (ol, ok, len(ow)), (j, r, ol, ok, len(ow))
                    assert np.array_equal(self.bitmaps[j], np.packbits(ob)), j
        finally:
            st.close()
        self.headers = [(r.l, r.wlen, r.p, r.k, r.ones, r.raw) for r in self.results]
        self.max_l = max(r.l for r in self.results)

    def assert_mixed(self):
        """Coded pairs of at least three sizes, an empty mask and a dense one."""
        res = self.results
        assert len({r.l for r in res if not r.raw}) >= 3
        assert any(r.raw and r.ones == 0 for r in res) and any(r.raw and r.ones > 0 for r in res)


def fit_slot(max_l):
    """The smallest multiple of 16 bytes that holds a bit array of max_l bits."""
    return ((max_l + 7) // 8 + 15) // 16 * 16


class Ranks:
    """Ranks 0..N-1 of one stream: rank r's FrameStream (its block of pairs and the halo frame, `blocks` times over), receive
    buffer (2 x N x slots x slot_bytes) and 256-byte flag array belong to context r; every context holds the same pointer tables."""

    def __init__(self, pkg, ctxs, h, w, total_pairs, blocks=1):
        from new_bloom_filter_repo_b200 import distributed as rdist
        self.pkg, self.L, self.ctxs = pkg, pkg._cabi.lib(), ctxs
        self.N, self.P = len(ctxs), int(total_pairs)
        self.lay = [rdist.shard_layout(self.P, r, self.N) for r in range(self.N)]
        self.slots = self.lay[0]["slots"]
        self.rows = rdist.gathered_pair_rows(self.P, self.N)
        self.streams, self.recv, self.flags = [], [], []
        self.slot = None
        try:
            for r, c in enumerate(ctxs):
                with on_ctx(pkg, c):
                    self.streams.append(pkg.FrameStream(h, w, 3, np.uint8, max_frames=blocks * self.lay[r]["frames"],
                                                        max_pairs=self.slots))
        except BaseException:
            self.close()
            raise
        stride = C.c_uint64()
        self.check(self.L.rbf_stream_bitmap_region(self.streams[0]._h, None, C.byref(stride)), 0)
        self.stride = stride.value

    def check(self, rc, r):
        self.pkg._cabi.check(rc, self.ctxs[r])

    def connect(self, slot_bytes):
        """Fresh zeroed receive buffers and flag arrays, registered on every context (exchange numbers start again from 1)."""
        self.disconnect()
        L, N = self.L, self.N
        self.slot = int(slot_bytes)
        nbytes = 2 * N * self.slots * self.slot
        for r, c in enumerate(self.ctxs):
            for lst, nb in ((self.recv, nbytes), (self.flags, 256)):
                p = C.c_void_p()
                self.check(L.rbf_malloc(c, nb, C.byref(p)), r)
                lst.append(p)
                self.check(L.rbf_memset(c, p, 0, nb), r)
            self.check(L.rbf_sync(c), r)
        self.recv_tab = (C.c_void_p * N)(*[p.value for p in self.recv])
        self.flag_tab = (C.c_void_p * N)(*[p.value for p in self.flags])
        for r, c in enumerate(self.ctxs):
            self.check(L.rbf_peer_gather_init(c, r, N, self.recv_tab, self.flag_tab), r)

    def disconnect(self):
        for c in self.ctxs:
            self.L.rbf_peer_gather_shutdown(c)
        for lst in (self.recv, self.flags):
            for r, p in enumerate(lst):
                self.L.rbf_free(self.ctxs[r], p)
            lst.clear()

    def close(self):
        self.disconnect()
        for st in self.streams:
            st.close()
        self.streams = []

    def block(self, r, frames):
        lay = self.lay[r]
        return frames[lay["first_frame"]: lay["first_frame"] + lay["frames"]]

    def upload(self, r, frames, block=0):
        self.streams[r].upload(self.block(r, frames), first=block * self.lay[r]["frames"])

    def encode(self, r, ref, block=0):
        """Encode rank r's block; its PairResults must be the single-stream encode's of the same pairs."""
        lay = self.lay[r]
        idx = np.arange(block * lay["frames"], (block + 1) * lay["frames"], dtype=np.uint32)
        res = self.streams[r].encode(idx[:-1], idx[1:], THR)
        got = [(x.l, x.wlen, x.p, x.k, x.ones, x.raw) for x in res]
        assert got == ref.headers[lay["lo"]: lay["hi"]], r
        return res

    def exchange(self, r, pairs=None, slot_bytes=None, recv=None):
        return self.L.rbf_stream_allgather_bitmaps(self.streams[r]._h, self.slots if pairs is None else pairs,
                                                   self.slot if slot_bytes is None else slot_bytes, None,
                                                   self.recv[r] if recv is None else recv)

    def half(self, r):
        h = C.c_uint32()
        self.check(self.L.rbf_peer_gather_half(self.ctxs[r], C.byref(h)), r)
        return h.value

    def buffer(self, r):
        """Rank r's whole receive buffer as uint8[2, N, slots, slot_bytes] (rbf_memcpy_d2h: joins a pending exchange)."""
        buf = np.empty(2 * self.N * self.slots * self.slot, dtype=np.uint8)
        self.check(self.L.rbf_memcpy_d2h(self.ctxs[r], self.pkg._cabi.ptr(buf), self.recv[r], buf.size), r)
        return buf.reshape(2, self.N, self.slots, self.slot)

    def read(self, r):
        self.check(self.L.rbf_sync(self.ctxs[r]), r)
        return self.half(r), self.buffer(r)

    def assert_rows(self, half_buf, ref, what, owners=None):
        """Every (rank, slot) row that gathered_pair_rows names, of the ranks in `owners`, holds the owner's bit array of that
        pair, zero to the end of the slot."""
        assert len(self.rows) == self.P
        for j, (r, t) in enumerate(self.rows):
            if owners is not None and r not in owners:
                continue
            want, row = ref.bitmaps[j], half_buf[r, t]
            assert want.size <= row.size
            assert np.array_equal(row[: want.size], want), "%s: pair %d in row (%d, %d)" % (what, j, r, t)
            assert not row[want.size:].any(), "%s: pair %d, row (%d, %d): bytes after the bit array are not zero" % (what, j, r, t)

    def assert_layout(self):
        """The gathered order names each rank's pairs in stream order and never a rank's unused last slot."""
        owned = [(r, t) for r in range(self.N) for t in range(self.lay[r]["pairs"])]
        assert self.rows == owned
        short = [r for r in range(self.N) if self.lay[r]["pairs"] < self.slots]
        assert short and all((r, self.slots - 1) not in self.rows for r in short)


def run_rounds(rk, streams, refs, overlap):
    """Exchange number q = s + 1 carries streams[s].  overlap: right after a rank's exchange call, the rank uploads and encodes the
    next stream before anything synchronises it; the push must still carry the old bit arrays.  After each exchange every rank
    reads: half q & 1 holds exchange q, the other half still holds exchange q - 1 (zeros before the first)."""
    def encode(r, s):
        rk.upload(r, streams[s])
        rk.encode(r, refs[s])

    if overlap:
        for r in range(rk.N):
            encode(r, 0)
    for s in range(len(streams)):
        for r in range(rk.N):
            if not overlap:
                encode(r, s)
            rk.check(rk.exchange(r), r)
            if overlap and s + 1 < len(streams):
                encode(r, s + 1)
        q = s + 1
        for r in range(rk.N):
            half, buf = rk.read(r)
            assert half == q & 1, (r, q, half)
            rk.assert_rows(buf[q & 1], refs[s], "rank %d, exchange %d" % (r, q))
            if s == 0:
                assert not buf[1 - (q & 1)].any(), "rank %d: the other half was written by the first exchange" % r
            else:
                rk.assert_rows(buf[1 - (q & 1)], refs[s - 1], "rank %d, exchange %d after exchange %d" % (r, q - 1, q))


# ------------------------------------------------------------------ A. the C ABI, one host thread
@pytest.mark.parametrize("overlap", [False, True], ids=["serial", "overlap"])
@pytest.mark.parametrize("slot_kind", ["fit", "fit+16", "stride"])
@pytest.mark.parametrize("ctxs", sorted(PAIRS), indirect=True, ids=lambda n: "N%d" % n)
def test_every_rank_receives_every_pair(pkg, co, ctxs, slot_kind, overlap):
    """Three exchanges of different streams.  Slots: the smallest multiple of 16 that holds the largest bit array of the three,
    that plus 16, and the stream's whole mask stride (the largest slot accepted)."""
    N = len(ctxs)
    P = PAIRS[N]
    streams = [make_stream(H, W, P, 1000 * N + s, P_SEQ, shift=s) for s in range(3)]
    refs = [Reference(pkg, co, f) for f in streams]
    for ref in refs:
        ref.assert_mixed()
    rk = Ranks(pkg, ctxs, H, W, P)
    try:
        rk.assert_layout()
        fit = fit_slot(max(ref.max_l for ref in refs))
        rk.connect({"fit": fit, "fit+16": fit + 16, "stride": rk.stride}[slot_kind])
        assert rk.slot <= rk.stride
        run_rounds(rk, streams, refs, overlap)
    finally:
        rk.close()


@pytest.mark.parametrize("ctxs", [2], indirect=True, ids=lambda n: "N%d" % n)
def test_push_spans_more_than_one_grid_pass(pkg, co, ctxs):
    """4K blocks in slots of the whole mask stride: each rank pushes more 16-byte granules to each destination than one pass of
    k_push_slots' grid (sm_count x 8 CTAs of 256 threads) covers, so its grid-stride loop runs more than once."""
    h, w, P = 2160, 3840, 9
    p_seq = [0.05, 0.0, 0.2, 0.01, 0.4, 0.1]
    sm = pkg._cabi.device_info()["sm_count"]
    rk = Ranks(pkg, ctxs, h, w, P)
    try:
        ends = [x for lay in rk.lay for x in (lay["lo"], lay["hi"] - 1)]
        streams = [make_stream(h, w, P, 4000 + s, p_seq, shift=s) for s in range(2)]
        refs = [Reference(pkg, co, f, oracle_pairs=ends) for f in streams]
        refs[0].assert_mixed()
        rk.connect(rk.stride)
        assert rk.slots * rk.slot > sm * 8 * 256 * 16, (rk.slots, rk.slot, sm)
        run_rounds(rk, streams, refs, overlap=True)
    finally:
        rk.close()


@pytest.mark.parametrize("ctxs", [2], indirect=True, ids=lambda n: "N%d" % n)
def test_rank_running_ahead_waits_for_the_unread_half(pkg, co, ctxs):
    """Rank 0 issues exchanges 3 and 4 before rank 1 has read exchange 2.  Exchange 4 reuses the half that holds exchange 2; the
    wait in front of its push holds it until rank 1 signals exchange 3, so rank 1 still reads exchange 2 there."""
    P = PAIRS[2]
    streams = [make_stream(H, W, P, 3000 + s, P_SEQ, shift=s) for s in range(4)]
    refs = [Reference(pkg, co, f) for f in streams]
    rk = Ranks(pkg, ctxs, H, W, P, blocks=4)
    try:
        for s in range(4):                                  # every frame is resident before the exchanges start
            for r in range(2):
                rk.upload(r, streams[s], block=s)
        rk.connect(fit_slot(max(ref.max_l for ref in refs)))

        def issue(r, s):
            rk.encode(r, refs[s], block=s)
            rk.check(rk.exchange(r), r)

        for r in range(2):
            issue(r, 0)
        for r in range(2):
            half, buf = rk.read(r)
            assert half == 1
            rk.assert_rows(buf[1], refs[0], "rank %d, exchange 1" % r)
        for r in range(2):
            issue(r, 1)
        half, buf = rk.read(0)
        assert half == 0
        rk.assert_rows(buf[0], refs[1], "rank 0, exchange 2")
        # Rank 0 runs ahead.  From here on nothing touches context 0 until rank 1 has issued exchange 3: a call that synchronises
        # context 0 would wait for rank 1, which this same thread drives.
        issue(0, 2)
        issue(0, 3)
        time.sleep(0.05)                                    # a push that did not wait would have landed by now
        half, buf = rk.read(1)
        assert half == 0
        rk.assert_rows(buf[0], refs[1], "rank 1 reading exchange 2 while rank 0 has issued exchange 4")
        rk.assert_rows(buf[1], refs[2], "rank 1: rank 0's rows of exchange 3", owners={0})
        rk.assert_rows(buf[1], refs[0], "rank 1: its own rows of exchange 1", owners={1})
        issue(1, 2)
        issue(1, 3)
        for r in range(2):
            half, buf = rk.read(r)
            assert half == 0
            rk.assert_rows(buf[0], refs[3], "rank %d, exchange 4" % r)
            rk.assert_rows(buf[1], refs[2], "rank %d, exchange 3" % r)
    finally:
        rk.close()


@pytest.mark.parametrize("ctxs", [3], indirect=True, ids=lambda n: "N%d" % n)
def test_launch_counts(pkg, co, ctxs):
    """The first exchange of a context launches the push and the signal, every later one also the wait in front of the push; the
    first call that joins an exchange (rbf_sync, rbf_memcpy_d2h, rbf_timer_stop_ms) launches the wait for the other ranks, and
    only that one."""
    L, N, P = pkg._cabi.lib(), 3, PAIRS[3]
    streams = [make_stream(H, W, P, 5000 + s, P_SEQ, shift=s) for s in range(3)]
    refs = [Reference(pkg, co, f) for f in streams]
    rk = Ranks(pkg, ctxs, H, W, P)

    def exchange_all(s, added):
        for r in range(N):
            rk.upload(r, streams[s])
            rk.encode(r, refs[s])
            n0 = launches(pkg, ctxs[r])
            rk.check(rk.exchange(r), r)
            assert launches(pkg, ctxs[r]) - n0 == added, (r, s)

    def joined_by(r, call):
        n0 = launches(pkg, ctxs[r])
        out = call()
        assert launches(pkg, ctxs[r]) - n0 == 1, r
        n0 = launches(pkg, ctxs[r])
        rk.check(L.rbf_sync(ctxs[r]), r)                   # already joined
        half = rk.half(r)
        assert launches(pkg, ctxs[r]) == n0, r
        return half, out

    try:
        rk.connect(fit_slot(max(ref.max_l for ref in refs)))
        exchange_all(0, 2)
        for r in range(N):
            half, _ = joined_by(r, lambda: rk.check(L.rbf_sync(ctxs[r]), r))
            n0 = launches(pkg, ctxs[r])
            buf = rk.buffer(r)
            assert launches(pkg, ctxs[r]) == n0 and half == 1
            rk.assert_rows(buf[1], refs[0], "rank %d, exchange 1" % r)
        exchange_all(1, 3)
        for r in range(N):
            half, buf = joined_by(r, lambda: rk.buffer(r))
            assert half == 0
            rk.assert_rows(buf[0], refs[1], "rank %d, exchange 2" % r)
        exchange_all(2, 3)
        ms = C.c_double()
        for r in range(N):
            rk.check(L.rbf_timer_start(ctxs[r]), r)
            half, _ = joined_by(r, lambda: rk.check(L.rbf_timer_stop_ms(ctxs[r], C.byref(ms)), r))
            assert half == 1
            rk.assert_rows(rk.buffer(r)[1], refs[2], "rank %d, exchange 3" % r)
        rk.connect(rk.slot)                                 # registered again: the next exchange is a first one
        exchange_all(0, 2)
        for r in range(N):
            half, buf = joined_by(r, lambda: rk.buffer(r))
            assert half == 1
            rk.assert_rows(buf[1], refs[0], "rank %d, first exchange after a new registration" % r)
    finally:
        rk.close()


@pytest.mark.parametrize("ctxs", [3], indirect=True, ids=lambda n: "N%d" % n)
def test_invalid_arguments_launch_nothing(pkg, co, ctxs):
    """Bad registrations, exchanges and half queries return an error, launch nothing and leave the registered state as it was."""
    L, N, P = pkg._cabi.lib(), 3, PAIRS[3]
    frames = make_stream(H, W, P, 6000, P_SEQ)
    ref = Reference(pkg, co, frames)
    rk = Ranks(pkg, ctxs, H, W, P)
    try:
        rk.connect(fit_slot(ref.max_l))
        for r in range(N):
            rk.upload(r, frames)
            rk.encode(r, ref)
        counts = [launches(pkg, c) for c in ctxs]
        half = C.c_uint32()
        for c in ctxs:
            assert L.rbf_peer_gather_half(c, C.byref(half)) == RBF_ERR_STATE          # registered, nothing exchanged yet

        def table_with_null(tab, i):
            t = (C.c_void_p * N)(*[p for p in tab])
            t[i] = None
            return t

        c0 = ctxs[0]
        bad_inits = [(0, 0, rk.recv_tab, rk.flag_tab), (17, 0, rk.recv_tab, rk.flag_tab), (N, -1, rk.recv_tab, rk.flag_tab),
                     (N, N, rk.recv_tab, rk.flag_tab), (N, 0, None, rk.flag_tab), (N, 0, rk.recv_tab, None)]
        bad_inits += [(N, 0, table_with_null(rk.recv_tab, i), rk.flag_tab) for i in range(N)]
        bad_inits += [(N, 0, rk.recv_tab, table_with_null(rk.flag_tab, i)) for i in range(N)]
        for nranks, rank, rt, ft in bad_inits:
            assert L.rbf_peer_gather_init(c0, rank, nranks, rt, ft) == RBF_ERR_INVALID, (nranks, rank)
        bad_exchanges = [lambda r: dict(recv=rk.recv[(r + 1) % N]),                   # another rank's buffer
                         lambda r: dict(recv=C.c_void_p(rk.recv[r].value + 16)),
                         lambda r: dict(slot_bytes=0), lambda r: dict(slot_bytes=8), lambda r: dict(slot_bytes=rk.slot + 8),
                         lambda r: dict(slot_bytes=rk.stride + 16), lambda r: dict(pairs=0), lambda r: dict(pairs=rk.slots + 1)]
        for bad in bad_exchanges:
            for r in range(N):
                assert rk.exchange(r, **bad(r)) == RBF_ERR_INVALID, (r, bad(r))
        assert L.rbf_stream_allgather_bitmaps(rk.streams[0]._h, rk.slots, rk.slot, None, None) == RBF_ERR_INVALID
        for c in ctxs:
            assert L.rbf_peer_gather_half(c, C.byref(half)) == RBF_ERR_STATE          # no exchange number was taken
        assert [launches(pkg, c) for c in ctxs] == counts
        # the registration survived: one exchange still delivers every pair to every rank
        for r in range(N):
            rk.check(rk.exchange(r), r)
        for r in range(N):
            h, buf = rk.read(r)
            assert h == 1
            rk.assert_rows(buf[1], ref, "rank %d after the refused calls" % r)
        rk.disconnect()
        for c in ctxs:
            assert L.rbf_peer_gather_half(c, C.byref(half)) == RBF_ERR_STATE          # not registered any more
    finally:
        rk.close()


# ------------------------------------------------------------------ B. ShardedStreamEncoder, one thread per rank
class ThreadGroup:
    """What distributed.py asks of torch.distributed, for `world` threads of one process.  Every collective meets at a
    threading.Barrier with a time-out, and a rank that fails aborts it, so a broken rank fails the test instead of hanging it."""

    class ReduceOp:
        MAX = "max"

    def __init__(self, world, timeout=120.0):
        self.world = world
        self._bar = threading.Barrier(world, timeout=timeout)
        self._slots = [None] * world

    def abort(self):
        self._bar.abort()

    def rank(self, r):
        return _RankView(self, r)

    def _gather(self, r, obj):
        self._slots[r] = obj
        self._bar.wait()
        out = list(self._slots)
        self._bar.wait()                                    # nobody overwrites a slot before every rank has copied them
        return out


class _RankView:
    def __init__(self, group, rank):
        self.group, self.r = group, rank
        self.ReduceOp = group.ReduceOp

    def get_rank(self):
        return self.r

    def get_world_size(self):
        return self.group.world

    def get_backend(self):
        return "gloo"

    def barrier(self):
        self.group._bar.wait()

    def all_gather_object(self, out, obj):
        out[:] = self.group._gather(self.r, obj)

    def all_reduce(self, t, op):
        assert op == self.ReduceOp.MAX
        t.fill_(max(self.group._gather(self.r, int(t.item()))))


class RawPointerIpc:
    """_cabi.lib() with the raw device pointer in place of a CUDA IPC handle: rbf_peer_export writes it into the 64-byte handle,
    rbf_peer_open reads it back, and rbf_peer_close of such a pointer does nothing.  Every other symbol is the library's."""
    TAG = b"raw device ptr\0\0"

    def __init__(self, real):
        self._real = real
        self._lock = threading.Lock()
        self.opened, self.closed = [], []

    def __getattr__(self, name):
        return getattr(self._real, name)

    def rbf_peer_export(self, ctx, d_ptr, handle_out):
        addr = d_ptr.value if isinstance(d_ptr, C.c_void_p) else int(d_ptr)
        C.memmove(handle_out.value, self.TAG + addr.to_bytes(8, "little") + bytes(40), 64)
        return 0

    def rbf_peer_open(self, ctx, handle, out):
        raw = C.string_at(handle.value, 64)
        assert raw[:16] == self.TAG
        addr = int.from_bytes(raw[16:24], "little")
        out._obj.value = addr                               # out is C.byref(c_void_p)
        with self._lock:
            self.opened.append(addr)
        return 0

    def rbf_peer_close(self, ctx, d_ptr):
        addr = d_ptr.value if isinstance(d_ptr, C.c_void_p) else d_ptr
        with self._lock:
            if addr in self.opened:
                self.closed.append(addr)
                return 0
        return self._real.rbf_peer_close(ctx, d_ptr)


@pytest.fixture(scope="module")
def exchange_kernels_loaded(pkg):
    """One single-rank exchange on the process-wide context, so that the exchange kernels are loaded before ranks in threads
    depend on each other's progress (loading a module can wait for the device)."""
    from new_bloom_filter_repo_b200 import distributed as rdist
    st = pkg.FrameStream(H, W, 3, np.uint8, max_frames=3)
    try:
        st.upload(make_stream(H, W, 2, 7, P_SEQ))
        st.encode_consecutive(3, THR)
        pg = rdist.PeerGather(None, 2, 256)
        try:
            pg.exchange(st)
            pg.result()
        finally:
            pg.close()
    finally:
        st.close()


def run_ranks(pkg, world, body, timeout=300.0):
    """body(rank, dist) in one thread per rank, each with a context of its own as _cabi.ctx() and RawPointerIpc as _cabi.lib().
    -> (per-rank return values, per-rank exceptions, the IPC stand-in)."""
    L = pkg._cabi.lib()
    hs = []
    for _ in range(world):
        h = C.c_void_p()
        pkg._cabi.check(L.rbf_ctx_create(_device(), C.byref(h)))
        hs.append(h)
    tls = threading.local()
    ipc = RawPointerIpc(L)
    group = ThreadGroup(world)
    out, errors = [None] * world, [None] * world

    def main(r):
        tls.ctx = hs[r]
        try:
            out[r] = body(r, group.rank(r))
        except BaseException as e:                          # noqa: B036 -- reported by the caller
            errors[r] = e
            group.abort()

    alive = []
    try:
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr(pkg._cabi, "lib", lambda: ipc)
            mp.setattr(pkg._cabi, "ctx", lambda: tls.ctx)
            threads = [threading.Thread(target=main, args=(r,), daemon=True) for r in range(world)]
            for t in threads:
                t.start()
            deadline = time.monotonic() + timeout
            for t in threads:
                t.join(max(0.0, deadline - time.monotonic()))
            alive = [r for r, t in enumerate(threads) if t.is_alive()]
    finally:
        if not alive:                                       # a context still in use by a thread is left alone
            for h in hs:
                L.rbf_ctx_destroy(h)
    assert not alive, "ranks %s did not finish" % alive
    return out, errors, ipc


def raise_first(errors):
    """Raise the first rank's error that is not a broken barrier (a consequence of another rank's), naming every rank's."""
    failed = [(r, e) for r, e in enumerate(errors) if e is not None]
    if failed:
        first = next((e for _, e in failed if not isinstance(e, threading.BrokenBarrierError)), failed[0][1])
        raise AssertionError("; ".join("rank %d: %s: %s" % (r, type(e).__name__, e) for r, e in failed)) from first


# rounds 1 and 2 have no density as high as round 0's 0.15, so their bit arrays fit the slot agreed at the first encode
P_SEQ_LOW = [0.02, 0.4, 0.05, 0.0, 0.01, 0.3, 0.03]


@pytest.mark.parametrize("world,total_frames,headroom", [(2, 8, False), (3, 11, False), (4, 14, True), (4, 5, True)])
def test_sharded_encoder_threads(pkg, co, exchange_kernels_loaded, world, total_frames, headroom):
    """ShardedStreamEncoder with the peer exchange, a thread per rank: after each of three encodes of different streams, and after
    renegotiate() to a larger slot and one more encode, every rank's gathered() and headers() are the single-stream encode's.
    headroom: the slot is agreed in the constructor (max_l_bits), else at the first encode."""
    import torch  # noqa: F401 -- agree_slot_bytes imports it; a first import inside a collective could outlast the barrier
    from new_bloom_filter_repo_b200 import distributed as rdist
    P = total_frames - 1
    seqs = [P_SEQ, P_SEQ_LOW, P_SEQ_LOW, P_SEQ]
    streams = [make_stream(H, W, P, 7000 + 10 * world + s, seqs[s], shift=s) for s in range(4)]
    refs = [Reference(pkg, co, f) for f in streams]
    max_l = max(ref.max_l for ref in refs[:3])
    if not headroom:
        assert max_l <= 8 * fit_slot(refs[0].max_l)                 # encodes 2 and 3 fit the slot agreed at the first
    grow = 8 * fit_slot(max_l) + 512
    assert refs[3].max_l <= grow                                    # so does the encode after renegotiate(grow)

    def body(r, dist):
        enc = rdist.ShardedStreamEncoder(dist, H, W, 3, np.uint8, total_frames, max_l_bits=max_l if headroom else None)
        rec = []
        try:
            for s in range(4):
                if s == 3:
                    enc.renegotiate(grow)
                lay = enc.layout
                enc.upload(streams[s][lay["first_frame"]: lay["first_frame"] + lay["frames"]])
                res = enc.encode(THR)
                got = enc.gathered()
                flags = enc._peer.flags.to_host()[: 4 * world].view(np.uint32).copy()   # before headers(): no rank is ahead
                half = C.c_uint32()
                pkg._cabi.check(pkg._cabi.lib().rbf_peer_gather_half(pkg._cabi.ctx(), C.byref(half)), pkg._cabi.ctx())
                rec.append(dict(gather=enc.gather, slot=enc.slot, got=got, headers=enc.headers(), flags=flags, half=half.value,
                                mine=[(x.l, x.wlen, x.p, x.k, x.ones, x.raw) for x in res[: enc.layout["pairs"]]],
                                lo=enc.layout["lo"], hi=enc.layout["hi"]))
        finally:
            enc.close()
        return rec

    out, errors, ipc = run_ranks(pkg, world, body)
    raise_first(errors)
    assert len(ipc.opened) == 2 * world * 2 * (world - 1)           # two registrations: 2 buffers of each other rank
    assert sorted(ipc.closed) == sorted(ipc.opened)
    for r in range(world):
        slot0 = out[r][0]["slot"]
        assert slot0 == (fit_slot(max_l) if headroom else fit_slot(refs[0].max_l))
        for s, rec in enumerate(out[r]):
            what = "rank %d, encode %d" % (r, s + 1)
            assert rec["gather"] == "p2p", what
            assert rec["slot"] == (slot0 if s < 3 else fit_slot(grow)), what
            q = s + 1 if s < 3 else 1                               # renegotiate() registers new buffers: numbering restarts
            assert rec["half"] == q & 1 and rec["flags"].tolist() == [q] * world, (what, rec["half"], rec["flags"])
            assert rec["mine"] == refs[s].headers[rec["lo"]: rec["hi"]], what
            assert rec["headers"] == refs[s].headers, what
            got = rec["got"]
            assert got.shape == (P, rec["slot"]), what
            for j in range(P):
                want = refs[s].bitmaps[j]
                assert np.array_equal(got[j, : want.size], want) and not got[j, want.size:].any(), (what, j)


def test_sharded_encoder_rejects_ranks_without_pairs(pkg):
    """Fewer frame pairs than ranks: every rank raises ValueError in the constructor, before any collective or allocation."""
    from new_bloom_filter_repo_b200 import distributed as rdist

    def body(r, dist):
        with pytest.raises(ValueError, match="every rank needs at least one pair"):
            rdist.ShardedStreamEncoder(dist, H, W, 3, np.uint8, 3)
        return r

    out, errors, _ = run_ranks(pkg, 4, body, timeout=120.0)
    raise_first(errors)
    assert out == [0, 1, 2, 3]


def test_contexts_in_threads_encode_concurrently(pkg, co):
    """What the threaded tests above stand on: contexts driven from several host threads encode at the same time and each gets
    the single-thread result.  The two streams' bit arrays differ about fourfold in size, and so does the shared memory of their
    query launches, whose per-kernel limit is one value for the whole process: ranks that start an encode together could lower
    it between another rank's set and launch, as the lockstep ranks of test_sharded_encoder_threads did."""
    h, w = 270, 480
    streams = [synth_stream(h, w, 3, 9100, [0.01]), synth_stream(h, w, 3, 9101, [0.15])]
    refs = [Reference(pkg, co, f) for f in streams]
    assert not any(r.raw for ref in refs for r in ref.results) and refs[1].max_l > 3 * refs[0].max_l

    def body(r, dist):
        st = pkg.FrameStream(h, w, 3, np.uint8, max_frames=6)
        try:
            st.upload(streams[0], first=0)
            st.upload(streams[1], first=3)
            for i in range(24):
                k = (i + r) % 2
                dist.barrier()                                  # the ranks' launches start together, half of them with each size
                res = st.encode([3 * k, 3 * k + 1], [3 * k + 1, 3 * k + 2], THR)
                assert [(x.l, x.wlen, x.p, x.k, x.ones, x.raw) for x in res] == refs[k].headers, (r, i)
                for t in range(2):
                    assert np.array_equal(st.fetch(t, want_mask=False)[0], refs[k].bitmaps[t]), (r, i, t)
        finally:
            st.close()
        return r

    out, errors, _ = run_ranks(pkg, 4, body)
    raise_first(errors)
    assert out == [0, 1, 2, 3]
