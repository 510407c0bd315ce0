"""
Multi-GPU plumbing: one process per GPU.  Inter-frame pairs are independent units
(BloomFilterCompressor.compress keeps no state between frames, ivc:198-266), so ranks take
contiguous blocks of pairs (each block needs one halo frame: its first `prev`) and the only
exchange is ONE all-gather of the packed Bloom bit arrays: either ncclAllGather, or (PeerGather) a
kernel of the library that stores the slots straight into every rank's receive buffer over NVLink
peer memory.  torch.distributed is used for the rendezvous only (NCCL unique id / CUDA IPC handles,
barriers, max-over-ranks timing).
"""
from __future__ import annotations

import ctypes as C
from typing import Tuple

import numpy as np

from . import _cabi


def shard_pairs(pairs: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous block [lo, hi) of pair indices owned by `rank` (sizes differ by at most one)."""
    base, rem = divmod(int(pairs), int(world))
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_layout(total_pairs: int, rank: int, world: int) -> dict:
    """Block partition of ONE stream's pairs over the ranks (strong scaling, SURVEY 8e): rank r codes pairs [lo, hi), for which
    it needs frames lo .. hi (one halo frame: its first `prev`); every rank contributes the same number of all-gather slots
    (`slots` = ceil(total_pairs / world); a rank with fewer pairs leaves its last slot unused)."""
    lo, hi = shard_pairs(total_pairs, rank, world)
    return {"lo": lo, "hi": hi, "pairs": hi - lo, "first_frame": lo, "frames": hi - lo + 1, "slots": -(-int(total_pairs) // int(world))}


def gathered_pair_rows(total_pairs: int, world: int):
    """(rank, slot) of every pair 0 .. total_pairs-1 inside the gathered buffer [world][slots][slot_bytes]."""
    rows = []
    for r in range(world):
        lo, hi = shard_pairs(total_pairs, r, world)
        rows += [(r, t) for t in range(hi - lo)]
    return rows


def broadcast_unique_id(dist, make_id) -> np.ndarray:
    """Rank 0 calls make_id() -> uint8[128]; every rank returns the same 128 bytes (torch.distributed broadcast)."""
    import torch
    ident = np.zeros(128, dtype=np.uint8)
    if dist.get_rank() == 0:
        ident[:] = make_id()
    t = torch.from_numpy(ident.copy())
    if dist.get_backend() == "nccl":
        t = t.cuda()
    dist.broadcast(t, src=0)
    return t.cpu().numpy().copy()


def agree_slot_bytes(dist, local_max_bits: int, align: int = 16) -> int:
    """Fixed all-gather slot: max over ranks of ceil(l/8), rounded up (every rank must use the same size)."""
    import torch
    t = torch.tensor([(int(local_max_bits) + 7) // 8], dtype=torch.int64)
    if dist.get_backend() == "nccl":
        t = t.cuda()
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return (int(t.item()) + align - 1) // align * align


def _nccl_unique_id() -> np.ndarray:
    ident = np.zeros(128, dtype=np.uint8)
    _cabi.check(_cabi.lib().rbf_nccl_unique_id(_cabi.ptr(ident)))
    return ident


def init_nccl_from_torch(dist) -> None:
    """Create the library's NCCL communicator; the 128-byte unique id travels over torch.distributed."""
    ident = broadcast_unique_id(dist, _nccl_unique_id)
    _cabi.check(_cabi.lib().rbf_nccl_init(_cabi.ctx(), _cabi.ptr(ident), dist.get_rank(), dist.get_world_size()), _cabi.ctx())


class DeviceBuffer:
    def __init__(self, nbytes: int):
        self.ptr = C.c_void_p()
        self.nbytes = int(nbytes)
        _cabi.check(_cabi.lib().rbf_malloc(_cabi.ctx(), self.nbytes, C.byref(self.ptr)), _cabi.ctx())

    def to_host(self) -> np.ndarray:
        out = np.empty(self.nbytes, dtype=np.uint8)
        _cabi.check(_cabi.lib().rbf_memcpy_d2h(_cabi.ctx(), _cabi.ptr(out), self.ptr, self.nbytes), _cabi.ctx())
        return out

    def free(self):
        if self.ptr:
            _cabi.lib().rbf_free(_cabi.ctx(), self.ptr)
            self.ptr = None


def allgather_bitmaps(stream, pairs: int, slot_bytes: int, world: int):
    """One ncclAllGather of `pairs` fixed-size bitmap slots per rank -> DeviceBuffer [world][pairs][slot]."""
    send = DeviceBuffer(slot_bytes * pairs)
    recv = DeviceBuffer(slot_bytes * pairs * world)
    _cabi.check(_cabi.lib().rbf_stream_allgather_bitmaps(stream._h, pairs, slot_bytes, send.ptr, recv.ptr), _cabi.ctx())
    return send, recv


class PeerGather:
    """Receive buffers of all ranks mapped into this process (CUDA IPC) so that rbf_stream_allgather_bitmaps becomes one
    kernel writing over NVLink.  Layout of `recv`: [half 0|1][rank][pair][slot_bytes]; `result()` returns the half that
    holds the last exchange as uint8[world, pairs, slot]."""

    def __init__(self, dist, pairs: int, slot_bytes: int, _final_barrier: bool = True):
        L, ctx = _cabi.lib(), _cabi.ctx()
        self.world = dist.get_world_size() if dist is not None else 1
        self.rank = dist.get_rank() if dist is not None else 0
        self.pairs, self.slot = int(pairs), int(slot_bytes)
        self.recv = self.flags = None
        self._opened = []
        recv_ptrs, flag_ptrs = (C.c_void_p * self.world)(), (C.c_void_p * self.world)()
        mine = np.zeros((2, 64), dtype=np.uint8)
        exported = None
        try:                                              # allocation + export may fail on one rank only: the handle gather below
            self.recv = DeviceBuffer(2 * self.world * self.pairs * self.slot)    # is entered by every rank regardless
            self.flags = DeviceBuffer(256)
            _cabi.check(L.rbf_memset(ctx, self.flags.ptr, 0, 256), ctx)
            _cabi.check(L.rbf_sync(ctx), ctx)
            if self.world > 1:
                _cabi.check(L.rbf_peer_export(ctx, self.recv.ptr, _cabi.ptr(mine[0])), ctx)
                _cabi.check(L.rbf_peer_export(ctx, self.flags.ptr, _cabi.ptr(mine[1])), ctx)
            exported = mine.tobytes()
        except _cabi.RbfError:
            if self.world == 1:
                raise
        if self.world > 1:
            handles = [None] * self.world
            dist.all_gather_object(handles, exported)
            if any(h is None for h in handles):
                raise _cabi.RbfError("peer exchange: CUDA IPC export failed on rank(s) %s" % [r for r, h in enumerate(handles) if h is None])
            for r in range(self.world):                   # no collectives below: a failure here is reported through try_create
                if r == self.rank:
                    recv_ptrs[r], flag_ptrs[r] = self.recv.ptr.value, self.flags.ptr.value
                    continue
                h = np.frombuffer(handles[r], dtype=np.uint8).reshape(2, 64).copy()
                pr, pf = C.c_void_p(), C.c_void_p()
                _cabi.check(L.rbf_peer_open(ctx, _cabi.ptr(h[0]), C.byref(pr)), ctx)
                self._opened.append(pr)
                _cabi.check(L.rbf_peer_open(ctx, _cabi.ptr(h[1]), C.byref(pf)), ctx)
                self._opened.append(pf)
                recv_ptrs[r], flag_ptrs[r] = pr.value, pf.value
        else:
            recv_ptrs[0], flag_ptrs[0] = self.recv.ptr.value, self.flags.ptr.value
        _cabi.check(L.rbf_peer_gather_init(ctx, self.rank, self.world, recv_ptrs, flag_ptrs), ctx)
        if dist is not None and _final_barrier:
            dist.barrier()                                  # nobody pushes before every rank has mapped and zeroed

    @classmethod
    def try_create(cls, dist, pairs: int, slot_bytes: int):
        """PeerGather, or None on EVERY rank when CUDA IPC / peer access is unavailable on any rank (the caller then uses NCCL)."""
        obj, ok = None, True
        try:
            obj = cls(dist, pairs, slot_bytes, _final_barrier=False)
        except _cabi.RbfError:
            ok = False
        flags = [None] * dist.get_world_size()
        dist.all_gather_object(flags, ok)
        if all(flags):
            dist.barrier()
            return obj
        if obj is not None:
            obj.close(None)
        return None

    def exchange(self, stream) -> None:
        """Enqueue the push of the last encode's bit arrays (overlaps the next encode; complete after rbf_sync)."""
        _cabi.check(_cabi.lib().rbf_stream_allgather_bitmaps(stream._h, self.pairs, self.slot, None, self.recv.ptr), _cabi.ctx())

    def result(self) -> np.ndarray:
        half = C.c_uint32()
        _cabi.check(_cabi.lib().rbf_sync(_cabi.ctx()), _cabi.ctx())
        _cabi.check(_cabi.lib().rbf_peer_gather_half(_cabi.ctx(), C.byref(half)), _cabi.ctx())
        n = self.world * self.pairs * self.slot
        return self.recv.to_host()[half.value * n:(half.value + 1) * n].reshape(self.world, self.pairs, self.slot)

    def close(self, dist=None) -> None:
        L, ctx = _cabi.lib(), _cabi.ctx()
        L.rbf_peer_gather_shutdown(ctx)
        if dist is not None:
            dist.barrier()                                  # peers may still be writing into this rank's buffers
        for p in self._opened:
            L.rbf_peer_close(ctx, p)
        self._opened = []
        for b in (self.recv, self.flags):
            if b is not None:
                b.free()


class ShardedStreamEncoder:
    """One caller stream of `total_frames` frames coded by all ranks together (BASELINE configs[3], strong scaling): each rank
    uploads frames first_frame .. first_frame+frames-1 of the stream (its block plus the halo frame), `encode` runs the hot path
    on the block and exchanges the packed bit arrays with ONE all-gather, after which every rank holds the bit array of every
    pair of the stream.  The per-pair headers (l, |w|, p, k, ones, raw) travel as a small object gather next to it."""

    def __init__(self, dist, height: int, width: int, channels: int, dtype, total_frames: int, gather: str = "p2p",
                 max_l_bits: int = None):
        from .stream import FrameStream
        self.dist = dist
        self.world, self.rank = dist.get_world_size(), dist.get_rank()
        self.total_pairs = int(total_frames) - 1
        if self.total_pairs < self.world:
            # a rank without a pair has no block to code (its stream would hold the halo frame alone) and would leave the other
            # ranks waiting in the first collective; every rank sees the same arguments, so every rank raises here, before any
            # collective and before any device allocation
            raise ValueError("a stream of %d frames has %d frame pairs for %d ranks: every rank needs at least one pair"
                             % (int(total_frames), max(self.total_pairs, 0), self.world))
        self.layout = shard_layout(self.total_pairs, self.rank, self.world)
        self.gather = gather
        self.stream = FrameStream(height, width, channels, dtype, max_frames=self.layout["frames"],
                                  max_pairs=max(self.layout["pairs"], self.layout["slots"]))
        self.slot = 0
        self._send = self._recv = self._peer = None
        self._nccl_ready = False
        self.results = None
        if max_l_bits:                                        # size the all-gather slots for the densest frame expected, up front
            self._ensure_buffers(int(max_l_bits))

    def upload(self, frames_of_this_rank: np.ndarray) -> None:
        if frames_of_this_rank.shape[0] != self.layout["frames"]:
            raise ValueError("rank %d codes frames %d..%d of the stream: %d frames expected" %
                             (self.rank, self.layout["first_frame"], self.layout["first_frame"] + self.layout["frames"] - 1, self.layout["frames"]))
        self.stream.upload(frames_of_this_rank)

    def _ensure_buffers(self, max_l_bits: int) -> None:
        need = agree_slot_bytes(self.dist, max_l_bits)
        if need <= self.slot:
            return
        if self._peer is not None:
            self._peer.close(self.dist)
        for b in (self._send, self._recv):
            if b is not None:
                b.free()
        self.slot = need
        n = self.layout["slots"]
        if self.gather == "p2p":
            self._peer = PeerGather.try_create(self.dist, n, self.slot)
            if self._peer is None:
                self.gather = "nccl (p2p unavailable: CUDA IPC failed on some rank)"
        if self._peer is None:
            if not self._nccl_ready:
                init_nccl_from_torch(self.dist)
                self._nccl_ready = True
            self._send = DeviceBuffer(self.slot * n)
            self._recv = DeviceBuffer(self.slot * n * self.world)

    def encode(self, threshold: float, **kw):
        """Code this rank's block and enqueue the exchange (it overlaps the next encode; complete after `gathered()` / rbf_sync)."""
        self.results = self.stream.encode_consecutive(self.layout["frames"], threshold, **kw)
        max_l = max(r.l for r in self.results)
        if self.slot == 0:                                   # first encode: every rank is here, the agreement is collective
            self._ensure_buffers(max_l)                       # no head room: pass max_l_bits to the constructor for varying densities
        elif max_l > 8 * self.slot:
            # growing the slot is a collective decision; one rank must not start it alone (the others would never join)
            raise _cabi.RbfError("a bit array of %d bits does not fit the agreed all-gather slot of %d bytes: call renegotiate() on "
                                 "every rank (e.g. with the largest l expected) and encode again" % (max_l, self.slot))
        if self._peer is not None:
            self._peer.exchange(self.stream)
        else:
            _cabi.check(_cabi.lib().rbf_stream_allgather_bitmaps(self.stream._h, self.layout["slots"], self.slot, self._send.ptr,
                                                                 self._recv.ptr), _cabi.ctx())
        return self.results

    def renegotiate(self, max_l_bits: int) -> None:
        """Collective: re-agree the slot size (max over ranks of the given bound) and re-create the exchange buffers."""
        self.slot = 0
        self._ensure_buffers(int(max_l_bits))

    def gathered(self) -> np.ndarray:
        """uint8[total_pairs, slot]: the packbits bit array of every pair of the stream, in stream order (host copy)."""
        got = self._peer.result() if self._peer is not None else self._recv.to_host().reshape(self.world, self.layout["slots"], self.slot)
        return np.stack([got[r, t] for r, t in gathered_pair_rows(self.total_pairs, self.world)])

    def headers(self):
        """Per pair of the whole stream: (l, wlen, p, k, ones, raw) gathered from the owners."""
        mine = [(r.l, r.wlen, r.p, r.k, r.ones, r.raw) for r in self.results[: self.layout["pairs"]]]
        table = [None] * self.world
        self.dist.all_gather_object(table, mine)
        return [h for part in table for h in part]

    def close(self) -> None:
        if self._peer is not None:
            self._peer.close(self.dist)
        for b in (self._send, self._recv):
            if b is not None:
                b.free()
        self.stream.close()
