"""
FrameStream: Python handle on the C ABI's rbf_stream -- a device-resident store of
interleaved H x W x C frames plus the per-pair outputs of the batched hot path
(K1 threshold -> exact (k, l, T) on the host -> K2 insert -> K3 query -> K3b witness).
No PyTorch; device memory belongs to the C library.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence

import numpy as np

from . import _cabi
from ._cabi import MaskInfo


class PairResult:
    """What BloomFilterCompressor.compress returns for one frame pair (ivc:266), in wire form."""
    __slots__ = ("n", "ones", "resid", "l", "wlen", "p", "k", "raw", "floor_k", "act_T")

    def __init__(self, mi: MaskInfo):
        self.n, self.ones, self.resid, self.l, self.wlen = int(mi.n), int(mi.ones), int(mi.resid), int(mi.l), int(mi.wlen)
        self.p, self.k, self.raw, self.floor_k, self.act_T = float(mi.p), float(mi.k), bool(mi.raw), int(mi.floor_k), int(mi.act_T)

    def __repr__(self):
        return "PairResult(n=%d ones=%d l=%d wlen=%d k=%r raw=%s)" % (self.n, self.ones, self.l, self.wlen, self.k, self.raw)


class FrameStream:
    def __init__(self, height: int, width: int, channels: int = 3, dtype=np.uint8, max_frames: int = 2,
                 max_pairs: Optional[int] = None, k1_only: bool = False, mask_mode: int = 0, gray_mode: bool = False):
        dt = np.dtype(dtype)
        if dt not in (np.dtype(np.uint8), np.dtype(np.uint16)):
            raise ValueError("frames must be uint8 or uint16")
        self.H, self.W, self.C, self.dtype = int(height), int(width), int(channels), dt
        self.max_frames = int(max_frames)
        self.max_pairs = int(max_pairs if max_pairs is not None else max(1, max_frames - 1))
        self.npix = self.H * self.W
        self.mv_shape = ((self.H + 15) // 16, (self.W + 15) // 16)      # 16 x 16 motion blocks (rows, columns)
        self._h = C.c_void_p()
        _cabi.check(_cabi.lib().rbf_stream_create(_cabi.ctx(), self.H, self.W, self.C, dt.itemsize, self.max_frames,
                                                  self.max_pairs, C.byref(self._h)), _cabi.ctx())
        self._infos = (MaskInfo * self.max_pairs)()
        self.pairs = 0
        self.k1_only = bool(k1_only)
        for key, val in (("k1_only", int(bool(k1_only))), ("mask_mode", int(mask_mode)), ("gray_mode", int(bool(gray_mode)))):
            self.set_option(key, val)

    def set_option(self, key: str, value: int) -> None:
        """Per-stream option of the C ABI (rbf_stream_set_option): k1_only, mask_mode, gray_mode, value_mode (0: gather_changed and
        zlib_changed return the current samples; 1: residuals (curr - prev) mod 2^bits per sample), motion_values (1: residuals
        against the motion-compensated previous frame of the last motion_search)."""
        _cabi.check(_cabi.lib().rbf_stream_set_option(self._h, key.encode(), int(value)), _cabi.ctx())
        if key == "k1_only":
            self.k1_only = bool(value)

    def close(self):
        if getattr(self, "_h", None):
            _cabi.lib().rbf_stream_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ data movement
    def upload(self, frames: np.ndarray, first: int = 0) -> None:
        """frames: [count, H, W, C] (or [H, W, C]) contiguous array of the stream's dtype."""
        a = np.ascontiguousarray(frames)
        if a.ndim == 3 and self.C > 1 or (a.ndim == 2 and self.C == 1):
            a = a[None]
        if a.dtype != self.dtype or a.shape[1:3] != (self.H, self.W):
            raise ValueError("frame shape/dtype mismatch: %r %r" % (a.shape, a.dtype))
        _cabi.check(_cabi.lib().rbf_stream_upload(self._h, int(first), int(a.shape[0]), _cabi.ptr(a)), _cabi.ctx())

    # ------------------------------------------------------------------ the hot path
    def encode(self, prev_idx: Sequence[int], curr_idx: Sequence[int], threshold: float,
               seeds=_cabi.IVC_SEEDS, k_override=None, l_override=None) -> List[PairResult]:
        p = np.ascontiguousarray(np.asarray(prev_idx, dtype=np.uint32))
        c = np.ascontiguousarray(np.asarray(curr_idx, dtype=np.uint32))
        if p.shape != c.shape or p.ndim != 1:
            raise ValueError("prev_idx and curr_idx must be 1-D and equally long")
        sd = _cabi.seeds_struct(seeds)
        ko = lo = None
        if k_override is not None:
            ko = np.ascontiguousarray(np.asarray(k_override, dtype=np.float64))
            lo = np.ascontiguousarray(np.asarray(l_override, dtype=np.uint64))
        _cabi.check(_cabi.lib().rbf_stream_encode(self._h, _cabi.ptr(p), _cabi.ptr(c), p.size, float(threshold), C.byref(sd),
                                                  _cabi.ptr(ko) if ko is not None else None,
                                                  _cabi.ptr(lo) if lo is not None else None, self._infos), _cabi.ctx())
        self.pairs = int(p.size)
        return [PairResult(self._infos[i]) for i in range(self.pairs)]

    def encode_consecutive(self, nframes: int, threshold: float, **kw) -> List[PairResult]:
        idx = np.arange(nframes, dtype=np.uint32)
        return self.encode(idx[:-1], idx[1:], threshold, **kw)

    def fetch(self, pair: int, want_mask: bool = True):
        """-> (bitmap_packbits uint8[ceil(l/8)], witness_packbits uint8[ceil(wlen/8)], mask uint8[n] or None)."""
        mi = self._infos[pair]
        if self.k1_only:                                   # the encode stopped after K1: only the mask exists
            bm, wt = np.zeros(0, dtype=np.uint8), np.zeros(0, dtype=np.uint8)
        else:
            bm = np.zeros((int(mi.l) + 7) // 8, dtype=np.uint8)
            wt = np.zeros((int(mi.wlen) + 7) // 8, dtype=np.uint8)
        mk = np.zeros((self.npix + 7) // 8, dtype=np.uint8) if want_mask else None
        args = []                                          # one-pair slots of exactly each output's bytes; NULL, 0 for what is not copied
        for a, coded in ((bm, not mi.raw), (wt, not mi.raw), (mk, True)):
            copy = a is not None and a.size > 0 and coded
            args += [_cabi.ptr(a) if copy else None, a.size if copy else 0]
        _cabi.check(_cabi.lib().rbf_stream_fetch_batch(self._h, int(pair), 1, *args), _cabi.ctx())
        mask = np.unpackbits(mk, bitorder="little")[: self.npix] if mk is not None else None
        return bm, wt, mask

    def fetch_batch(self, first: int, count: int, want_masks: bool = False):
        """Packed outputs of pairs [first, first+count) with one D2H copy per kind and one sync:
        -> (bitmaps uint8[count, bslot], witnesses uint8[count, wslot], masks uint8[count, ceil(n/8)] or None);
        pair j's bitmap is bitmaps[j, :ceil(l_j/8)] (np.packbits order), its witness witnesses[j, :ceil(wlen_j/8)]."""
        infos = [self._infos[first + j] for j in range(count)]
        bslot = max(16, (max((int(m.l) + 7) // 8 for m in infos) + 15) // 16 * 16)
        wslot = max(16, (max((int(m.wlen) + 7) // 8 for m in infos) + 15) // 16 * 16)
        bm = np.zeros((count, bslot), dtype=np.uint8)
        wt = np.zeros((count, wslot), dtype=np.uint8)
        mslot = (self.npix + 7) // 8
        mk = np.zeros((count, mslot), dtype=np.uint8) if want_masks else None
        coded = not self.k1_only
        _cabi.check(_cabi.lib().rbf_stream_fetch_batch(self._h, int(first), int(count), _cabi.ptr(bm) if coded else None, bslot,
                                                       _cabi.ptr(wt) if coded else None, wslot,
                                                       _cabi.ptr(mk) if mk is not None else None, mslot), _cabi.ctx())
        return bm, wt, mk

    def decode_verify(self, pairs: Optional[int] = None) -> np.ndarray:
        """Decode every encoded pair on the GPU from its own bitmap + witness (ivc:268-307) and
        return the number of mismatching mask words per pair (all zeros == round trip holds)."""
        n = self.pairs if pairs is None else int(pairs)
        out = np.zeros(n, dtype=np.uint64)
        _cabi.check(_cabi.lib().rbf_stream_decode_verify(self._h, n, _cabi.ptr(out)), _cabi.ctx())
        return out

    # ------------------------------------------------------------------ N1 / N2 (SURVEY 8f)
    def gather_changed(self, pairs: Optional[int] = None) -> List[np.ndarray]:
        """Per encoded pair: interleaved channel values of the current frame at the mask's set positions (ivc:810-842)."""
        n = self.pairs if pairs is None else int(pairs)
        offs = np.zeros(n + 1, dtype=np.uint64)
        _cabi.check(_cabi.lib().rbf_stream_gather_changed(self._h, n, None, 0, _cabi.ptr(offs)), _cabi.ctx())
        buf = np.empty(int(offs[-1]), dtype=np.uint8)
        if buf.size:
            _cabi.check(_cabi.lib().rbf_stream_gather_changed(self._h, n, _cabi.ptr(buf), buf.size, _cabi.ptr(offs)), _cabi.ctx())
        return [buf[int(offs[i]):int(offs[i + 1])].view(self.dtype) for i in range(n)]

    def changed_offsets(self, pairs: Optional[int] = None) -> np.ndarray:
        """Byte offsets [pairs+1] of every encoded pair's changed values (what gather_changed returns), without the values."""
        n = self.pairs if pairs is None else int(pairs)
        offs = np.zeros(n + 1, dtype=np.uint64)
        _cabi.check(_cabi.lib().rbf_stream_gather_changed(self._h, n, None, 0, _cabi.ptr(offs)), _cabi.ctx())
        return offs

    def zlib_changed(self, pairs: Optional[int] = None) -> List[bytes]:
        """Per encoded pair: a zlib stream of what gather_changed returns, gathered and deflated on the GPU."""
        n = self.pairs if pairs is None else int(pairs)
        vo = self.changed_offsets(n)
        cap = sum(_cabi.zlib_bound(int(vo[i + 1] - vo[i])) for i in range(n))
        out = np.empty(cap, dtype=np.uint8)
        offs = np.zeros(n + 1, dtype=np.uint64)
        _cabi.check(_cabi.lib().rbf_stream_zlib_changed(self._h, n, _cabi.ptr(out), cap, _cabi.ptr(offs)), _cabi.ctx())
        return [out[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(n)]

    def motion_search(self, pairs: Optional[int] = None) -> np.ndarray:
        """Block motion of every encoded pair, prev -> curr: int8 [pairs, by, bx, 2] of (dx, dy) per 16 x 16 block in [-16, 16], the
        vector minimising the SAD of curr against prev(clamp(y + dy), clamp(x + dx)); ties go to the smaller |dx| + |dy|, then dy,
        then dx.  The fields stay in the stream for gathers with motion_values 1 until the next encode."""
        n = self.pairs if pairs is None else int(pairs)
        out = np.zeros((n,) + self.mv_shape + (2,), dtype=np.int8)
        _cabi.check(_cabi.lib().rbf_stream_motion_search(self._h, n, _cabi.ptr(out)), _cabi.ctx())
        return out

    def apply_diff(self, base_frame: int, mask: np.ndarray, values: np.ndarray) -> int:
        """Frame (base_frame + 1) % max_frames = frame base_frame with the pixels where `mask` is non-zero replaced by `values`, C
        samples of the stream's dtype per pixel in row-major order (apply_chain of one pair); returns pixels applied.  When values
        does not hold exactly C samples per set pixel, that frame is a copy of base_frame and 0 is returned (ivc:882).
        VideoFrameCompressor._apply_frame_diff passes `mask == 1` (ivc:869)."""
        m = np.asarray(mask)
        if m.size != self.npix:
            raise ValueError(f"a mask of {m.size} entries for frames of {self.npix} pixels")
        v = np.asarray(values)
        if v.dtype != self.dtype:
            raise ValueError(f"values of dtype {v.dtype} for a stream of {self.dtype}")
        mk = np.packbits((m != 0).reshape(-1), bitorder="little")
        vals = np.ascontiguousarray(v).view(np.uint8).reshape(-1)
        applied = C.c_uint64()
        _cabi.check(_cabi.lib().rbf_stream_apply_diff(self._h, int(base_frame), _cabi.ptr(mk), _cabi.ptr(vals) if vals.size else None,
                                                      vals.size, C.byref(applied)), _cabi.ctx())
        return int(applied.value)

    def download(self, frame: int) -> np.ndarray:
        return self.download_batch(frame, 1)[0]

    # ------------------------------------------------------------------ batched decode (K4b / K4c)
    def decode_masks(self, bitmaps: np.ndarray, witnesses: np.ndarray, l, wlen, k, raw, seeds=_cabi.IVC_SEEDS):
        """BloomFilterCompressor.decompress (ivc:268-307) of a group of pairs in one launch; the masks land in mask slots 0..count-1.
        bitmaps uint8[count, bslot]: row i holds np.packbits of pair i's l-bit array, or of its n-bit mask when raw[i];
        witnesses uint8[count, wslot] (wslot may be 0 when every pair is raw).  Bytes past a row's payload are ignored.
        -> (consumed uint64[count]: positions that passed the Bloom test, ones uint64[count]: set bits of each decoded mask)."""
        bm = np.ascontiguousarray(bitmaps, dtype=np.uint8)
        wt = np.ascontiguousarray(witnesses, dtype=np.uint8)
        count = bm.shape[0]
        ls, ws = np.ascontiguousarray(l, dtype=np.uint64), np.ascontiguousarray(wlen, dtype=np.uint64)
        ks, rs = np.ascontiguousarray(k, dtype=np.float64), np.ascontiguousarray(raw, dtype=np.uint8)
        if wt.shape[0] != count or not (ls.size == ws.size == ks.size == rs.size == count):
            raise ValueError("one bitmap, witness, l, wlen, k and raw flag per pair")
        consumed = np.zeros(count, dtype=np.uint64)
        ones = np.zeros(count, dtype=np.uint64)
        sd = _cabi.seeds_struct(seeds)
        wslot = wt.shape[1] if wt.ndim == 2 else 0
        _cabi.check(_cabi.lib().rbf_stream_decode_masks(self._h, count, _cabi.ptr(bm), bm.shape[1], _cabi.ptr(wt) if wslot else None,
                                                        wslot, _cabi.ptr(ls), _cabi.ptr(ws), _cabi.ptr(ks), _cabi.ptr(rs),
                                                        C.byref(sd), _cabi.ptr(consumed), _cabi.ptr(ones)), _cabi.ctx())
        self.pairs = 0
        return consumed, ones

    def apply_chain(self, base_frame: int, values: Optional[Sequence[np.ndarray]] = None, *, inflated: Optional[Sequence[int]] = None,
                    modes: Optional[Sequence[int]] = None, motion: Optional[Sequence[Optional[np.ndarray]]] = None) -> np.ndarray:
        """Frame base_frame+1+i = frame base_frame+i with mask slot i applied, pair i's values replacing its set pixels in rank order
        (ivc:849-909), for every pair i; slots are taken modulo max_frames.  Pair i's values are either values[i] (host arrays) or,
        with `inflated`, the first inflated[i] bytes of the i-th stream the last inflate_values placed (every one of them inflated
        on the device, in order): those never cross PCIe, and the call ends their use.  Exactly one of the two is given.
        modes[i] = 1 adds the values to the set pixels per sample (mod 2^bits) instead: the residuals a value_mode=1 gather returns.
        modes[i] = 2 adds them to the motion-compensated prediction from frame base_frame+i under motion[i], pair i's int8 field
        of motion_search's shape [by, bx, 2] (motion[j] is ignored, and may be None, for the other pairs): the residuals a
        motion_values=1 gather returns.  A mode-2 pair whose motion[i] is None raises ValueError, and one without `motion` raises
        RbfError.  -> uint64[count] pixels applied per pair: 0 from the first pair whose value count does not match its mask
        (ivc:882), whose frame and every later one are not written."""
        if (values is None) == (inflated is None):
            raise ValueError("pass either values or inflated")
        buf = None
        if values is not None:
            parts = [memoryview(np.ascontiguousarray(v)).cast("B") for v in values]
            sizes = [p.nbytes for p in parts]
            buf = np.frombuffer(b"".join(parts), dtype=np.uint8)
        else:
            sizes = np.asarray(inflated, dtype=np.uint64)
        count = len(sizes)
        offs = np.zeros(count + 1, dtype=np.uint64)
        offs[1:] = np.cumsum(sizes)
        applied = np.zeros(count, dtype=np.uint64)
        flags = fields = None
        if modes is not None:
            flags = np.ascontiguousarray(np.asarray(modes, dtype=np.uint8))
            if flags.shape != (count,):
                raise ValueError("one value mode per pair")
            if motion is not None and (flags == 2).any():
                fields = self._motion_fields(flags, motion)
        _cabi.check(_cabi.lib().rbf_stream_apply_chain(self._h, int(base_frame), count, _cabi.ptr(buf) if buf is not None and buf.size else None,
                                                       _cabi.ptr(offs), _cabi.ptr(flags) if flags is not None else None,
                                                       _cabi.ptr(fields) if fields is not None else None, _cabi.ptr(applied)),
                    _cabi.ctx())
        return applied

    def _motion_fields(self, flags: np.ndarray, motion) -> np.ndarray:
        """The [count, by, bx, 2] int8 fields of apply_chain's mode-2 pairs (zero for the others)."""
        fields = np.zeros((flags.size,) + self.mv_shape + (2,), dtype=np.int8)
        for i in np.flatnonzero(flags == 2):
            f = motion[i] if i < len(motion) else None
            if f is None:
                raise ValueError(f"pair {i} is a motion pair without a motion field")
            f = np.asarray(f)
            if f.dtype != np.int8 or f.size != fields[i].size:
                raise ValueError(f"pair {i}: a motion field is {fields[i].size} int8 values, not {f.size} {f.dtype}")
            fields[i] = f.reshape(fields[i].shape)
        return fields

    def inflate_values(self, streams: Sequence, bounds: Sequence[int]):
        """The zlib value streams of a group inflated on the GPU into the stream's value buffer, for apply_chain(inflated=...).
        bounds[i]: the most stream i may hold (its value count x sample bytes).  -> (inflated bytes uint64[n], on_device bool[n]);
        a declined stream (not the device coder's layout, or larger than its bound) has on_device False and 0 bytes."""
        views = [np.frombuffer(memoryview(s).cast("B"), dtype=np.uint8) for s in streams]
        n = len(views)
        lens = np.array([v.size for v in views], dtype=np.uint64)
        bnd = np.ascontiguousarray(np.asarray(bounds, dtype=np.uint64))
        srcs = (C.c_void_p * n)(*[v.ctypes.data if v.size else None for v in views])
        out = np.zeros(n, dtype=np.uint64)
        ok = np.zeros(n, dtype=np.uint8)
        _cabi.check(_cabi.lib().rbf_stream_inflate_values(self._h, n, srcs, _cabi.ptr(lens), _cabi.ptr(bnd), _cabi.ptr(out), _cabi.ptr(ok)),
                    _cabi.ctx())
        return out, ok.astype(bool)

    def download_batch(self, first: int, count: int) -> np.ndarray:
        """Frames first .. first+count-1 (slots modulo max_frames) -> [count, H, W(, C)], one copy and one synchronisation."""
        shape = (int(count), self.H, self.W, self.C) if self.C > 1 else (int(count), self.H, self.W)
        out = np.empty(shape, dtype=self.dtype)
        _cabi.check(_cabi.lib().rbf_stream_download_batch(self._h, int(first), int(count), _cabi.ptr(out)), _cabi.ctx())
        return out

    def copy_frames(self, first: int, count: int, ptr: int, capacity: int, stream: int = 0) -> None:
        """download_batch into device memory: frames first .. first+count-1 (slots modulo max_frames) to the device address `ptr`,
        back to back, `capacity` bytes at most.  `stream` (a __cuda_array_interface__ v3 stream: 0 none, 1 legacy default, 2
        per-thread default, else a cudaStream_t) is waited for before the buffer is written; returns when the copy is done."""
        _cabi.check(_cabi.lib().rbf_stream_copy_frames(self._h, int(first), int(count), C.c_void_p(int(ptr) or None), int(capacity),
                                                       int(stream)), _cabi.ctx())

    def stage_ms(self) -> dict:
        out = (C.c_double * 6)()
        _cabi.check(_cabi.lib().rbf_stream_stage_ms(self._h, out), _cabi.ctx())
        return dict(zip(("k1_threshold", "front_k1_host_k2", "k2_insert", "k3_query", "k3b_witness", "encode_total"),
                        [float(x) for x in out]))

    def encode_host(self, frames: np.ndarray, threshold: float, seeds=_cabi.IVC_SEEDS, bitmap_slot: int = 0,
                    witness_slot: int = 0, out_bitmaps: np.ndarray = None, out_witness: np.ndarray = None):
        """End-to-end call: host frames in, packed bitmaps/witnesses back in host slots (copies included)."""
        a = np.ascontiguousarray(frames)
        nfr = a.shape[0]
        sd = _cabi.seeds_struct(seeds)
        _cabi.check(_cabi.lib().rbf_stream_encode_host(
            self._h, _cabi.ptr(a), nfr, float(threshold), C.byref(sd), self._infos,
            _cabi.ptr(out_bitmaps) if out_bitmaps is not None else None, int(bitmap_slot),
            _cabi.ptr(out_witness) if out_witness is not None else None, int(witness_slot)), _cabi.ctx())
        self.pairs = nfr - 1
        return [PairResult(self._infos[i]) for i in range(self.pairs)]
