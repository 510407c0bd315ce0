"""
zlib streams coded on the GPU (rbf_zlib_compress_batch, csrc/rbf_deflate.cuh).  Every stream is a valid zlib stream that
zlib.decompress reads; its bytes differ from zlib.compress's (independent 64 KiB segments, greedy LZ77, one dynamic-Huffman
block per segment), the decoded data do not.  No CPU fallback: without the library and an H100 these functions raise.

decompress_many inflates streams in that layout on the GPU (rbf_zlib_decompress_batch, csrc/rbf_inflate.cuh) and every other
stream with zlib.decompress, so it returns exactly what zlib.decompress returns, or raises its zlib.error.
"""
from __future__ import annotations

import ctypes as C
import zlib
from typing import Iterable, List, Optional, Sequence, Tuple

import numpy as np

from . import _cabi


def _byte_view(buf) -> np.ndarray:
    m = memoryview(buf)
    if not m.c_contiguous:
        raise ValueError("deflate needs C-contiguous buffers")
    return np.frombuffer(m.cast("B"), dtype=np.uint8) if m.nbytes else np.zeros(0, dtype=np.uint8)


def compress_many(buffers: Iterable) -> List[bytes]:
    """One zlib stream per buffer (bytes-like objects or C-contiguous arrays), coded in one batch on the GPU."""
    views = [_byte_view(b) for b in buffers]
    n = len(views)
    if n == 0:
        return []
    lens = np.array([v.size for v in views], dtype=np.uint64)
    srcs = (C.c_void_p * n)(*[v.ctypes.data if v.size else None for v in views])
    cap = sum(_cabi.zlib_bound(int(x)) for x in lens)
    out = np.empty(cap, dtype=np.uint8)
    offs = np.zeros(n + 1, dtype=np.uint64)
    _cabi.check(_cabi.lib().rbf_zlib_compress_batch(_cabi.ctx(), n, srcs, _cabi.ptr(lens), 0, _cabi.ptr(out), cap,
                                                    _cabi.ptr(offs)), _cabi.ctx())
    return [out[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(n)]


def compress(data) -> bytes:
    """zlib stream of one buffer, coded on the GPU."""
    return compress_many([data])[0]


_DEVICE_HEADER = b"\x78\x9c"
_MAX_RATIO = 1032                     # deflate's largest inflate ratio: the default bound of a stream


def decompress_routed(streams: Iterable, bounds: Optional[Sequence[int]] = None) -> Tuple[List[bytes], List[bool]]:
    """(decompress_many(streams, bounds), whether each stream was inflated on the GPU)."""
    views = [_byte_view(s) for s in streams]
    out: List[Optional[bytes]] = [None] * len(views)
    on_device = [False] * len(views)
    dev = [i for i, v in enumerate(views) if v.size >= 2 and v[:2].tobytes() == _DEVICE_HEADER]
    if dev:
        n = len(dev)
        lens = np.array([views[i].size for i in dev], dtype=np.uint64)
        bnd = np.array([int(bounds[i]) if bounds is not None else _MAX_RATIO * views[i].size for i in dev], dtype=np.uint64)
        srcs = (C.c_void_p * n)(*[views[i].ctypes.data for i in dev])
        cap = min(int(bnd.sum()), 1 << 31)
        buf = np.empty(max(cap, 1), dtype=np.uint8)
        offs = np.zeros(n + 1, dtype=np.uint64)
        ok = np.zeros(n, dtype=np.uint8)
        _cabi.check(_cabi.lib().rbf_zlib_decompress_batch(_cabi.ctx(), n, srcs, _cabi.ptr(lens), _cabi.ptr(bnd), _cabi.ptr(buf), cap,
                                                          _cabi.ptr(offs), _cabi.ptr(ok)), _cabi.ctx())
        for k, i in enumerate(dev):
            if ok[k]:
                out[i] = buf[int(offs[k]):int(offs[k + 1])].tobytes()
                on_device[i] = True
    return [o if o is not None else zlib.decompress(v) for o, v in zip(out, views)], on_device


def decompress_many(streams: Iterable, bounds: Optional[Sequence[int]] = None) -> List[bytes]:
    """[zlib.decompress(s) for s in streams], with the streams in the device coder's layout inflated on the GPU in one batch.
    bounds[i], when given, is the most stream i may inflate to on the GPU (it sizes the device scratch; the default is deflate's
    largest ratio); a stream beyond its bound, outside the layout, or not starting with 78 9C goes to zlib.decompress, which
    also raises for bad streams."""
    return decompress_routed(streams, bounds)[0]


def decompress(data) -> bytes:
    """zlib.decompress(data), inflated on the GPU when the stream is in the device coder's layout."""
    return decompress_many([data])[0]
