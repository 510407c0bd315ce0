"""
zlib streams coded on the GPU (rbf_zlib_compress_batch, csrc/rbf_deflate.cuh).  Every stream is a valid zlib stream that
zlib.decompress reads; its bytes differ from zlib.compress's (independent 64 KiB segments, greedy LZ77, one dynamic-Huffman
block per segment), the decoded data do not.  No CPU fallback: without the library and an H100 these functions raise.
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, List

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
