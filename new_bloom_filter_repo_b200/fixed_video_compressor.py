"""
Keyframe codec + YUV frame wrapper: host glue kept byte-compatible with the reference's
fixed_video_compressor.py (FixedVideoCompressor fvc:15-334) so that keyframe payloads written by
either implementation decode with the other.  zlib entropy coding is CPU work outside the
accelerated path (SURVEY.md section 8f, N4); nothing here touches the GPU (decompress_video inflates keyframe blobs of the
device coder on the GPU and builds the frame with build_frame).
"""
from __future__ import annotations

import math
import struct
import zlib
from typing import Dict, List

import numpy as np


class YUVFrame:
    """ndarray wrapper carrying the separate Y/U/V planes (fvc:289-334 `add_yuv_info_to_frame`)."""

    def __init__(self, data: np.ndarray, yuv_info: Dict = None):
        self.data = data
        if yuv_info is None:
            yuv_info = {"format": "YUV444", "y_plane": data[:, :, 0].copy(), "u_plane": data[:, :, 1].copy(),
                        "v_plane": data[:, :, 2].copy()}
        self.yuv_info = yuv_info

    shape = property(lambda self: self.data.shape)
    dtype = property(lambda self: self.data.dtype)
    nbytes = property(lambda self: self.data.nbytes)
    size = property(lambda self: self.data.size)
    T = property(lambda self: self.data.T)

    def __array__(self, dtype=None, copy=None):
        return self.data if dtype is None else self.data.astype(dtype)

    def copy(self):
        return YUVFrame(self.data.copy(), {k: (v.copy() if hasattr(v, "copy") else v) for k, v in self.yuv_info.items()})

    def __getitem__(self, key):
        return self.data[key]

    def __setitem__(self, key, value):
        self.data[key] = value

    def tobytes(self):
        return self.data.tobytes()

    def astype(self, dtype):
        return self.data.astype(dtype)

    def flatten(self):
        return self.data.flatten()

    def reshape(self, *a, **k):
        return self.data.reshape(*a, **k)


_DTYPES = {1: np.uint8, 2: np.uint16}


_PLANES = ("y_plane", "u_plane", "v_plane")


def keyframe_raws(frame) -> List[bytes]:
    """The buffers a keyframe payload compresses: the frame, then (YUV frames) the Y, U and V planes."""
    info = getattr(frame, "yuv_info", None)
    return [frame.tobytes()] + ([info[name].tobytes() for name in _PLANES] if info is not None else [])


def assemble_keyframe(frame, blobs: List[bytes]) -> bytes:
    """The keyframe byte layout around already compressed blobs (one per keyframe_raws(frame) entry, any zlib stream)."""
    info = getattr(frame, "yuv_info", None)
    parts: List[bytes] = [struct.pack("<III", frame.shape[0], frame.shape[1], frame.dtype.itemsize),
                          struct.pack("<I", len(blobs[0])), blobs[0], struct.pack("<B", 1 if info is not None else 0)]
    if info is not None:
        fmt = info.get("format", "YUV444").encode("utf-8")
        parts += [struct.pack("<H", len(fmt)), fmt]
        for zi, name in zip(blobs[1:], _PLANES):
            parts += [struct.pack("<I", len(zi)), zi, struct.pack("<II", *info[name].shape)]
    return b"".join(parts)


class FixedVideoCompressor:
    """Per-frame zlib level-9 codec (fvc:15-285): `<III` h, w, itemsize | `<I` len | zlib(frame) |
    `<B` has_yuv [| `<H` len fmt | fmt | 3 x (`<I` len | zlib(plane) | `<II` shape)]."""

    def __init__(self, verbose=True):
        self.verbose = verbose

    def compress_frame(self, frame) -> bytes:                                    # fvc:27-74
        return assemble_keyframe(frame, [zlib.compress(r, 9) for r in keyframe_raws(frame)])

    def decompress_frame(self, data: bytes):                                     # fvc:76-181
        return self.build_frame(data, zlib.decompress)

    @staticmethod
    def _parts(data: bytes, inflate):
        """The layout parse of a keyframe payload, one part at a time in payload order: ("frame", inflate(blob), (h, w, itemsize)),
        then for a YUV payload ("format", its utf-8 bytes, None) and ("y_plane" | "u_plane" | "v_plane", inflate(blob), (ph, pw)).
        Each blob is inflated as soon as its length is read, before the parse reads on, and each part is yielded before the next
        is read, so errors arise in payload order.  Raises struct.error on a truncated layout."""
        h, w, isz = struct.unpack_from("<III", data, 0)
        (zlen,) = struct.unpack_from("<I", data, 12)
        yield "frame", inflate(data[16:16 + zlen]), (h, w, isz)
        pos = 16 + zlen
        if not (pos < len(data) and data[pos] == 1):
            return
        (flen,) = struct.unpack_from("<H", data, pos + 1)
        yield "format", data[pos + 3:pos + 3 + flen], None
        pos += 3 + flen
        for name in _PLANES:
            (zl,) = struct.unpack_from("<I", data, pos)
            raw = inflate(data[pos + 4:pos + 4 + zl])
            yield name, raw, struct.unpack_from("<II", data, pos + 4 + zl)
            pos += 12 + zl

    @staticmethod
    def keyframe_blobs(data: bytes):
        """[(zlib blob, most bytes it may inflate to)] for the frame and, YUV frames, the three planes, in payload order; the
        bounds are h w itemsize 4 for the frame and ph pw for a plane.  Raises struct.error (or another exception) on a
        truncated layout, as decompress_frame would reach it."""
        return [(blob, math.prod(shape) * (4 if name == "frame" else 1))
                for name, blob, shape in FixedVideoCompressor._parts(data, lambda blob: blob) if name != "format"]

    def build_frame(self, data: bytes, inflate):
        """decompress_frame with inflate(blob) in place of zlib.decompress: called for the frame blob, then for each plane blob,
        at the points of the parse where decompress_frame inflates them."""
        parts = self._parts(data, inflate)
        _, raw, (h, w, isz) = next(parts)
        dtype = _DTYPES.get(isz, np.float32)
        gray = h * w * isz
        if len(raw) > gray and len(raw) % gray == 0:
            frame = np.frombuffer(raw, dtype=dtype).reshape((h, w, len(raw) // gray))
        else:
            frame = np.frombuffer(raw, dtype=dtype).reshape((h, w))
        info = {}
        for name, raw, shape in parts:
            info[name] = raw.decode("utf-8") if name == "format" else np.frombuffer(raw, dtype=np.uint8).reshape(shape)
        return YUVFrame(frame, info) if info else frame

    def compress_video(self, frames) -> List[bytes]:                             # fvc:183-198
        return [self.compress_frame(f) for f in frames]

    def decompress_video(self, compressed_frames) -> list:                       # fvc:200-215
        return [self.decompress_frame(c) for c in compressed_frames]

    def verify_lossless(self, original_frames, decompressed_frames) -> Dict:     # fvc:217-285
        if len(original_frames) != len(decompressed_frames):
            return {"lossless": False,
                    "reason": f"Frame count mismatch: {len(original_frames)} vs {len(decompressed_frames)}",
                    "avg_difference": float("inf")}
        exact, diff_frames, max_diff, max_diff_frame = 0, [], 0, -1
        for i, (o, d) in enumerate(zip(original_frames, decompressed_frames)):
            od = o.data if hasattr(o, "yuv_info") else np.asarray(o)
            dd = d.data if hasattr(d, "yuv_info") else np.asarray(d)
            if np.array_equal(od, dd):
                exact += 1
                continue
            fd = np.mean(np.abs(od.astype(np.float32) - dd.astype(np.float32)))
            diff_frames.append(i)
            if fd > max_diff:
                max_diff, max_diff_frame = fd, i
        ok = exact == len(original_frames)
        res = {"lossless": ok, "exact_lossless": ok, "avg_difference": 0.0 if not diff_frames else max_diff,
               "max_difference": max_diff, "max_diff_frame": max_diff_frame, "exact_frame_matches": exact,
               "total_frames": len(original_frames), "diff_frames": diff_frames}
        if self.verbose:
            print(f"Lossless verification: {'SUCCESS' if ok else 'FAILED'}")
            print(f"Exact frame matches: {exact}/{len(original_frames)}")
        return res

    def add_yuv_info_to_frame(self, yuv_frame):                                  # fvc:287-334
        return YUVFrame(yuv_frame)
