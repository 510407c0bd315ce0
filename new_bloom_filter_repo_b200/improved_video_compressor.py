"""
Drop-in for the reference's improved_video_compressor.py on the rational-Bloom hot path:

    RationalBloomFilter      ivc:39-138    (integer indices, seeds 0x12345678 / 0x87654321 / 999)
    BloomFilterCompressor    ivc:140-307   (compress / decompress of a 0/1 vector)
    VideoFrameCompressor     ivc:671-1234  (_calculate_frame_diff, _apply_frame_diff,
                                            _compress/_decompress_frame_differences, keyframe codec)
    ImprovedVideoCompressor  ivc:309-523   (compress_video / decompress_video / verify_lossless)

Same names, arguments, return shapes and error behaviour; the per-pixel thresholding, the XXH64
double hashing, the probabilistic floor(k*)+1'th probe and the bit-array set/test run as sm_90a
kernels behind the C ABI (include/rbf_b200.h).  No host implementation of those exists in this
package: without librbf_b200.so and an H100 every entry point raises.

Where the reference is unwired (SURVEY.md section 0): `VideoFrameCompressor.bloom_compressor` is
assigned here (the reference never does), and `ImprovedVideoCompressor.compress_video` gains the
keyframe / inter-frame loop the reference's `keyframe_interval` argument promises; with
`keyframe_interval=1` its output is byte-identical to the reference's (all keyframes, ivc:390).
"""
from __future__ import annotations

import bisect
import ctypes as C
import io
import math
import operator
import os
import struct
import time
import zlib
from concurrent.futures import Future
from functools import partial
from typing import Dict, List, Optional, Tuple

import numpy as np

from . import _cabi, deflate
from .fixed_video_compressor import FixedVideoCompressor, YUVFrame, assemble_keyframe, keyframe_raws
from .rational_bloom_filter import _DeviceFilter
from .stream import FrameStream


class RationalBloomFilter:
    """ivc.RationalBloomFilter (ivc:39-138).  `bit_array` is fetched from / written to the device copy."""

    def __init__(self, size: int, k_star: float, seeds=None):
        self.size = size                                      # ivc:55
        self.k_star = k_star                                  # ivc:56
        self.floor_k = math.floor(k_star)                     # ivc:57
        self.p_activation = k_star - self.floor_k             # ivc:58
        self.h1_seed = 0x12345678 if seeds is None else seeds[0]   # ivc:62
        self.h2_seed = 0x87654321 if seeds is None else seeds[1]   # ivc:63
        self._act_seed = 999 if seeds is None else seeds[2]        # ivc:94
        self._dev = _DeviceFilter(size, k_star, (self.h1_seed, self.h2_seed, self._act_seed))

    @property
    def bit_array(self) -> np.ndarray:                        # ivc:59 (np.uint8[size], one byte per bit)
        """A read-only snapshot of the device bits: in-place writes (`f.bit_array[i] = 1`) would be lost, so they raise;
        assign a whole array instead (`f.bit_array = bits`, as ivc:290 does)."""
        a = self._dev.get_bits()
        a.setflags(write=False)
        return a

    @bit_array.setter
    def bit_array(self, bits) -> None:                        # `bloom_filter.bit_array = bloom_bitmap`, ivc:290
        self._dev.set_bits(bits)

    def _get_hash_indices(self, item: int, i: int) -> int:    # ivc:65-81
        b = str(item).encode("utf-8")
        return _cabi.lib().rbf_probe_index(_cabi.xxh64(b, self.h1_seed), _cabi.xxh64(b, self.h2_seed), int(i), int(self.size))

    def _determine_activation(self, item: int) -> bool:       # ivc:83-97
        return _cabi.xxh64(str(item).encode("utf-8"), self._act_seed) < _cabi.activation_threshold(self.p_activation)

    @staticmethod
    def _split(indices):
        """uint32 items go to the decimal-index kernels; anything else the reference would hash as str(item) -- negative or
        >= 2**32 integers, floats, strings, bools ("True") -- goes through the string kernels, so `str(item)` semantics hold."""
        arr = np.asarray(indices)
        if arr.dtype.kind in "iu" and arr.size and (arr.dtype.kind == "u" or int(arr.min()) >= 0) and int(arr.max()) < 2 ** 32:
            return arr.astype(np.uint32, copy=False).reshape(-1), None
        if arr.size == 0:
            return np.zeros(0, dtype=np.uint32), None
        return None, [str(int(x)) if isinstance(x, (int, np.integer)) and not isinstance(x, (bool, np.bool_)) else str(x)
                      for x in np.asarray(indices, dtype=object).reshape(-1)]

    def add_index(self, index: int) -> None:                  # ivc:99-114
        self.add_indices([index])

    def check_index(self, index: int) -> bool:                # ivc:116-138
        return bool(self.check_indices([index])[0])

    def add_indices(self, indices) -> None:                   # batch form: one launch
        u32, strs = self._split(indices)
        if strs is None:
            self._dev.add_indices(u32)
        else:
            self._dev.add_strings(strs)

    def check_indices(self, indices) -> np.ndarray:
        u32, strs = self._split(indices)
        if strs is None:
            return self._dev.check_indices(u32).astype(bool)
        return self._dev.check_strings(strs).astype(bool)


class BloomFilterCompressor:
    """ivc.BloomFilterCompressor (ivc:140-307)."""

    P_STAR = 0.32453                                          # ivc:150

    def __init__(self, verbose: bool = False, seeds=_cabi.IVC_SEEDS):
        self.verbose = verbose
        self._seeds = seeds

    def _calculate_optimal_params(self, n: int, p: float) -> Tuple[float, int]:   # ivc:161-196
        if p <= 0.0001:
            return 0, 0
        if p >= self.P_STAR:
            return 0, 0
        q = 1 - p
        L = math.log(2)
        k = math.log2(q * (L ** 2) / p)
        if math.isnan(k) or k <= 0:
            return 0, 0
        gamma = 1 / L
        l = int(p * n * k * gamma)
        return max(0.1, k), max(1, l)

    def compress(self, binary_input: np.ndarray, k_l_override=None):             # ivc:198-266
        """-> (bloom_filter_bitmap, witness, density, input_length, compression_ratio)"""
        arr = np.asarray(binary_input)
        n = len(arr)
        if n == 0:                                            # the reference divides 0/0 -> nan and falls through to the
            with np.errstate(invalid="ignore", divide="ignore"):   # raw-passthrough branch (ivc:212, ivc:188-189, ivc:223-225)
                p = np.float64(0.0) / np.float64(0.0)
            return binary_input, [], p, 0, 1.0
        m8 = np.ascontiguousarray(arr, dtype=np.uint8)
        if m8.size and m8.max() > 1:
            raise ValueError("binary_input must hold 0/1 values")
        info = _cabi.MaskInfo()
        bitmap = np.empty(n, dtype=np.uint8)
        witness = np.empty(n, dtype=np.uint8)
        sd = _cabi.seeds_struct(self._seeds)
        ko, lo = (0.0, 0) if k_l_override is None else (float(k_l_override[0]), int(k_l_override[1]))
        _cabi.check(_cabi.lib().rbf_compress_mask(_cabi.ctx(), _cabi.ptr(m8), n, C.byref(sd), ko, lo, C.byref(info),
                                                  _cabi.ptr(bitmap), _cabi.ptr(witness)), _cabi.ctx())
        p = np.float64(info.p)
        self.last_info = info
        if info.raw:                                          # ivc:215-218, ivc:223-225
            if self.verbose and p >= self.P_STAR:
                print(f"Density {p:.4f} is >= threshold {self.P_STAR}, compression not effective")
            return binary_input, [], p, n, 1.0
        l, wlen = int(info.l), int(info.wlen)
        if self.verbose:
            print(f"Input length: {n}, Density: {p:.4f}")
            print(f"Optimal parameters: k={info.k:.4f}, l={l}")
            print(f"Bloom filter size: {l} bits")
            print(f"Witness size: {wlen} bits")
        ratio = (l + wlen) / n                                # ivc:256-258
        return bitmap[:l].copy(), list(witness[:wlen]), p, n, ratio

    def decompress(self, bloom_bitmap: np.ndarray, witness: list, n: int, k: float) -> np.ndarray:   # ivc:268-307
        if len(witness) == 0:                                 # ivc:282-284
            return bloom_bitmap
        bm = np.ascontiguousarray(np.asarray(bloom_bitmap, dtype=np.uint8))
        wt = np.ascontiguousarray(np.asarray(witness, dtype=np.uint8))
        out = np.empty(n, dtype=np.uint8)
        consumed = C.c_uint64()
        sd = _cabi.seeds_struct(self._seeds)
        _cabi.check(_cabi.lib().rbf_decompress_mask(_cabi.ctx(), _cabi.ptr(bm), len(bm), _cabi.ptr(wt), len(wt), int(n),
                                                    float(k), C.byref(sd), _cabi.ptr(out), C.byref(consumed)), _cabi.ctx())
        if consumed.value > len(wt):                          # the reference's witness[witness_idx] raises here
            raise IndexError("list index out of range")
        return out


def _frame_data(frame) -> np.ndarray:
    return frame.data if hasattr(frame, "yuv_info") else np.asarray(frame)


def _done(value) -> Future:
    f = Future()
    f.set_result(value)
    return f


class VideoFrameCompressor:
    """The inter-frame pieces of ivc.VideoFrameCompressor (ivc:671-1234)."""

    def __init__(self, noise_tolerance: float = 10.0, keyframe_interval: int = 30, min_diff_threshold: float = 3.0,
                 max_diff_threshold: float = 30.0, bloom_threshold_modifier: float = 1.0, num_threads: int = None,
                 use_direct_yuv: bool = False, verbose: bool = False):
        self.noise_tolerance = noise_tolerance
        self.keyframe_interval = keyframe_interval
        self.min_diff_threshold = min_diff_threshold
        self.max_diff_threshold = max_diff_threshold
        self.bloom_threshold_modifier = bloom_threshold_modifier
        self.use_direct_yuv = use_direct_yuv
        self.verbose = verbose
        self.num_threads = max(1, (os.cpu_count() or 2) - 1) if num_threads is None else max(1, num_threads)  # ivc:714-717
        self.bloom_compressor = BloomFilterCompressor(verbose=False)   # the attribute ivc:927 needs
        self._streams: Dict[tuple, FrameStream] = {}

    def _estimate_noise_level(self, frame: np.ndarray) -> float:                  # ivc:727-746
        """N3: the 5x5 median runs on the device (k_median5, bit-exact with cv2.medianBlur); the float32 std is numpy's,
        exactly as in the reference.  An (h, w, 1) plane is filtered as (h, w), which is the shape cv2 returns for it; the
        difference then broadcasts (h, w, 1) against (h, w) as the reference's does, so it raises ValueError unless numpy can
        broadcast the two shapes."""
        a = np.ascontiguousarray(_frame_data(frame))
        if not (a.ndim == 2 or (a.ndim == 3 and a.shape[2] == 1)) or a.dtype not in (np.uint8, np.uint16):
            raise NotImplementedError("noise estimate is implemented for 2-D uint8/uint16 planes (the Y / gray plane)")
        smoothed = np.empty(a.shape[:2], dtype=a.dtype)
        _cabi.check(_cabi.lib().rbf_median_blur5(_cabi.ctx(), _cabi.ptr(a), a.shape[0], a.shape[1], a.dtype.itemsize,
                                                 _cabi.ptr(smoothed)), _cabi.ctx())
        noise = a.astype(np.float32) - smoothed.astype(np.float32)                 # ivc:741
        return np.std(noise)                                                       # ivc:744

    def _adaptive_diff_threshold(self, frame: np.ndarray) -> float:               # ivc:748-766
        noise_level = self._estimate_noise_level(frame)
        return max(self.min_diff_threshold, min(self.max_diff_threshold, noise_level * self.noise_tolerance))

    def _stream_for(self, shape, dtype, k1_only: bool = False, gray: bool = False) -> FrameStream:
        """Cached 2-frame device store per (shape, dtype, options).  Options are per-stream state of the C ABI, so several
        compressors (or threads with their own compressor) never flip a shared switch."""
        key = (tuple(shape), np.dtype(dtype).str, bool(k1_only), bool(gray))
        s = self._streams.get(key)
        if s is None:
            ch = shape[2] if len(shape) == 3 else 1
            s = FrameStream(shape[0], shape[1], ch, dtype, max_frames=2, max_pairs=1, k1_only=k1_only, gray_mode=gray)
            self._streams[key] = s
        return s

    @staticmethod
    def _bgr2gray(a: np.ndarray) -> np.ndarray:
        """cv2.cvtColor(a, cv2.COLOR_BGR2GRAY) for uint8/uint16 (OpenCV's 15-bit fixed point; ivc:794-795) -- used on the host
        only to feed the adaptive-threshold noise estimate; the mask itself is computed by K1 in gray mode."""
        x = a.astype(np.uint32)
        return ((x[:, :, 0] * 3735 + x[:, :, 1] * 19235 + x[:, :, 2] * 9798 + 16384) >> 15).astype(a.dtype)

    def _calculate_frame_diff(self, prev_frame, curr_frame, threshold: Optional[float] = None):
        """ivc:768-847 -> (binary_diff uint8, changed_values, diff_density).  The mask is computed by K1: on the first
        channel (Y) for `use_direct_yuv` frames, on the BGR->gray conversion otherwise (ivc:788-795), or on the single plane.
        It is H x W for colour frames and has the frame's shape otherwise, (h, w, 1) included (ivc:797-808)."""
        pd, cd = _frame_data(prev_frame), _frame_data(curr_frame)
        is_color = pd.ndim > 2 and pd.shape[2] > 1
        gray = is_color and not (self.use_direct_yuv and pd.shape[2] >= 3)
        if gray and pd.shape[2] != 3:
            raise NotImplementedError("BGR->gray masks are implemented for 3-channel frames (cv2.COLOR_BGR2GRAY, ivc:794-795)")
        if pd.dtype not in (np.uint8, np.uint16) or pd.shape != cd.shape or pd.dtype != cd.dtype:
            raise ValueError("frames must be equal-shape uint8/uint16 arrays")
        if threshold is None:                                  # ivc:804-805: adaptive threshold from the current Y / gray plane
            plane = (self._bgr2gray(cd) if gray else cd[:, :, 0].copy()) if is_color else cd.copy()
            threshold = self._adaptive_diff_threshold(plane)
        st = self._stream_for(pd.shape, pd.dtype, k1_only=True, gray=gray)
        st.upload(np.stack([pd, cd]))
        res = st.encode([0], [1], float(threshold))[0]
        _, _, flat = st.fetch(0)                               # k1_only stream: the mask is the only output
        binary_diff = flat.reshape(pd.shape[:2] if is_color else pd.shape).astype(np.uint8)
        vals = st.gather_changed(1)[0]                        # N1: ordered gather on the device (ivc:810-842)
        if is_color and self.use_direct_yuv and hasattr(curr_frame, "yuv_info"):
            changed = vals.astype(np.uint8)                   # ivc:825 allocates uint8: 16-bit samples are truncated there too
        else:
            changed = vals.copy()                             # ivc:832-842 keep the frame dtype
        density = res.ones / binary_diff.size                  # ivc:845
        self._last_pair_result = res
        return binary_diff, changed, density

    def _apply_frame_diff(self, base_frame, diff_mask: np.ndarray, changed_values: np.ndarray):   # ivc:849-909
        """N2: the apply runs on the device (the K4c sweep of one pair); the result is a copy of base_frame's type.  Only mask entries
        equal to 1 are applied (ivc:869).  Colour frames keep the base when the value count is not pixels x channels (ivc:882);
        grayscale frames, (h, w, 1) included, follow numpy's `frame[mask == 1] = values` (ivc:906-907): one value is broadcast,
        another count raises ValueError, and a mask without a set pixel leaves the frame as it is whatever the values.
        Formats the device store does not hold, and values of another dtype, are applied by the same numpy indexing on the host."""
        nxt = base_frame.copy()
        data = _frame_data(nxt)
        vals = np.asarray(changed_values)
        sel = np.asarray(diff_mask) == 1                       # ivc:869
        color = data.ndim == 3 and data.shape[2] > 1
        device = (data.dtype in (np.uint8, np.uint16) and vals.dtype == data.dtype and vals.ndim == 1 and
                  data.ndim in (2, 3) and (data.ndim == 2 or data.shape[2] in (1, 3)) and
                  sel.shape == (data.shape[:2] if color else data.shape))
        if device and not color and vals.size != np.count_nonzero(sel):
            device = False                                     # numpy decides: a broadcast, a ValueError or an empty mask
        if device:
            st = self._stream_for(data.shape, data.dtype, k1_only=True)
            st.upload(np.ascontiguousarray(data)[None], first=0)
            st.apply_diff(0, sel, vals)                        # frame 1; a value-count mismatch leaves the base unchanged (ivc:882)
            data[...] = st.download(1).reshape(data.shape)
        elif color:                                            # ivc:872-903
            rows, cols = np.nonzero(sel)
            if len(vals) == len(rows) * data.shape[2]:
                data[rows, cols] = vals.reshape(-1, data.shape[2])
        else:                                                  # ivc:904-907
            idx = np.nonzero(sel)
            if len(idx[0]) > 0:
                data[idx] = vals
        if self.use_direct_yuv and hasattr(nxt, "yuv_info") and data.ndim == 3:
            nxt.yuv_info["y_plane"] = data[:, :, 0].copy()
            nxt.yuv_info["u_plane"] = data[:, :, 1].copy()
            nxt.yuv_info["v_plane"] = data[:, :, 2].copy()
        return nxt

    def _compress_frame_differences(self, binary_diff: np.ndarray, changed_values: np.ndarray) -> Tuple[bytes, float]:
        """ivc:911-967: `<f` p | `<I` n | `<f` k | `<I` l | `<I` |w| | packbits(bitmap) | packbits(witness) | zlib(values)."""
        flat = binary_diff.flatten()
        bitmap, witness, p, n, _ = self.bloom_compressor.compress(flat)
        buf = io.BytesIO()
        buf.write(struct.pack("<f", p))
        buf.write(struct.pack("<I", n))
        k, l = self.bloom_compressor._calculate_optimal_params(n, p)     # ivc:937
        buf.write(struct.pack("<f", k))
        buf.write(struct.pack("<I", len(bitmap)))
        buf.write(struct.pack("<I", len(witness)))
        bb = np.packbits(bitmap).tobytes()
        buf.write(struct.pack("<I", len(bb)))
        buf.write(bb)
        wb = np.packbits(np.array(witness, dtype=np.uint8)).tobytes()
        buf.write(struct.pack("<I", len(wb)))
        buf.write(wb)
        vb = zlib.compress(changed_values.tobytes(), level=9)
        buf.write(struct.pack("<I", len(vb)))
        buf.write(struct.pack("<I", len(changed_values)))
        buf.write(vb)
        original_size = n + len(changed_values) * 8
        return buf.getvalue(), buf.tell() * 8 / original_size

    def _decompress_frame_differences(self, compressed_data: bytes, frame_shape, k_exact: Optional[float] = None):
        """ivc:969-1027.  `k_exact` (not in the reference) overrides the float32 k of the payload -- the reference
        decodes with the rounded k (ivc:938/986), which can break the round trip (SURVEY.md hard part 3i)."""
        buf = io.BytesIO(compressed_data)
        p = struct.unpack("<f", buf.read(4))[0]
        n = struct.unpack("<I", buf.read(4))[0]
        k = struct.unpack("<f", buf.read(4))[0]
        bitmap_length = struct.unpack("<I", buf.read(4))[0]
        witness_length = struct.unpack("<I", buf.read(4))[0]
        bsz = struct.unpack("<I", buf.read(4))[0]
        bloom_bitmap = np.unpackbits(np.frombuffer(buf.read(bsz), dtype=np.uint8))[:bitmap_length]
        wsz = struct.unpack("<I", buf.read(4))[0]
        witness = np.unpackbits(np.frombuffer(buf.read(wsz), dtype=np.uint8))[:witness_length].tolist()
        vsz = struct.unpack("<I", buf.read(4))[0]
        vcount = struct.unpack("<I", buf.read(4))[0]
        changed = np.frombuffer(zlib.decompress(buf.read(vsz)), dtype=np.uint8)[:vcount]
        if witness_length > 0:
            flat = self.bloom_compressor.decompress(bloom_bitmap, witness, n, k if k_exact is None else k_exact)
        else:
            flat = bloom_bitmap
        if len(frame_shape) == 3 and frame_shape[2] > 1:
            binary_diff = flat.reshape((frame_shape[0], frame_shape[1]))
        else:
            binary_diff = flat.reshape(frame_shape)
        return binary_diff, changed

    def compress_frame(self, frame, is_keyframe: bool = True):                    # ivc:1029-1104
        if not is_keyframe:
            raise ValueError("Non-keyframe compression should be handled by compress_video")
        body = FixedVideoCompressor(verbose=False).compress_frame(frame)
        data = struct.pack("<B", 1) + body                                         # ivc:1053: type tag 1 = keyframe
        meta = {"type": "keyframe", "shape": frame.shape, "original_size": frame.nbytes, "compressed_size": len(data),
                "compression_ratio": len(data) / frame.nbytes, "has_yuv_info": hasattr(frame, "yuv_info")}
        return data, meta

    def decompress_frame(self, compressed_data: bytes):                            # ivc:1106-1234
        if compressed_data[0] != 1:
            raise ValueError(f"Unknown frame type: {compressed_data[0]}")
        frame = FixedVideoCompressor(verbose=False).decompress_frame(compressed_data[1:])
        if hasattr(frame, "yuv_info") and not self.use_direct_yuv:                 # ivc:1163
            return frame.data
        return frame


_INTER_TAG_V1 = b"\xff\xff\xff\xffRBF1"   # round-1 layout: raw-passthrough masks stored as plain np.packbits bytes
_INTER_TAG = b"\xff\xff\xff\xffRBF2"      # current: raw-passthrough masks zlib-compressed (a static scene costs ~1 KB, not n/8 B)
_INTER_TAG_V3 = b"\xff\xff\xff\xffRBF3"   # value_coding "adaptive": RBF2 plus a vmode byte after the raw flag (0 values, 1 residuals)
_INTER_TAG_V4 = b"\xff\xff\xff\xffRBF4"   # value_coding "motion": RBF3 whose vmode may be 2, followed by <I length + zlib(motion field)
# none can be a FixedVideoCompressor payload (height 0xFFFFFFFF).  NOTE: inter payloads exist only in this implementation --
# the reference's decoder knows keyframes only (ivc:1124); files written with keyframe_interval=1 are interchangeable.
_INTER_TAGS = (_INTER_TAG, _INTER_TAG_V1, _INTER_TAG_V3, _INTER_TAG_V4)


class _InterPayload:
    """The fields of one inter-frame payload (ImprovedVideoCompressor._parse_inter); the byte fields are views of the payload.
    vmode 1: the value stream holds residuals (curr - prev) mod 2^(8 isz) per sample instead of the current samples; vmode 2: residuals
    against the motion-compensated previous frame, whose block vectors `fz` holds (zlib)."""
    __slots__ = ("v1", "h", "w", "isz", "ch", "raw", "vmode", "k", "l", "wlen", "ones", "mask_bytes", "witness_bytes", "vcount",
                 "vz", "fz")


class _InterJob:
    """An inter frame on its way through decompress_video: the parsed payload (or its parse error) and its inflates."""
    __slots__ = ("p", "err", "values", "mask", "field", "values_arr", "mask_arr", "field_arr", "l", "wlen", "vlen", "vsize")

    def __init__(self):
        self.p = self.err = self.values = self.mask = self.field = self.values_arr = self.mask_arr = self.field_arr = None
        self.vlen = None                                     # bytes of the value stream inflated on the GPU (_inflate_group)
        self.l = self.wlen = self.vsize = 0


def _is_inter(payload) -> bool:
    """Whether a payload is an inter frame (its first 8 bytes are an inter tag) rather than a keyframe."""
    return bytes(payload[:len(_INTER_TAG)]) in _INTER_TAGS


class _Jobs:
    """The decode jobs of a file's payloads (ImprovedVideoCompressor._start_inter / _start_key), started in file order from
    payload(i), for payloads before `stop` only.  take(i) hands job i over, starting it and the `ahead` payloads after it first if
    they have not been, and forgets it, so a decode holds only the payloads of the jobs it is working on and of those started ahead."""

    def __init__(self, comp: "ImprovedVideoCompressor", payload, inter: List[bool], pool, stop: int, ahead: int = 0):
        self._comp, self._payload, self._inter, self._pool, self._stop, self._ahead = comp, payload, inter, pool, stop, ahead
        self._jobs: Dict[int, object] = {}
        self._next = 0

    def start(self, upto: int, first: int = 0) -> None:
        """Starts the jobs of payloads [max(first, next), upto) (`first`: where the decode begins; earlier payloads are never read)."""
        self._next = max(self._next, first)
        for i in range(self._next, min(upto, self._stop)):
            c = self._payload(i)
            self._jobs[i] = self._comp._start_inter(c, self._pool) if self._inter[i] else self._comp._start_key(c, self._pool)
            self._next = i + 1

    def take(self, i: int):
        self.start(i + 1 + self._ahead, i)
        return self._jobs.pop(i)


class _DeviceOut:
    """A caller's device buffer, any object with __cuda_array_interface__, that file frames start .. stop-1 are written to with
    FrameStream.copy_frames.  The shape must be (stop - start, H, W) for one channel or (stop - start, H, W, C) for more, the dtype
    uint8 or uint16, the layout C-contiguous.  The interface's stream (v3) is waited for before each copy; an interface without
    one (v2, as torch exports) is ordered after the legacy default stream, where torch's default stream runs."""

    def __init__(self, out, start: int, stop: int):
        cai = getattr(out, "__cuda_array_interface__", None)
        if not isinstance(cai, dict):
            raise ValueError("out must be device memory with __cuda_array_interface__")
        shape, dtype = tuple(int(x) for x in cai["shape"]), np.dtype(cai["typestr"])
        if len(shape) not in (3, 4) or shape[0] != stop - start or (len(shape) == 4 and shape[3] < 2):
            raise ValueError(f"out has shape {shape}, not ({stop - start}, H, W) or ({stop - start}, H, W, C) with C > 1")
        if dtype not in (np.dtype(np.uint8), np.dtype(np.uint16)):
            raise ValueError(f"out has dtype {dtype}; frames are uint8 or uint16")
        strides = cai.get("strides")                         # None: C-contiguous
        if strides is not None and any(n > 1 and s != dtype.itemsize * math.prod(shape[d + 1:])
                                       for d, (n, s) in enumerate(zip(shape, strides))):
            raise ValueError("out must be C-contiguous")
        ptr, readonly = cai["data"]
        if readonly:
            raise ValueError("out is read-only")
        self.ptr, self.start, self.stop, self.dtype = int(ptr), start, stop, dtype
        self.frame_shape = shape[1:] if len(shape) == 4 else shape[1:3]
        self.frame_bytes = math.prod(self.frame_shape) * dtype.itemsize
        stream = cai.get("stream", 1) if int(cai.get("version", 2)) >= 3 else 1
        self.stream = 0 if stream is None else int(stream)

    def check(self, headers: Dict[int, Optional[tuple]]) -> None:
        """Raises ValueError when a frame's header -- (h, w, sample bytes, channels or None when its payload does not say) -- does not
        match out.  A frame without a readable header (None) raises its own error when the decode reaches it."""
        h, w = self.frame_shape[:2]
        ch = self.frame_shape[2] if len(self.frame_shape) == 3 else 1
        for i, hdr in headers.items():
            if hdr is not None and (hdr[:3] != (h, w, self.dtype.itemsize) or hdr[3] not in (None, ch)):
                raise ValueError(f"frame {i} is {hdr[0]} x {hdr[1]} x {hdr[3] or '?'} of {hdr[2]}-byte samples; out holds "
                                 f"{self.frame_shape} of {self.dtype}")

    def frame(self, data: np.ndarray, i: int) -> np.ndarray:
        if data.shape != self.frame_shape or data.dtype != self.dtype:
            raise ValueError(f"frame {i} is {data.shape} {data.dtype}; out holds {self.frame_shape} {self.dtype}")
        return data

    def put(self, st: FrameStream, slot: int, count: int, index: int) -> None:
        """Stream slots slot .. slot+count-1 to file frames index .. index+count-1 of out."""
        st.copy_frames(slot, count, self.ptr + (index - self.start) * self.frame_bytes, (self.stop - index) * self.frame_bytes,
                       self.stream)


class ImprovedVideoCompressor:
    """ivc.ImprovedVideoCompressor (ivc:309-523) with the GOP loop wired in.

    Frame i is a keyframe when i % keyframe_interval == 0 (zlib codec, byte-identical to the reference's
    payload); otherwise it is coded against the ORIGINAL previous frame: K1 mask -> Bloom + witness coder ->
    changed pixel values (zlib).  `inter_frame_mode`:
      "lossless"  (default) mask = any byte of the pixel differs, so reconstruction is always exact;
      "reference" mask = |dY| > inter_frame_threshold exactly as _calculate_frame_diff (ivc:788-808); a frame whose
                  unflagged pixels changed (chroma-only or sub-threshold changes) falls back to a keyframe.
    The entropy stage (zlib level 9, ivc:956 / fvc:31) stays on the CPU but runs in a thread pool (`num_threads`; zlib
    releases the GIL), and a group of `batch_size` inter frames costs ONE encode call and ONE batched device->host copy.
    `entropy_coder`:
      "zlib"  (default) zlib level 9 on the CPU: keyframe_interval=1 writes exactly the reference's bytes;
      "gpu"   every zlib stream of the payloads (keyframe blobs, changed values, raw-passthrough masks) is coded on the GPU
              (deflate.py): other compressed bytes, the same decoded data, read by the unchanged decoders.
    `value_coding`, what an inter frame's value stream holds:
      "plain"     (default) the current frame's samples at the changed pixels ('RBF2' payloads);
      "adaptive"  per inter frame, whichever zlib stream is shorter: those samples, or the residuals (curr - prev) mod 2^bits per
                  sample; a tie goes to the samples ('RBF3' payloads, whose vmode byte says which).  The decoder adds residuals to
                  the previous frame, which equals the encoder's original previous frame in both inter_frame_modes.
      "motion"    per inter frame, the cheapest of those two and the residuals against the motion-compensated previous frame: one
                  (dx, dy) in [-16, 16]^2 per 16 x 16 block, found by a full SAD search on the GPU, predicts each pixel from
                  prev(clamp(y + dy), clamp(x + dx)).  That option costs its stream plus 4 + the zlib'd field; the strict minimum wins and a
                  tie goes to the lower vmode ('RBF4' payloads: 'RBF3' plus the field when vmode is 2).
    """

    def __init__(self, noise_tolerance: float = 10.0, keyframe_interval: int = 30, min_diff_threshold: float = 3.0,
                 max_diff_threshold: float = 30.0, bloom_threshold_modifier: float = 1.0, batch_size: int = 30,
                 num_threads: int = None, use_direct_yuv: bool = False, verbose: bool = False):
        self.noise_tolerance = noise_tolerance
        self.keyframe_interval = keyframe_interval
        self.min_diff_threshold = min_diff_threshold
        self.max_diff_threshold = max_diff_threshold
        self.bloom_threshold_modifier = bloom_threshold_modifier
        self.batch_size = batch_size
        self.num_threads = max(1, min(32, (os.cpu_count() or 2))) if num_threads is None else max(1, int(num_threads))
        self.use_direct_yuv = use_direct_yuv
        self.verbose = verbose
        self.compressor = FixedVideoCompressor(verbose=verbose)                    # ivc:356
        self.inter_frame_mode = "lossless"
        self.inter_frame_threshold = 0.0
        self.entropy_coder = "zlib"
        self.value_coding = "plain"
        _cabi.ctx()                                                                 # fail now if there is no H100

    # ------------------------------------------------------------------ encode
    @staticmethod
    def _raw_mask_bits(shape, mask_row) -> bytes:
        """Passthrough branch (ivc:215-225): the mask itself in np.packbits order."""
        n = shape[0] * shape[1]
        return np.packbits(np.unpackbits(mask_row, bitorder="little")[:n]).tobytes()

    @staticmethod
    def _choose(streams: List[bytes], fz: Optional[bytes]):
        """-> (value stream, vmode, zlib'd field or None) from the zlib'd value streams of kinds 0 (values), 1 (residuals) and, for
        value_coding "motion", 2 (motion residuals, which cost their length + 4 + len(fz)).  The strict minimum wins and a tie goes to
        the lower vmode; vmode is None (an 'RBF2' payload) for value_coding "plain", whose one stream is kind 0."""
        if len(streams) == 1:
            return streams[0], None, None
        costs = [len(z) + (4 + len(fz) if kind == 2 else 0) for kind, z in enumerate(streams)]
        vmode = costs.index(min(costs))
        return streams[vmode], vmode, fz if vmode == 2 else None

    @staticmethod
    def _inter_payload(shape, itemsize, ch, r, bm_row, wt_row, rz, streams, fz) -> bytes:
        """One inter-frame payload from the futures of its zlib'd raw mask (raw pairs only), value streams (one per value kind) and
        motion field (value_coding "motion" only).  Runs as a pool job submitted after those futures."""
        vz, vmode, fz = ImprovedVideoCompressor._choose([s.result() for s in streams], None if fz is None else fz.result())
        return ImprovedVideoCompressor._inter_layout(shape, itemsize, ch, r, bm_row, wt_row, None if rz is None else rz.result(), vz,
                                                     r.ones * ch, vmode, fz, len(streams) == 3)

    @staticmethod
    def _inter_layout(shape, itemsize, ch, r, bm_row, wt_row, rz, vz, vcount, vmode=None, fz=None, v4=False) -> bytes:
        """The inter-frame byte layout around the compressed raw mask `rz` (raw pairs only) and changed values `vz`.  vmode None
        writes 'RBF2'; 0 (values) or 1 (residuals) writes 'RBF3', which carries it in one byte after the raw flag.  v4 writes 'RBF4',
        byte for byte the 'RBF3' layout, where vmode 2 (motion residuals) is followed by <I len(fz) and fz, the zlib'd motion field."""
        if vmode == 2 and (not v4 or fz is None):
            raise ValueError("vmode 2 is an 'RBF4' payload with a motion field")
        tag = _INTER_TAG if vmode is None else (_INTER_TAG_V4 if v4 else _INTER_TAG_V3)
        hdr = tag + struct.pack("<IIIBB", shape[0], shape[1], itemsize, ch, 1 if r.raw else 0)
        if vmode is not None:
            hdr += struct.pack("<B", vmode)
        if vmode == 2:
            hdr += struct.pack("<I", len(fz)) + fz
        body = struct.pack("<dIIQ", r.k, r.l, r.wlen, r.ones)
        if r.raw:
            body += struct.pack("<I", len(rz)) + rz + struct.pack("<I", 0)
        else:
            nb, nw = (r.l + 7) // 8, (r.wlen + 7) // 8
            body += struct.pack("<I", nb) + bm_row[:nb].tobytes() + struct.pack("<I", nw) + wt_row[:nw].tobytes()
        body += struct.pack("<II", len(vz), vcount) + vz
        return hdr + body

    @staticmethod
    def _parse_inter(payload: bytes) -> "_InterPayload":
        """The fields of an inter-frame payload (the inverse of _inter_layout; also reads round 1's 'RBF1' tag, whose raw masks are
        plain np.packbits bytes).  Nothing is decompressed: `mask_bytes` is the stored raw mask or bitmap, `vz` the value stream."""
        p = _InterPayload()
        tag = bytes(payload[:len(_INTER_TAG)])
        p.v1 = tag == _INTER_TAG_V1
        mv = memoryview(payload)
        pos = len(_INTER_TAG)
        p.h, p.w, p.isz, p.ch, p.raw = struct.unpack_from("<IIIBB", payload, pos)
        pos += struct.calcsize("<IIIBB")
        p.vmode = 0
        p.fz = None
        if tag in (_INTER_TAG_V3, _INTER_TAG_V4):
            (p.vmode,) = struct.unpack_from("<B", payload, pos)
            pos += 1
            if tag == _INTER_TAG_V3 and p.vmode not in (0, 1):
                raise ValueError(f"corrupt inter frame: value coding {p.vmode} is neither 0 (values) nor 1 (residuals)")
            if p.vmode not in (0, 1, 2):
                raise ValueError(f"corrupt inter frame: value coding {p.vmode} is not 0 (values), 1 (residuals) or 2 (motion residuals)")
            if p.vmode == 2:
                (fl,) = struct.unpack_from("<I", payload, pos); pos += 4
                if pos + fl > len(payload):
                    raise ValueError(f"corrupt inter frame: a motion field of {fl} bytes runs past the payload")
                p.fz = mv[pos:pos + fl]; pos += fl
        p.k, p.l, p.wlen, p.ones = struct.unpack_from("<dIIQ", payload, pos)
        pos += struct.calcsize("<dIIQ")
        (bl,) = struct.unpack_from("<I", payload, pos); pos += 4
        p.mask_bytes = mv[pos:pos + bl]; pos += bl
        (wl,) = struct.unpack_from("<I", payload, pos); pos += 4
        p.witness_bytes = mv[pos:pos + wl]; pos += wl
        vlen, p.vcount = struct.unpack_from("<II", payload, pos); pos += 8
        p.vz = mv[pos:pos + vlen]
        return p

    def _encode_inter_frames(self, datas: List[np.ndarray], inter: List[int], pool) -> Dict[int, object]:
        """Futures of the inter-frame payloads for frame indices `inter` (each coded against frame i-1); None = keyframe instead."""
        out: Dict[int, object] = {}
        if not inter:
            return out
        shape, dtype = datas[0].shape, datas[0].dtype
        ch = shape[2] if len(shape) == 3 else 1
        group = max(2, int(self.batch_size))
        kinds = {"plain": 1, "adaptive": 2, "motion": 3}[self.value_coding]      # value kinds 0 .. kinds-1 (_value_streams)
        st = FrameStream(shape[0], shape[1], ch, dtype, max_frames=2 * group, max_pairs=group,
                         mask_mode=1 if self.inter_frame_mode == "lossless" else 0)
        try:
            for g0 in range(0, len(inter), group):
                idxs = inter[g0:g0 + group]
                need = sorted(set(idxs) | {i - 1 for i in idxs})
                slot = {f: s for s, f in enumerate(need)}
                st.upload(np.stack([datas[f] for f in need]))
                res = st.encode([slot[i - 1] for i in idxs], [slot[i] for i in idxs], float(self.inter_frame_threshold))
                any_raw = any(r.raw for r in res)
                bms, wts, masks = st.fetch_batch(0, len(idxs), want_masks=any_raw)   # one D2H per kind, one sync per group
                # the pairs coded as inter frames; the others are not exactly representable: keyframes instead
                keep = [j for j, r in enumerate(res) if not (r.resid and self.inter_frame_mode != "lossless")]
                streams, fields = [], None
                for kind in range(kinds):
                    if kind == 2:
                        fields = st.motion_search()
                    streams.append(self._value_streams(st, kind, keep, pool))
                raw = [j for j in keep if res[j].raw]
                rzs = dict(zip(raw, self._zlib(pool, [masks[j] for j in raw], partial(self._raw_mask_bits, shape))))
                fzs = self._zlib(pool, [fields[j] for j in keep]) if fields is not None else None
                out.update(dict.fromkeys(idxs))
                for k, j in enumerate(keep):
                    out[idxs[j]] = pool.submit(self._inter_payload, shape, dtype.itemsize, ch, res[j], bms[j], wts[j], rzs.get(j),
                                               [s[k] for s in streams], None if fzs is None else fzs[k])
        finally:
            st.close()
        return out

    def _value_streams(self, st: FrameStream, kind: int, keep: List[int], pool) -> List[Future]:
        """Futures of the zlib'd value streams of the encoded pairs `keep`, gathered as value kind `kind`: 0 the current samples,
        1 their residuals against the previous frame (value_mode 1), 2 the residuals against the motion-compensated previous frame
        of the last motion_search (motion_values 1)."""
        option = (None, "value_mode", "motion_values")[kind]
        if option is None:
            return self._zlib(pool, keep, st=st)
        st.set_option(option, 1)
        try:
            return self._zlib(pool, keep, st=st)
        finally:
            st.set_option(option, 0)

    def _zlib(self, pool, items, make=lambda buf: buf, st: Optional[FrameStream] = None) -> List[Future]:
        """Futures of zlib streams, one per item: of the buffer make(item), or with `st`, of the changed values of its encoded pair
        `item` (all of its pairs are gathered).  This is the one step where the entropy coders differ.  "zlib": the host gathers the
        values, and each make(item) with its level-9 zlib.compress runs as a job of `pool`.  "gpu": one device batch now, the values
        deflated where zlib_changed gathers them."""
        if self.entropy_coder == "gpu":
            if st is not None:
                zs = st.zlib_changed()
                zs = [zs[j] for j in items]
            else:
                zs = deflate.compress_many([make(x) for x in items])
            return [_done(z) for z in zs]
        if st is not None:
            vals = st.gather_changed()                     # N1: changed values of every pair, one launch, one copy
            items = [vals[j] for j in items]
        return [pool.submit(lambda x: zlib.compress(make(x), 9), x) for x in items]

    def _keyframe_job(self, frame, pool):
        """Callable returning the keyframe payload of `frame`, whose blobs _zlib codes."""
        zs = self._zlib(pool, keyframe_raws(frame))
        return lambda: assemble_keyframe(frame, [z.result() for z in zs])

    def compress_video(self, frames: List[np.ndarray], output_path: str = None, input_color_space: str = "BGR") -> Dict:
        if self.entropy_coder not in ("zlib", "gpu"):
            raise ValueError(f"entropy_coder must be 'zlib' or 'gpu', not {self.entropy_coder!r}")
        if self.value_coding not in ("plain", "adaptive", "motion"):
            raise ValueError(f"value_coding must be 'plain', 'adaptive' or 'motion', not {self.value_coding!r}")
        if not frames:
            raise ValueError("No frames provided for compression")                 # ivc:372-373
        start_time = time.time()
        if input_color_space.upper() == "YUV":                                      # ivc:378-384 (wraps in place)
            self.use_direct_yuv = True
            for i in range(len(frames)):
                if not hasattr(frames[i], "yuv_info"):
                    frames[i] = self.compressor.add_yuv_info_to_frame(frames[i])
        original_size = sum(frame.nbytes for frame in frames)
        datas = [np.ascontiguousarray(_frame_data(f)) for f in frames]
        ki = max(1, int(self.keyframe_interval))
        uniform = all(d.shape == datas[0].shape and d.dtype == datas[0].dtype for d in datas) and \
            datas[0].dtype in (np.uint8, np.uint16) and (datas[0].ndim == 2 or datas[0].shape[2] == 3)
        inter = [i for i in range(len(frames)) if i % ki != 0] if uniform else []
        from concurrent.futures import ThreadPoolExecutor
        compressed_frames: List[bytes] = []
        keyframes = 0
        with ThreadPoolExecutor(self.num_threads) as pool:
            # keyframes (zlib level 9 of whole frames, fvc:31) start in the pool first; the GPU encodes the groups meanwhile
            inter_set = set(inter)
            key_jobs = {i: self._keyframe_job(frames[i], pool) for i in range(len(frames)) if i not in inter_set}
            payloads = self._encode_inter_frames(datas, inter, pool)
            for i, f in enumerate(frames):
                fut = payloads.get(i)
                if fut is None:
                    kj = key_jobs.get(i)
                    pl = (kj if kj is not None else self._keyframe_job(f, pool))()
                    keyframes += 1
                else:
                    pl = fut.result()
                compressed_frames.append(pl)
        if output_path:                                                             # ivc:393-406
            os.makedirs(os.path.dirname(os.path.abspath(output_path)), exist_ok=True)
            with open(output_path, "wb") as fh:
                fh.write(b"BFVC")
                fh.write(struct.pack("<I", len(frames)))
                for c in compressed_frames:
                    fh.write(struct.pack("<I", len(c)))
                    fh.write(c)
        if output_path and os.path.exists(output_path):
            compressed_size = os.path.getsize(output_path)
        else:
            compressed_size = sum(len(c) for c in compressed_frames) + 4 + 4 + 4 * len(compressed_frames)   # ivc:413-415
        self._last_compressed_frames = compressed_frames
        ratio = compressed_size / original_size
        dt = time.time() - start_time
        results = {"frame_count": len(frames), "original_size": original_size, "compressed_size": compressed_size,
                   "compression_ratio": ratio, "space_savings": 1.0 - ratio, "compression_time": dt,
                   "frames_per_second": len(frames) / dt if dt > 0 else float("inf"), "keyframes": keyframes,
                   "keyframe_ratio": keyframes / len(frames), "output_path": output_path,
                   "color_space": input_color_space, "overall_ratio": ratio}       # ivc:424-437
        if self.verbose:
            print(f"Compression Ratio: {ratio:.4f}  keyframes: {keyframes}/{len(frames)}")
        return results

    # ------------------------------------------------------------------ decode
    def _start_inter(self, payload: bytes, pool) -> "_InterJob":
        """Parse an inter payload and start its inflates (changed values, zlib'd raw mask) in `pool`.  A parse error is kept and
        raised when decoding reaches this frame, so the first bad frame of the file decides the exception."""
        job = _InterJob()
        try:
            job.p = self._parse_inter(payload)
        except Exception as e:                               # re-raised in file order by _check_inter
            job.err = e
            return job
        if bytes(job.p.vz[:2]) != deflate._DEVICE_HEADER:  # the device coder's streams are inflated per group on the GPU
            job.values = pool.submit(zlib.decompress, job.p.vz)
        if job.p.vmode == 2:
            job.field = pool.submit(zlib.decompress, job.p.fz)
        if job.p.raw and not job.p.v1:
            job.mask = pool.submit(zlib.decompress, job.p.mask_bytes)
        return job

    @staticmethod
    def _check_inter(job: "_InterJob", pdata: np.ndarray) -> None:
        """The checks of one inter frame that need no GPU, in the order a frame-by-frame decode makes them; keeps the inflated
        values and the effective mask fields on `job`."""
        if job.err is not None:
            raise job.err
        p = job.p
        dtype = np.dtype(np.uint8 if p.isz == 1 else np.uint16)
        if job.vlen is None:                                 # (a stream left for the GPU that no group inflated: here)
            raw = job.values.result() if job.values is not None else zlib.decompress(p.vz)
            job.values_arr = np.frombuffer(raw, dtype=dtype)[:p.vcount]
            job.vsize = job.values_arr.size
        else:                                                # on the device: the same count, and numpy's error for a ragged length
            if job.vlen % dtype.itemsize:
                np.frombuffer(bytes(job.vlen % dtype.itemsize), dtype=dtype)
            job.vsize = min(job.vlen // dtype.itemsize, p.vcount)
        exp_shape = (p.h, p.w, p.ch) if p.ch > 1 else (p.h, p.w)
        if pdata.shape != exp_shape or pdata.dtype != dtype:
            raise ValueError(f"inter frame {exp_shape}/{dtype} does not match the previous frame {pdata.shape}/{pdata.dtype}")
        if job.vsize != p.ones * p.ch:
            raise ValueError(f"corrupt inter frame: {job.vsize} changed values for {p.ones} changed pixels x {p.ch} channels")
        if p.vmode == 2:
            nfield = 2 * ((p.h + 15) // 16) * ((p.w + 15) // 16)
            job.field_arr = np.frombuffer(job.field.result(), dtype=np.int8)
            if job.field_arr.size != nfield:
                raise ValueError(f"corrupt inter frame: a motion field of {job.field_arr.size} bytes for {nfield // 2} blocks")
            if job.field_arr.size and np.abs(job.field_arr.astype(np.int16)).max() > 16:
                raise ValueError("corrupt inter frame: a motion vector component outside [-16, 16]")
        if p.raw:
            job.mask_arr = np.frombuffer(p.mask_bytes if p.v1 else job.mask.result(), dtype=np.uint8)
            if job.mask_arr.size < (p.h * p.w + 7) // 8:
                raise ValueError(f"corrupt inter frame: the raw mask holds {8 * job.mask_arr.size} of {p.h * p.w} bits")
            return
        job.l = min(p.l, 8 * len(p.mask_bytes))              # the bits that are there, as np.unpackbits(..)[:l] keeps them
        job.wlen = min(p.wlen, 8 * len(p.witness_bytes))
        if job.l == 0 or job.wlen == 0:                      # the reference would take the l-bit bitmap as the n-bit mask (ivc:282-284)
            raise ValueError(f"corrupt inter frame: a coded mask with {job.l} Bloom bits and {job.wlen} witness bits")
        if not p.k >= 0.0:
            raise _cabi.RbfError(f"corrupt inter frame: k = {p.k}")

    @staticmethod
    def _decode_group(st: FrameStream, base: int, group: List["_InterJob"], skip: int = 0, out: "_DeviceOut" = None,
                      index: int = 0) -> Optional[np.ndarray]:
        """Frames base+1 .. base+len(group) of `st` (slots modulo st.max_frames) from frame `base` and the group's payloads: one
        decode_masks, one apply_chain (value modes and motion fields included) and one download_batch of all but the first `skip`
        frames, which stay on the device (None when that is all of them).  With `out`, those frames go to its device buffer as file
        frames index+skip .. instead, through one copy_frames, and None is returned.  Raises the first bad frame's error."""
        m, n = len(group), st.npix
        raws = [bool(j.p.raw) for j in group]
        nbs = [(n + 7) // 8 if r else (j.l + 7) // 8 for j, r in zip(group, raws)]
        nws = [0 if r else (j.wlen + 7) // 8 for j, r in zip(group, raws)]
        bms = np.zeros((m, max(16, (max(nbs) + 15) // 16 * 16)), dtype=np.uint8)
        wts = np.zeros((m, 0 if not any(nws) else max(16, (max(nws) + 15) // 16 * 16)), dtype=np.uint8)
        for i, j in enumerate(group):
            if raws[i]:
                bms[i, :nbs[i]] = j.mask_arr[:nbs[i]]
            else:
                bms[i, :nbs[i]] = np.frombuffer(j.p.mask_bytes, dtype=np.uint8, count=nbs[i])
                wts[i, :nws[i]] = np.frombuffer(j.p.witness_bytes, dtype=np.uint8, count=nws[i])
        consumed, ones = st.decode_masks(bms, wts, [0 if r else j.l for j, r in zip(group, raws)],
                                         [0 if r else j.wlen for j, r in zip(group, raws)], [j.p.k for j in group], raws)
        for i, j in enumerate(group):
            if not raws[i] and consumed[i] > j.wlen:         # the reference's witness[witness_idx] raises here
                raise IndexError("list index out of range")
            if ones[i] != j.p.ones:                          # the reference would silently return the base frame (ivc:882)
                raise ValueError(f"corrupt inter frame: the decoded mask selects {int(ones[i])} pixels, the payload announces {j.p.ones}")
        if group[0].vlen is not None:                        # the group's values are on the device (_inflate_group)
            vals = {"inflated": [j.vsize * j.p.isz for j in group]}
        else:
            vals = {"values": [j.values_arr for j in group]}
        applied = st.apply_chain(base, **vals, modes=[j.p.vmode for j in group], motion=[j.field_arr for j in group])
        if not np.array_equal(applied, ones):
            raise ValueError(f"corrupt inter frame: {applied.tolist()} pixels applied, {ones.tolist()} expected")
        if skip >= m:
            return None
        if out is not None:
            out.put(st, (base + 1 + skip) % st.max_frames, m - skip, index + skip)
            return None
        return st.download_batch((base + 1 + skip) % st.max_frames, m - skip)

    @staticmethod
    def _inflate_group(st: FrameStream, jobs: List["_InterJob"], pool) -> None:
        """The value streams of a group's payloads, when all are the device coder's, inflated on the GPU into `st` (job.vlen).  If
        any is not, or the device declines one, every stream of the group is inflated on the host as before."""
        parsed = [j for j in jobs if j.p is not None]
        dev = [j for j in parsed if j.values is None]
        if not dev:
            return
        if len(dev) == len(parsed):
            lens, ok = st.inflate_values([j.p.vz for j in dev], [j.p.vcount * j.p.isz for j in dev])
            if ok.all():
                for j, n in zip(dev, lens):
                    j.vlen = int(n)
                return
        for j in dev:
            j.values = pool.submit(zlib.decompress, j.p.vz)

    def _decode_span(self, inter: List[bool], jobs: "_Jobs", k: int, start: int, stop: int, streams: Dict[tuple, FrameStream],
                     pool, out: "_DeviceOut" = None):
        """Decodes payloads [k, stop) and yields the frames [start, stop) (k <= start: the last keyframe at or before start, or 0),
        one list per keyframe and per group; with `out`, writes them to its device buffer instead and yields their count.
        inter[i]: payload i is an inter payload.  Each run of inter payloads is rebuilt from the keyframe before it in groups of
        batch_size counted from the run's first frame, as in a whole-file decode.  The run's base frame is uploaded once; each group
        chains from the previous group's last frame, which stays on the device, and frames before start are never downloaded.  The
        first bad frame of [k, stop) raises, after the frames before it have been yielded."""
        group_size = max(1, int(self.batch_size))
        prev = st = pdata = None
        base, i = 0, k
        while i < stop:
            if not inter[i]:                                 # a keyframe: built on the host; a run after it starts from it
                prev, st, base = jobs.take(i).result(), None, 0
                pdata = np.ascontiguousarray(_frame_data(prev))
                if i >= start:
                    if out is None:
                        yield [prev]
                    else:                                    # through the slot the run after it would upload it to
                        st = self._run_stream(out.frame(pdata, i), group_size, streams)
                        out.put(st, 0, 1, i)
                        yield 1
                i += 1
                continue
            if prev is None:
                raise ValueError("inter frame without a preceding frame")
            end = i
            while end < stop and inter[end]:
                end += 1
            for g0 in range(i, end, group_size):
                run = [jobs.take(j) for j in range(g0, min(g0 + group_size, end))]
                group, err = [], None
                if any(j.p is not None and j.values is None for j in run):
                    if st is None:
                        st = self._run_stream(pdata, group_size, streams)
                    self._inflate_group(st, run, pool)
                for job in run:
                    try:
                        self._check_inter(job, pdata)
                    except Exception as e:                   # the frames before it are decoded first: their errors come first
                        err = e
                        break
                    group.append(job)
                if group:
                    if st is None:
                        st = self._run_stream(pdata, group_size, streams)
                    skip = max(0, start - g0)
                    dec = self._decode_group(st, base, group, skip, out, g0)
                    base = (base + len(group)) % st.max_frames
                    if skip < len(group):
                        yield len(group) - skip if out is not None else \
                            [YUVFrame(f) if hasattr(prev, "yuv_info") else f for f in dec]
                    dec = None                               # a reader holds one group of decoded frames, not two
                if err is not None:
                    raise err
            i = end

    @staticmethod
    def _run_stream(pdata: np.ndarray, group_size: int, streams: Dict[tuple, FrameStream]) -> FrameStream:
        """The device store a run decodes in (one per frame shape and dtype), with the run's base frame uploaded to slot 0."""
        ch = pdata.shape[2] if pdata.ndim == 3 else 1
        key = (pdata.shape, pdata.dtype.str)
        st = streams.get(key)
        if st is None:
            st = streams[key] = FrameStream(pdata.shape[0], pdata.shape[1], ch, pdata.dtype, max_frames=group_size + 1,
                                            max_pairs=group_size, k1_only=True)
        st.upload(pdata, first=0)
        return st

    def _start_key(self, payload: bytes, pool):
        """A keyframe's decode: its blobs inflated on the GPU in one batch when all are the device coder's (then built with
        build_frame when decoding reaches the frame), else decompress_frame in `pool`.  Anything the GPU route raises sends the
        frame to decompress_frame, which raises what it always did."""
        try:
            blobs = self.compressor.keyframe_blobs(payload)
        except Exception:
            blobs = None
        if not blobs or any(bytes(b[:2]) != deflate._DEVICE_HEADER for b, _ in blobs):
            return pool.submit(self.compressor.decompress_frame, payload)
        comp = self.compressor

        class _Job:
            @staticmethod
            def result():
                try:
                    raws = iter(deflate.decompress_many([b for b, _ in blobs], [n for _, n in blobs]))
                    return comp.build_frame(payload, lambda _blob: next(raws))
                except Exception:
                    return comp.decompress_frame(payload)
        return _Job()

    def decompress_video(self, input_path: str = None, output_path: Optional[str] = None,
                         compressed_frames: List[bytes] = None, metadata: Dict = None) -> List[np.ndarray]:
        """ivc:452-504.  Each run of inter frames is rebuilt on the GPU in groups of batch_size (_decode_span over the whole file;
        VideoReader runs the same driver over a span).  zlib streams of the GPU entropy coder (78 9C: keyframe blobs, changed values) are inflated on the GPU -- a group's value streams straight into
        the buffer its reconstruction reads; every other zlib stream (CPU zlib's 78 DA, raw masks, motion fields), and any stream
        the GPU declines, is inflated with zlib.decompress in a pool of num_threads."""
        if input_path and os.path.exists(input_path):                              # ivc:471-485
            with open(input_path, "rb") as fh:
                magic = fh.read(4)
                if magic != b"BFVC":
                    raise ValueError(f"Invalid file format: {magic}")
                count = struct.unpack("<I", fh.read(4))[0]
                compressed_frames = []
                for _ in range(count):
                    size = struct.unpack("<I", fh.read(4))[0]
                    compressed_frames.append(fh.read(size))
        if not compressed_frames:
            raise ValueError("No compressed frames provided")                       # ivc:487-488
        from concurrent.futures import ThreadPoolExecutor
        frames: list = []
        streams: Dict[tuple, FrameStream] = {}
        pool = ThreadPoolExecutor(self.num_threads)
        try:
            count = len(compressed_frames)
            inter = [_is_inter(c) for c in compressed_frames]
            jobs = _Jobs(self, compressed_frames.__getitem__, inter, pool, count)
            jobs.start(count)                                # every payload's inflates start up front
            for part in self._decode_span(inter, jobs, 0, 0, count, streams, pool):
                frames += part
        finally:
            pool.shutdown(wait=True, cancel_futures=True)
            for st in streams.values():
                st.close()
        if output_path:
            self.save_frames_as_video(frames, output_path)
        return frames

    def verify_lossless(self, original_frames, decompressed_frames) -> Dict:       # ivc:506-523
        return self.compressor.verify_lossless(original_frames, decompressed_frames)

    def save_frames_as_video(self, frames, output_path: str, fps: int = 30) -> str:   # ivc:525-581 (host glue, cv2)
        import cv2
        if not frames:
            raise ValueError("No frames provided")
        os.makedirs(os.path.dirname(os.path.abspath(output_path)), exist_ok=True)
        h, w = frames[0].shape[:2]
        color = len(frames[0].shape) > 2
        out = cv2.VideoWriter(output_path, cv2.VideoWriter_fourcc(*"mp4v"), fps, (w, h), isColor=color)
        if not out.isOpened():
            raise ValueError(f"Could not create video writer for {output_path}")
        for f in frames:
            d = _frame_data(f)
            if color and hasattr(f, "yuv_info") and self.use_direct_yuv:
                d = cv2.cvtColor(d, cv2.COLOR_YUV2BGR)
            elif not color:
                d = cv2.cvtColor(d, cv2.COLOR_GRAY2BGR)
            elif d.shape[2] == 3 and not hasattr(f, "yuv_info"):
                d = cv2.cvtColor(d, cv2.COLOR_RGB2BGR)
            out.write(d)
        out.release()
        return output_path


def _frame_header(payload, inter: bool) -> Optional[tuple]:
    """(h, w, sample bytes, channels) of a payload without decoding it; channels is None for a keyframe, whose layout does not
    carry it.  None when the layout cannot be read: the decode raises that payload's error."""
    try:
        if inter:
            p = ImprovedVideoCompressor._parse_inter(payload)
            return p.h, p.w, p.isz, p.ch
        return struct.unpack_from("<III", payload, 0) + (None,)
    except Exception:
        return None


class VideoReader:
    """Random access to a compressed video: any frame range decoded from the last keyframe at or before it.

        r = VideoReader(source, compressor=None)   # a BFVC path, or a sequence of payloads (decompress_video's compressed_frames)
        len(r); r.keyframes                        # frame count; indices of the keyframe payloads
        r.read(start, stop, out=None)              # == decompress_video(...)[start:stop]; with out=, into device memory
        r[i]; r[a:b]; for f in r: ...; with VideoReader(path) as r: ...

    `compressor` (default ImprovedVideoCompressor()) decodes, with its batch_size and num_threads.  Opening a file reads its
    length table and the first 8 bytes of every payload, which say whether it is a keyframe; a read of [start, stop) reads, parses
    and inflates payloads [k, stop) only, k the last keyframe at or before start, and raises what decompress_video raises for the
    first bad frame among them.  Frames before start are rebuilt on the device and never downloaded.  Iteration decodes one group
    at a time, reading the next group's payloads ahead.  close() releases the file and the device streams."""

    def __init__(self, source, compressor: Optional[ImprovedVideoCompressor] = None):
        self._comp = compressor if compressor is not None else ImprovedVideoCompressor()
        self._fh = self._src = None
        self._streams: Dict[tuple, FrameStream] = {}         # of read(): kept for the next read, released by close()
        self._live: List[Dict[tuple, FrameStream]] = []     # of iterators not yet finished
        if isinstance(source, (str, os.PathLike)):
            self._open(os.fspath(source))
        else:
            self._src = source
            self._inter = [_is_inter(source[i]) for i in range(len(source))]
        if not self._inter:
            self.close()
            raise ValueError("No compressed frames provided")
        self.keyframes = [i for i, x in enumerate(self._inter) if not x]

    def _open(self, path: str) -> None:
        """Reads the magic, the count and the length table, seeking from length prefix to length prefix, and each payload's
        first 8 bytes.  A payload cut short by the end of the file is read as short as it is there."""
        self._fh = open(path, "rb")
        magic = self._fh.read(4)
        if magic != b"BFVC":
            self.close()
            raise ValueError(f"Invalid file format: {magic}")
        try:
            count = struct.unpack("<I", self._fh.read(4))[0]
            self._spans, self._inter, pos = [], [], 8
            for _ in range(count):
                self._fh.seek(pos)
                size = struct.unpack("<I", self._fh.read(4))[0]
                self._inter.append(_is_inter(self._fh.read(min(size, len(_INTER_TAG)))))
                self._spans.append((pos + 4, size))
                pos += 4 + size
        except BaseException:
            self.close()
            raise

    def _payload(self, i: int):
        if self._src is not None:
            return self._src[i]
        if self._fh is None:
            raise ValueError("the reader is closed")
        off, size = self._spans[i]
        self._fh.seek(off)
        return self._fh.read(size)

    def __len__(self) -> int:
        return len(self._inter)

    def _decode(self, k: int, start: int, stop: int, payload, streams: Dict[tuple, FrameStream], out: "_DeviceOut" = None,
                ahead: Optional[int] = None):
        """_decode_span over payloads [k, stop): all started at once (ahead None), or each group's while the one before is decoded."""
        from concurrent.futures import ThreadPoolExecutor
        pool = ThreadPoolExecutor(self._comp.num_threads)
        try:
            jobs = _Jobs(self._comp, payload, self._inter, pool, stop, ahead or 0)
            if ahead is None:
                jobs.start(stop, k)
            yield from self._comp._decode_span(self._inter, jobs, k, start, stop, streams, pool, out)
        finally:
            pool.shutdown(wait=True, cancel_futures=True)

    def read(self, start: int, stop: int, out=None):
        """decompress_video(...)[start:stop], decoded from the last keyframe at or before start.  With `out` -- an object with
        __cuda_array_interface__ of shape (stop - start, H, W) or (stop - start, H, W, C), the frames' dtype, C-contiguous, on the
        library's device -- the frames' samples are written there instead and `out` is returned: keyframes through an upload into a
        device slot, inter frames straight from the slots they are rebuilt in, one copy per group; YUV planes are not produced.  A
        mismatched `out` raises ValueError before anything is launched."""
        start, stop, n = operator.index(start), operator.index(stop), len(self)
        if not 0 <= start <= stop <= n:
            raise IndexError(f"frames [{start}, {stop}) outside [0, {n}]")
        dev = None if out is None else _DeviceOut(out, start, stop)
        if start == stop:
            return [] if out is None else out
        at = bisect.bisect_right(self.keyframes, start)
        k = self.keyframes[at - 1] if at else 0
        payloads = {i: self._payload(i) for i in range(k, stop)}
        if dev is not None:
            dev.check({i: _frame_header(payloads[i], self._inter[i]) for i in range(start, stop)})
        frames: list = []
        for part in self._decode(k, start, stop, payloads.__getitem__, self._streams, dev):
            if dev is None:
                frames += part
        return frames if dev is None else out

    def __getitem__(self, key):
        if isinstance(key, slice):
            a, b, step = key.indices(len(self))
            if step != 1:
                raise ValueError(f"slice step must be 1, not {step}")
            return self.read(a, max(a, b))
        i = operator.index(key)
        if i < 0:
            i += len(self)
        if not 0 <= i < len(self):
            raise IndexError(f"frame index {key} out of range for {len(self)} frames")
        return self.read(i, i + 1)[0]

    def __iter__(self):
        """Every frame in order, as decompress_video returns them; holds one group of decoded frames at a time."""
        streams: Dict[tuple, FrameStream] = {}
        self._live.append(streams)
        parts = self._decode(0, 0, len(self), self._payload, streams, ahead=max(1, int(self._comp.batch_size)))
        try:
            for part in parts:
                part.reverse()
                while part:
                    yield part.pop()
        finally:
            parts.close()
            for st in streams.values():
                st.close()
            self._live = [s for s in self._live if s is not streams]

    def close(self) -> None:
        for streams in [self._streams] + self._live:
            for st in streams.values():
                st.close()
            streams.clear()
        if self._fh is not None:
            self._fh.close()
            self._fh = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
