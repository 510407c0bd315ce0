"""
new_bloom_filter_repo_b200 -- H100-native (sm_90a) implementation of the rational-Bloom-filter
insert/query hot path of ross39/new_bloom_filter_repo, behind the reference's own Python API.

    from new_bloom_filter_repo_b200 import ImprovedVideoCompressor, RationalBloomFilter

Host code is Python calling hand-written CUDA through a C ABI (include/rbf_b200.h) with ctypes.
There is no CPU fallback: importing is cheap, but every entry point needs librbf_b200.so and an H100.
"""
from . import _cabi
from . import deflate
from ._cabi import RbfError
from .improved_video_compressor import (BloomFilterCompressor, ImprovedVideoCompressor, VideoFrameCompressor, VideoReader)
from .improved_video_compressor import RationalBloomFilter as IndexRationalBloomFilter
from .rational_bloom_filter import RationalBloomFilter, StandardBloomFilter
from .fixed_video_compressor import FixedVideoCompressor, YUVFrame
from .stream import FrameStream, PairResult

__all__ = ["ImprovedVideoCompressor", "VideoReader", "VideoFrameCompressor", "BloomFilterCompressor", "IndexRationalBloomFilter",
           "RationalBloomFilter", "StandardBloomFilter", "FixedVideoCompressor", "YUVFrame", "FrameStream",
           "PairResult", "RbfError", "deflate"]
