// rbf_kernels.cuh -- device-side job descriptors and launcher prototypes shared by
// rbf_kernels.cu (kernels) and rbf_api.cu (C ABI + host pipeline).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "rbf_hash.cuh"

namespace rbf {

// One Bloom filter (= one inter-frame mask, or one user filter).  Device-resident array.
// Internal bit order everywhere on the device is LSB-first in little-endian 32-bit words
// (bit j -> word j>>5, bit j&31); conversion to the reference's np.packbits order
// (MSB-first per byte, ivc:945,951) is a per-byte bit reversal done once on the way out.
struct FrameJob {
    uint32_t n;           // positions (H*W)
    uint32_t l;           // Bloom size in bits; 0 => raw passthrough (ivc:215-225), no work
    uint32_t floor_k;     // ivc:57
    uint32_t has_act;     // p_activation > 0
    uint64_t act_T;       // h < act_T  <=>  h/(2^64-1) < p_activation   (ivc:95-97)
    uint64_t seed1, seed2, seedA;   // ivc:62-63, ivc:94
    FastMod fm;           // m = l
    const uint32_t* mask; // n bits, natural packing, >= 16 B zero padding after the last word
    uint32_t* bits;       // l bits (ceil(l/32) words rounded up to 16 B), zeroed before insert
    uint32_t* pass;       // Bloom-test pass mask, century-padded: 4 words (128 bit) per 100 positions
    uint32_t* witness;    // witness bit stream (K3b output / K4b input), zeroed before K3b
    uint32_t* out_mask;   // decode output, natural packing, zeroed before K4b
    uint32_t wlen_in;     // decode: number of valid witness bits
    uint32_t neg_m;       // 2^32 - l, for the one-instruction remainder step of the query kernels
};

// One frame pair for the threshold kernel (ivc:788-808).
struct PairJob {
    const uint8_t* prev;
    const uint8_t* curr;
    uint32_t* mask;       // n bits natural packing
};

struct GatherJob {
    const uint32_t* mask;     // n bits, natural packing
    const uint8_t* frame;     // source (curr) frame
    const uint8_t* prev;      // residual gather: the pair's previous frame (values = curr - prev per sample); otherwise unused
    uint8_t* values;          // output (rank-ordered pixel values)
    uint32_t npix;
    uint32_t pix_bytes;
    uint32_t width;           // motion residual gather: frame width (the height is npix / width)
    const int8_t* field;      // motion residual gather: the pair's (dx, dy) per 16 x 16 block, raster order; otherwise unused
};

// Block motion (rbf_motion.cuh): 16 x 16 px blocks in raster order, one (dx, dy) int8 pair per block, |dx|, |dy| <= 16.
// pred(y, x) = prev(clamp(y + dy, 0, H - 1), clamp(x + dx, 0, W - 1)) with the vector of the block holding (y, x).
static constexpr int MV_BLOCK = 16;
static constexpr int MV_RANGE = 16;
__host__ __device__ __forceinline__ uint32_t mv_blocks_x(uint32_t W) { return (W + MV_BLOCK - 1u) / MV_BLOCK; }
__host__ __device__ __forceinline__ uint32_t mv_blocks(uint32_t H, uint32_t W) { return mv_blocks_x(W) * ((H + MV_BLOCK - 1u) / MV_BLOCK); }


// K4c (rbf_k4c_apply.cuh): a chain of decoded masks applied to one base frame, frames base+1 .. base+count
static constexpr int AP_THREADS = 128;
static constexpr uint32_t AP_TILE_WORDS = AP_THREADS;
static constexpr uint32_t AP_TILE_PX = 32u * AP_TILE_WORDS;     // 4096 px: 4 / 8 / 12 / 24 KB of shared memory at 1 / 2 / 3 / 6 B per pixel

struct ApplyChain {
    const uint32_t* masks;      // mask of pair t at masks + t * mask_stride_w
    size_t mask_stride_w;
    uint8_t* frames;            // the stream's frame store
    size_t frame_stride;
    uint32_t max_frames, base;  // slots; pair t reads slot (base + t) % max_frames and writes (base + t + 1) % max_frames
    uint32_t npix, ntiles, count, pix_bytes;
    const uint8_t* values;      // rank-ordered pixel values of every pair, back to back
    const uint64_t* value_off;  // [count + 1] byte offsets of each pair's values
    const uint8_t* residual;    // [count] 1: pair t's values are residuals, added per sample mod 2^(8 sample_bytes); NULL: all plain
    uint32_t sample_bytes;
    uint32_t* tile_pfx;         // [count][ntiles]: set bits per tile (k_tile_count), then set bits of the earlier tiles (k_tile_scan)
    uint32_t* totals;           // [count] set bits per pair
    uint32_t* first_bad;        // first pair whose value bytes do not match its mask (UINT32_MAX: none); pairs from there are not applied
};

// N4 deflate (rbf_deflate.cuh): one segment of at most 64 KiB per CTA, and the join of coded segments into zlib streams
static constexpr uint32_t kDeflateSeg = 65536;         // segment size (bytes); the layout is pinned in rbf_deflate.cuh
// worst-case output of one segment of n bytes (0 < n <= kDeflateSeg): stored blocks plus the sync flush
__host__ __device__ __forceinline__ uint32_t deflate_seg_bound(uint32_t n) { return n == 0 ? 0u : n + 5u * (n > 65535u ? 2u : 1u) + 5u; }
struct DeflateSeg {
    const uint8_t* src;   // segment bytes (device)
    uint8_t* out;         // output region (16 B aligned)
    uint32_t len;         // 0..kDeflateSeg
    uint32_t cap;         // region bytes
};
struct DeflateCopy {
    const uint8_t* src;   // a segment's coded bytes
    uint64_t dst;         // byte offset of those bytes in the joined range
    uint32_t len;
    uint32_t flags;       // 1: the zlib header goes in front (dst - 2); 2: the trailer goes behind (03 00 + adler)
    uint32_t adler;       // Adler-32 of the whole stream (flags & 2)
    uint32_t pad;
};

// inflate of that layout (rbf_inflate.cuh): candidate segment starts of each stream, each inflated into its own kDeflateSeg slot
enum : uint32_t {
    kInflateOk = 0, kInflateTruncated, kInflateFinal, kInflateBlockType, kInflateStoredLen, kInflateHeader, kInflateCodeLengths,
    kInflateRepeat, kInflateNoEnd, kInflateLitCode, kInflateDistCode, kInflateBadSymbol, kInflateBadDistance, kInflateTooFar,
    kInflateOutputFull,
};
static constexpr uint32_t kInflateScanChunk = 8192;    // candidate positions per k_inflate_scan job
struct InflateSegResult { uint32_t status, consumed, produced, adler; };   // adler: s2 << 16 | s1 of the segment, from (0, 0)
struct InflateScanJob {
    uint64_t base;        // the stream's first byte in the input buffer
    uint32_t begin, end;  // positions [begin, end) of the stream this job scans
    uint32_t stream, cand0, cap, pad;   // the stream's candidates go to cand[cand0 .. cand0 + cap)
};
struct InflateStream {
    uint64_t base, len;
    uint32_t cand0, slot0;   // its candidates in cand[] and its first slot
};
// Adler-32 (s1, s2) of a prefix followed by a part of len bytes whose own sums from (0, 0) are (a1, a2)
__host__ __device__ __forceinline__ void adler_combine(uint32_t& s1, uint32_t& s2, uint64_t len, uint32_t a1, uint32_t a2) {
    s2 = (uint32_t)((s2 + (len % 65521u) * s1 + a2) % 65521u);
    s1 = (uint32_t)((s1 + a1) % 65521u);
}

// What the launchers read from the context (rbf_set_option), and its kernel counter: every launcher adds the kernels it enqueued.
struct LaunchCfg {
    int sm_count = 0;
    int k1_variant = 0;
    int k1_ctas_per_sm = 32;       // grid cap of K1 over the whole GPU
    int insert_variant = 1;        // 1: dense warp-compacted K2 building the arrays in shared memory (default); 0: per-lane K2, RED.OR into L2
    int query_variant = 5;         // 0: per-lane; 1: staged A->B->C rings, L2 tail; 2, 3, 4: as 5; 5: decade tiles with carried stage-B
                                   // batches (half tiles for 2^23 < m <= 2^24, ring kernel beyond); 6: half-decade tiles for every m <= 2^24
    int query_smem_cap = 0;
    int query_warps = 0;           // warps per CTA of the tile query kernel (0 = default: 24 for full-decade tiles, 28 for half ones)
    int k2_clusters[9] = {0};      // resident K2 clusters of 1..8 CTAs, measured by the first K2 launch of each shape.  Not at
                                   // creation: querying it there slowed 8K K3 (which never uses this kernel) by 12 %, cause unknown
    int64_t launches = 0;          // kernels enqueued (rbf_get_counter "kernel_launches")
};

// launchers (all asynchronous on `st`); return cudaError_t of the launch
// chain: the F pairs satisfy pairs[t].curr == pairs[t+1].prev and their frames are 16 B aligned (K1 then reads each frame once);
// sms > 0: a chain's K1 runs on exactly that many SMs, so that K2 runs beside it on the others (a pair list that is not a chain
// takes the whole GPU whatever sms is); 0: the whole GPU, at most L.k1_ctas_per_sm CTAs per SM
cudaError_t launch_threshold(LaunchCfg& L, const PairJob* d_pairs, int F, uint32_t npix, int channels, int sample_bytes,
                             int thr_int, int any_mode, int gray_mode, uint32_t* d_ones, uint32_t* d_resid, bool chain, int sms,
                             cudaStream_t st);
// K2: variant 1 builds the arrays in (cluster) shared memory.  L.k2_clusters[1..8]: resident clusters of that many CTAs, 0 until
// the first launch of the shape measures it with cudaOccupancyMaxActiveClusters (a shape that cannot be scheduled is an error).
// sms: the SMs K2 gets (L.sm_count, or fewer while K1 runs beside it); its waves are sized for that share of the clusters
cudaError_t launch_insert(LaunchCfg& L, const FrameJob* d_jobs, int F, uint32_t max_centuries, uint32_t max_l_bits, int sms, cudaStream_t st);
cudaError_t launch_query(LaunchCfg& L, const FrameJob* d_jobs, const uint32_t* d_cent_prefix, int F, uint32_t total_centuries,
                         uint32_t max_l_bits, cudaStream_t st);
cudaError_t launch_witness(LaunchCfg& L, const FrameJob* d_jobs, int F, uint32_t max_centuries, uint32_t* d_scratch, uint32_t* d_wlen,
                           cudaStream_t st);
cudaError_t launch_expand(LaunchCfg& L, const FrameJob* d_jobs, int F, uint32_t max_centuries, uint32_t* d_scratch, uint32_t* d_consumed,
                          cudaStream_t st);
uint32_t gather_chunks(uint32_t npix);
// kind, as the per-pair modes of K4c: 0 gathers the current frame's samples; 1 curr - prev per sample of sample_bytes; 2 curr minus
// the motion-compensated prev.  A format other than a stream's (pix_bytes, sample_bytes) launches nothing (cudaErrorInvalidValue).
cudaError_t launch_gather(LaunchCfg& L, const GatherJob* d_jobs, int F, uint32_t npix, uint32_t pix_bytes, uint32_t sample_bytes,
                          int kind, uint32_t* d_counts, cudaStream_t st);
// block motion search of F pairs (pairs[f].prev -> pairs[f].curr): d_fields + f * mv_blocks(H, W) * 2 receives the pair's vectors
cudaError_t launch_motion_search(LaunchCfg& L, const PairJob* d_pairs, int F, uint32_t H, uint32_t W, uint32_t pix_bytes, uint32_t sample_bytes,
                                 int8_t* d_fields, cudaStream_t st);
// decode side of a group (rbf_k4c_apply.cuh): masks of the raw-passthrough jobs (l == 0) from their bitmap slots; set bits per mask
cudaError_t launch_raw_masks(LaunchCfg& L, const FrameJob* d_jobs, int F, uint32_t npix, cudaStream_t st);
cudaError_t launch_mask_popcount(LaunchCfg& L, const uint32_t* d_masks, size_t stride_w, uint32_t npix, int F, uint32_t* d_out,
                                 cudaStream_t st);
// K4c: tile counts, tile scan (+ the ivc:882 check) and the chained sweep; *A.first_bad must hold UINT32_MAX before the launch.
// h_modes[t] (host; NULL: every pair 0) is 0 plain, 1 residual, 2 motion-compensated residual; A.residual holds the same modes on
// the device (needed when a mode is not 0), d_fields the [count][mv_blocks(H, W)][2] block vectors (needed when a mode is 2).  One
// tile count + scan for the whole chain, then one k_apply_sweep per run of plain / residual pairs and one k_apply_motion per motion
// pair, in order on `st`; a run without a residual pair gets the plain sweep, which has no residual branch at all.  Without a motion
// pair the one run is the whole chain and gets A's arguments.  d_run_bad: count words of scratch (a run's first failing pair, counted
// from the run's start), read only after a motion pair.
cudaError_t launch_apply_chain(LaunchCfg& L, const ApplyChain& A, const uint8_t* h_modes, const int8_t* d_fields, uint32_t H,
                               uint32_t W, uint32_t* d_run_bad, cudaStream_t st);
cudaError_t launch_median5(LaunchCfg& L, const void* d_in, uint32_t H, uint32_t W, int sample_bytes, void* d_out, cudaStream_t st);
cudaError_t launch_bitrev(LaunchCfg& L, uint32_t* d_words, size_t nwords, cudaStream_t st);
cudaError_t launch_unpack_bits(LaunchCfg& L, const uint32_t* d_words, uint8_t* d_out, size_t nbits, cudaStream_t st);
cudaError_t launch_unpack_bits_msb(LaunchCfg& L, const uint32_t* d_words, uint8_t* d_out, size_t nbits, cudaStream_t st);
cudaError_t launch_popcount(LaunchCfg& L, const uint32_t* d_words, size_t nwords, uint32_t* d_out, cudaStream_t st);
cudaError_t launch_count_diff(LaunchCfg& L, const uint32_t* a, const uint32_t* b, size_t stride_words, size_t nwords, int F,
                              uint32_t* d_out, cudaStream_t st);
// nonzero = 0: a byte == 1 is a set bit (a 0/1 mask); nonzero = 1: any non-zero byte is (a caller's Bloom bit array)
cudaError_t launch_pack_bytes(LaunchCfg& L, const uint8_t* d_bytes, uint32_t* d_words, size_t nbits, int nonzero, cudaStream_t st);

// explicit-item kernels (drop-in RationalBloomFilter.add_index/check_index, rbf add/contains)
cudaError_t launch_items_u32(LaunchCfg& L, const FrameJob* d_job, const uint32_t* d_items, uint32_t count, uint8_t* d_result,
                             int insert, cudaStream_t st);
cudaError_t launch_items_str(LaunchCfg& L, const FrameJob* d_job, const uint8_t* d_blob, const uint64_t* d_offs, uint32_t count,
                             uint8_t* d_result, int insert, int standard_k, cudaStream_t st);
cudaError_t launch_hash_debug(LaunchCfg& L, const uint32_t* d_items, uint32_t count, uint64_t seed, uint64_t* d_out, int mode,
                              cudaStream_t st);

// exchange over peer memory: store `pairs` slots of slot_w words into recv[r] + dst_off_w of every rank, then signal `seq`
cudaError_t launch_push_slots(LaunchCfg& L, const uint32_t* d_bits, size_t stride_w, uint32_t slot_w, uint32_t pairs,
                              uint32_t* const* recv, uint32_t* const* flags, int nranks, int rank, size_t dst_off_w, uint32_t seq,
                              cudaStream_t st);
cudaError_t launch_peer_wait(LaunchCfg& L, const uint32_t* d_flags, int nranks, uint32_t seq, long long timeout_cycles, uint32_t* d_err,
                             cudaStream_t st);

cudaError_t launch_deflate_segments(LaunchCfg& L, const DeflateSeg* d_segs, int count, uint32_t* d_res, uint32_t* d_sizes,
                                    uint32_t* d_adler, uint32_t* d_err, cudaStream_t st);
cudaError_t launch_deflate_concat(LaunchCfg& L, const DeflateCopy* d_jobs, int count, uint8_t* d_dst, uint64_t cap, uint32_t* d_err,
                                  cudaStream_t st);
int deflate_code_lengths_host(const uint32_t* freqs, uint32_t nsym, uint32_t max_bits, uint8_t* lengths);
cudaError_t launch_inflate_scan(LaunchCfg& L, const InflateScanJob* d_jobs, int count, const uint8_t* d_in, uint32_t* d_counts,
                                uint32_t* d_cand, cudaStream_t st);
cudaError_t launch_inflate_segments(LaunchCfg& L, const uint32_t* d_slot_stream, const InflateStream* d_streams, int nslots,
                                    const uint8_t* d_in, const uint32_t* d_cand, uint8_t* d_slots, InflateSegResult* d_res,
                                    uint32_t* d_start, cudaStream_t st);
void inflate_segment_host(const uint8_t* in, uint64_t avail, uint8_t* out, InflateSegResult* res);

int query_max_smem_bytes();

}  // namespace rbf
