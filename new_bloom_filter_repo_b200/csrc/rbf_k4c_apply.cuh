// rbf_k4c_apply.cuh -- batched decode side of the GOP (ivc:268-307, ivc:849-909): masks of raw-passthrough pairs, per-pair mask
// popcounts, and K4c, the chained reconstruction of a group of inter frames.  Included by rbf_kernels.cu inside namespace rbf.
#pragma once

// ------------------------------------------------------------------------------------------
// Raw-passthrough pairs of rbf_stream_decode_masks (J.l == 0): the bitmap slot holds the mask itself (np.packbits order, already
// turned LSB-first by k_bitrev).  Copy its ceil(n/32) words to the mask slot; bits at or beyond n are cleared, so the mask's
// padding stays zero whatever the payload's last byte held (the reference unpacks and cuts at n, ivc:1001).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_raw_masks(const FrameJob* __restrict__ jobs) {
    const FrameJob& J = jobs[blockIdx.y];
    if (J.l != 0) return;
    const uint32_t nwords = (J.n + 31u) >> 5, tail = J.n & 31u;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nwords; i += gridDim.x * blockDim.x) {
        uint32_t v = J.bits[i];
        if (tail && i == nwords - 1u) v &= (1u << tail) - 1u;
        J.out_mask[i] = v;
    }
}

// per pair: set bits of its mask (stride_w words apart, bits at or beyond npix are zero)
__global__ void __launch_bounds__(256) k_mask_popcount(const uint32_t* __restrict__ masks, size_t stride_w, uint32_t nwords,
                                                       uint32_t* __restrict__ out) {
    const uint32_t* m = masks + (size_t)blockIdx.y * stride_w;
    uint32_t c = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nwords; i += gridDim.x * blockDim.x) c += __popc(__ldg(m + i));
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out + blockIdx.y, c);
}

// ------------------------------------------------------------------------------------------
// K4c: frame base+1+t = frame base+t with mask t applied (ivc:849-909), t = 0 .. count-1, in one launch.
// Fixed tiles of AP_TILE_PX pixels (AP_TILE_WORDS mask words, one per thread).  Where the values of a tile start comes from two
// small kernels: k_tile_count (set bits per (pair, tile), one warp per tile) and k_tile_scan (exclusive scan over the tiles of a
// pair, one CTA per pair), which also checks ivc:882 -- popcount x pixel bytes == the pair's value bytes -- and records the first
// pair that fails.  k_apply_sweep then runs persistent CTAs that each own a share of the tiles: the base frame's tile is loaded
// into shared memory once and walked through the chain -- replace the set pixels of mask t in rank order, store the tile as
// output frame t with 16 B stores -- for every t before the first failing pair.  A residual pair adds its values to the set
// pixels per sample instead of replacing them (value_mode 1 of the gather).  Each output frame is written once and nothing
// is copied device to device.  Frame slots are taken modulo max_frames, so a chain continues from the last frame of the
// previous one wherever it sits.
// Ragged end: the last tile of a frame is loaded and stored as whole 16 B units plus single bytes for the rest (frames start
// 256 B aligned and a tile is 16 B aligned); mask bits at or beyond npix are ignored.
// ------------------------------------------------------------------------------------------

__device__ __forceinline__ uint32_t mask_word_valid(const uint32_t* __restrict__ m, uint32_t w, uint32_t npix) {
    const uint32_t nwords = (npix + 31u) >> 5;
    if (w >= nwords) return 0u;
    uint32_t v = __ldg(m + w);
    if (w == nwords - 1u && (npix & 31u)) v &= (1u << (npix & 31u)) - 1u;
    return v;
}

__global__ void __launch_bounds__(256) k_tile_count(const ApplyChain A) {
    const uint32_t tile = blockIdx.x * 8u + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
    if (tile >= A.ntiles) return;
    const uint32_t* m = A.masks + (size_t)blockIdx.y * A.mask_stride_w;
    uint32_t c = 0;
#pragma unroll
    for (uint32_t q = 0; q < AP_TILE_WORDS / 32u; q++) c += __popc(mask_word_valid(m, tile * AP_TILE_WORDS + q * 32u + lane, A.npix));
    c = __reduce_add_sync(0xffffffffu, c);
    if (lane == 0) A.tile_pfx[(size_t)blockIdx.y * A.ntiles + tile] = c;
}

__global__ void __launch_bounds__(1024) k_tile_scan(const ApplyChain A) {
    __shared__ uint32_t s_warp[33];
    uint32_t* p = A.tile_pfx + (size_t)blockIdx.x * A.ntiles;
    uint32_t base = 0;
    for (uint32_t t0 = 0; t0 < A.ntiles; t0 += blockDim.x) {
        const uint32_t i = t0 + threadIdx.x;
        const uint32_t v = i < A.ntiles ? p[i] : 0u;
        uint32_t tot;
        const uint32_t ex = block_excl_scan(v, s_warp, tot);
        if (i < A.ntiles) p[i] = base + ex;
        base += tot;
    }
    if (threadIdx.x == 0) {
        A.totals[blockIdx.x] = base;
        if ((uint64_t)base * A.pix_bytes != A.value_off[blockIdx.x + 1] - A.value_off[blockIdx.x]) atomicMin(A.first_bad, blockIdx.x);   // ivc:882
    }
}

// RS = 0: every pair is plain (A.residual is not read).  RS = 1 or 2: pairs with A.residual[t] set add their values to the tile per
// sample of RS bytes, with wrap-around; the other pairs replace pixels as in the plain sweep.
template <int PB, int RS>
__global__ void __launch_bounds__(AP_THREADS) k_apply_sweep(const ApplyChain A) {
    __shared__ __align__(16) uint8_t tile[AP_TILE_PX * PB];
    __shared__ uint32_t s_warp[33];
    const uint32_t count = min(A.count, *A.first_bad);
    for (uint32_t tl = blockIdx.x; tl < A.ntiles; tl += gridDim.x) {
        const uint32_t px0 = tl * AP_TILE_PX;
        const uint32_t bytes = min(AP_TILE_PX, A.npix - px0) * PB, whole = bytes & ~15u;
        const uint8_t* src = A.frames + (size_t)A.base * A.frame_stride + (size_t)px0 * PB;
        for (uint32_t b = threadIdx.x * 16u; b < whole; b += AP_THREADS * 16u)
            *reinterpret_cast<uint4*>(tile + b) = __ldg(reinterpret_cast<const uint4*>(src + b));
        for (uint32_t b = whole + threadIdx.x; b < bytes; b += AP_THREADS) tile[b] = src[b];
        const uint32_t w = tl * AP_TILE_WORDS + threadIdx.x;
        // mask word and tile offset of pair t + 1 are fetched while pair t is applied
        uint32_t m = count ? mask_word_valid(A.masks, w, A.npix) : 0u;
        uint32_t pfx = count ? __ldg(A.tile_pfx + tl) : 0u;
        for (uint32_t t = 0; t < count; t++) {
            uint32_t m_next = 0u, pfx_next = 0u;
            if (t + 1u < count) {
                m_next = mask_word_valid(A.masks + (size_t)(t + 1u) * A.mask_stride_w, w, A.npix);
                pfx_next = __ldg(A.tile_pfx + (size_t)(t + 1u) * A.ntiles + tl);
            }
            uint32_t tot;
            // its barriers also order the previous iteration's stores (and the load above) before this iteration's writes
            const uint32_t rank = pfx + block_excl_scan(__popc(m), s_warp, tot);
            const uint8_t* v = A.values + A.value_off[t] + (size_t)rank * PB;
            bool add = false;
            if constexpr (RS != 0) add = __ldg(A.residual + t) != 0;
            while (m) {
                const uint32_t b = __ffs(m) - 1;
                m &= m - 1u;
                if constexpr (RS != 0) {
                    if (add) add_pixel<PB, RS>(tile + (threadIdx.x * 32u + b) * PB, v);
                    else copy_pixel<PB>(tile + (threadIdx.x * 32u + b) * PB, v);
                } else {
                    copy_pixel<PB>(tile + (threadIdx.x * 32u + b) * PB, v);
                }
                v += PB;
            }
            __syncthreads();
            uint32_t slot = A.base + t + 1u;
            if (slot >= A.max_frames) slot -= A.max_frames;
            uint8_t* dst = A.frames + (size_t)slot * A.frame_stride + (size_t)px0 * PB;
            for (uint32_t b = threadIdx.x * 16u; b < whole; b += AP_THREADS * 16u)
                *reinterpret_cast<uint4*>(dst + b) = *reinterpret_cast<const uint4*>(tile + b);
            for (uint32_t b = whole + threadIdx.x; b < bytes; b += AP_THREADS) dst[b] = tile[b];
            m = m_next;
            pfx = pfx_next;
        }
        __syncthreads();                                   // the tile is read out before the next one is loaded
    }
}
