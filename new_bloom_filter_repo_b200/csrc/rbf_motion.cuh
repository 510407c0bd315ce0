// rbf_motion.cuh -- block motion of the inter-frame value stream (value_coding "motion"): the full search over +-16 px per 16 x 16
// block, and the motion-compensated apply of the decoder.  Included by rbf_kernels.cu inside namespace rbf, after rbf_k4c_apply.cuh.
#pragma once

// ------------------------------------------------------------------------------------------
// k_motion_search: one CTA per (block, pair).  The block of curr (zero outside the frame) and the prev window it can see -- block
// +-16 px, each sample taken at the clamped coordinate, so window(wy, wx) = prev(clamp(y0 - 16 + wy), clamp(x0 - 16 + wx)) -- are
// staged in shared memory as 32-bit words.  Thread (g, dx), g < 3, owns the 11 candidates (dx, 11 g - 16 + j), j < 11: it walks the
// 26 window rows those candidates touch, funnel-shifts each row by dx into registers once, and adds its byte-SIMD SAD against every
// curr row that meets it under one of its candidates (4 samples per VABSDIFF4 for 8-bit samples, 2 per __vsadu2 for 16-bit ones).
// The minimum of (SAD, |dx| + |dy|, dy, dx) as one 64-bit key picks the vector, so every tie is broken the same way.
// Columns and rows outside the frame (right / bottom edge blocks) add nothing: curr is zero there and the window words are masked.
// ------------------------------------------------------------------------------------------
static constexpr int MV_WIN = MV_BLOCK + 2 * MV_RANGE;                 // 48 window rows / columns
static constexpr int MV_NCAND = 2 * MV_RANGE + 1;                      // 33 candidates per axis
static constexpr int MV_DYS = 11;                                      // dy per thread; 3 groups cover the 33
static constexpr int MV_THREADS = 128;                                 // 99 search threads; all 128 stage

template <int S>
__device__ __forceinline__ uint32_t sad_word(uint32_t a, uint32_t b, uint32_t acc) {
    if constexpr (S == 1) return acc + __vsadu4(a, b);                 // VABSDIFF4.U8.ACC
    else return acc + __vsadu2(a, b);
}

template <int PB, int S>
__global__ void __launch_bounds__(MV_THREADS) k_motion_search(const PairJob* __restrict__ pairs, uint32_t H, uint32_t W,
                                                              int8_t* __restrict__ fields) {
    constexpr int NW = 4 * PB;                                         // words per block row (16 px)
    constexpr int WP = 12 * PB + 1;                                    // words per window row (48 px) + 1 for the funnel shift
    __shared__ __align__(16) uint32_t s_cur[MV_BLOCK * NW];
    __shared__ uint32_t s_win[MV_WIN * WP];
    __shared__ unsigned long long s_best[MV_THREADS / 32];
    const PairJob P = pairs[blockIdx.y];
    const uint32_t bxn = mv_blocks_x(W);
    const uint32_t by = blockIdx.x / bxn, bx = blockIdx.x - by * bxn;
    const int y0 = (int)(by * MV_BLOCK), x0 = (int)(bx * MV_BLOCK);
    const uint32_t bh = min((uint32_t)MV_BLOCK, H - (uint32_t)y0), bw = min((uint32_t)MV_BLOCK, W - (uint32_t)x0);
    uint8_t* win = reinterpret_cast<uint8_t*>(s_win);
    for (uint32_t i = threadIdx.x; i < (uint32_t)(MV_WIN * MV_WIN); i += MV_THREADS) {
        const int wy = (int)(i / MV_WIN), wx = (int)(i % MV_WIN);
        const int gy = min(max(y0 - MV_RANGE + wy, 0), (int)H - 1), gx = min(max(x0 - MV_RANGE + wx, 0), (int)W - 1);
        copy_pixel<PB>(win + (size_t)wy * WP * 4 + wx * PB, P.prev + ((size_t)gy * W + gx) * PB);
    }
    if (threadIdx.x < (uint32_t)MV_WIN) s_win[threadIdx.x * WP + WP - 1] = 0u;
    uint8_t* cur = reinterpret_cast<uint8_t*>(s_cur);
    for (uint32_t i = threadIdx.x; i < (uint32_t)(MV_BLOCK * MV_BLOCK); i += MV_THREADS) {
        const uint32_t py = i / MV_BLOCK, px = i % MV_BLOCK;
        if (py < bh && px < bw) copy_pixel<PB>(cur + i * PB, P.curr + ((size_t)(y0 + py) * W + x0 + px) * PB);
        else for (int q = 0; q < PB; q++) cur[i * PB + q] = 0;
    }
    __syncthreads();

    unsigned long long best = ~0ull;
    if (threadIdx.x < (uint32_t)(3 * MV_NCAND)) {
        const int g = (int)threadIdx.x / MV_NCAND, dx = (int)threadIdx.x % MV_NCAND - MV_RANGE;
        const uint32_t o = (uint32_t)((dx + MV_RANGE) * PB), k0 = o >> 2, sh = 8u * (o & 3u);
        const uint32_t vb = bw * PB;                                   // valid bytes of a block row
        uint32_t acc[MV_DYS];
#pragma unroll
        for (int j = 0; j < MV_DYS; j++) acc[j] = 0u;
#pragma unroll 1
        for (uint32_t r = 0; r < (uint32_t)(MV_DYS + MV_BLOCK - 1); r++) {
            // candidate dy = 11 g - 16 + j meets block row py = r - j in window row py + 16 + dy = 11 g + r
            const uint32_t* wr = s_win + (size_t)(MV_DYS * g + r) * WP + k0;
            uint32_t p[NW];
#pragma unroll
            for (int k = 0; k < NW; k++) p[k] = __funnelshift_r(wr[k], wr[k + 1], sh);
            if (vb < (uint32_t)(MV_BLOCK * PB)) {                      // right edge block: bytes past the frame add nothing
#pragma unroll
                for (int k = 0; k < NW; k++) {
                    const uint32_t b = 4u * k;
                    p[k] &= b >= vb ? 0u : (b + 4u <= vb ? ~0u : (1u << (8u * (vb - b))) - 1u);
                }
            }
#pragma unroll
            for (int j = 0; j < MV_DYS; j++) {
                const uint32_t py = r - (uint32_t)j;
                if (py < bh) {
                    const uint4* cr = reinterpret_cast<const uint4*>(s_cur + py * NW);
#pragma unroll
                    for (int q = 0; q < PB; q++) {
                        const uint4 c = cr[q];
                        acc[j] = sad_word<S>(c.x, p[4 * q], acc[j]);
                        acc[j] = sad_word<S>(c.y, p[4 * q + 1], acc[j]);
                        acc[j] = sad_word<S>(c.z, p[4 * q + 2], acc[j]);
                        acc[j] = sad_word<S>(c.w, p[4 * q + 3], acc[j]);
                    }
                }
            }
        }
#pragma unroll
        for (int j = 0; j < MV_DYS; j++) {
            const int dy = MV_DYS * g - MV_RANGE + j;
            const uint32_t l1 = (uint32_t)(abs(dx) + abs(dy));
            const unsigned long long key = ((unsigned long long)acc[j] << 18) | (l1 << 12) | ((uint32_t)(dy + MV_RANGE) << 6) |
                                           (uint32_t)(dx + MV_RANGE);
            best = key < best ? key : best;
        }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        const unsigned long long o = __shfl_xor_sync(0xffffffffu, best, d);
        best = o < best ? o : best;
    }
    if ((threadIdx.x & 31u) == 0) s_best[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long b = s_best[0];
#pragma unroll
        for (int w = 1; w < MV_THREADS / 32; w++) b = s_best[w] < b ? s_best[w] : b;
        int8_t* f = fields + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * 2;
        f[0] = (int8_t)((int)(b & 63u) - MV_RANGE);
        f[1] = (int8_t)((int)((b >> 6) & 63u) - MV_RANGE);
    }
}

// ------------------------------------------------------------------------------------------
// k_apply_motion: pair t of a K4c chain whose values are motion-compensated residuals.  One CTA per tile of AP_TILE_PX pixels, as
// k_apply_sweep with a chain of one: the tile of frame base + t is staged in shared memory, each set pixel becomes pred + value per
// sample (mod 2^(8 S)), where pred is read from frame base + t in global memory (the prediction crosses tiles, so the sweep cannot
// carry it), and the tile is stored as frame base + t + 1.  The rank of a set pixel comes from the chain's k_tile_scan prefixes.
// Nothing is written when t is at or past the chain's first failing pair.  A run of plain / residual pairs that starts at t + 1 is
// swept as a chain of its own, whose first failing pair is counted from t + 1: CTA 0 stores that count to *next_bad (if not NULL).
// ------------------------------------------------------------------------------------------
template <int PB, int S>
__global__ void __launch_bounds__(AP_THREADS) k_apply_motion(const ApplyChain A, uint32_t t, const int8_t* __restrict__ fields, uint32_t H,
                                                             uint32_t W, uint32_t* __restrict__ next_bad) {
    __shared__ __align__(16) uint8_t tile[AP_TILE_PX * PB];
    __shared__ uint32_t s_warp[33];
    const uint32_t first_bad = *A.first_bad;
    if (next_bad && blockIdx.x == 0 && threadIdx.x == 0) *next_bad = max(first_bad, t + 1u) - (t + 1u);
    if (t >= first_bad) return;
    const uint32_t tl = blockIdx.x, px0 = tl * AP_TILE_PX;
    const uint32_t bytes = min(AP_TILE_PX, A.npix - px0) * PB, whole = bytes & ~15u;
    uint32_t in_slot = A.base + t;
    if (in_slot >= A.max_frames) in_slot -= A.max_frames;
    const uint32_t out_slot = in_slot + 1u == A.max_frames ? 0u : in_slot + 1u;
    const uint8_t* in = A.frames + (size_t)in_slot * A.frame_stride;
    const uint8_t* src = in + (size_t)px0 * PB;
    for (uint32_t b = threadIdx.x * 16u; b < whole; b += AP_THREADS * 16u)
        *reinterpret_cast<uint4*>(tile + b) = __ldg(reinterpret_cast<const uint4*>(src + b));
    for (uint32_t b = whole + threadIdx.x; b < bytes; b += AP_THREADS) tile[b] = src[b];
    uint32_t m = mask_word_valid(A.masks + (size_t)t * A.mask_stride_w, tl * AP_TILE_WORDS + threadIdx.x, A.npix);
    uint32_t tot;
    // its barriers also order the tile load above before the writes below
    const uint32_t rank = __ldg(A.tile_pfx + (size_t)t * A.ntiles + tl) + block_excl_scan(__popc(m), s_warp, tot);
    const uint8_t* v = A.values + A.value_off[t] + (size_t)rank * PB;
    const int8_t* field = fields + (size_t)t * mv_blocks(H, W) * 2;
    while (m) {
        const uint32_t b = __ffs(m) - 1;
        m &= m - 1u;
        const uint32_t lp = threadIdx.x * 32u + b;
        uint8_t* dst = tile + (size_t)lp * PB;
        copy_pixel<PB>(dst, in + motion_src(field, W, H, px0 + lp) * PB);
        add_pixel<PB, S>(dst, v);
        v += PB;
    }
    __syncthreads();
    uint8_t* dst = A.frames + (size_t)out_slot * A.frame_stride + (size_t)px0 * PB;
    for (uint32_t b = threadIdx.x * 16u; b < whole; b += AP_THREADS * 16u)
        *reinterpret_cast<uint4*>(dst + b) = *reinterpret_cast<const uint4*>(tile + b);
    for (uint32_t b = whole + threadIdx.x; b < bytes; b += AP_THREADS) dst[b] = tile[b];
}
