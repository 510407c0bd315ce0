// rbf_k1_threshold.cuh -- K1: |Y_prev - Y_curr| > thr -> packed mask + counts (ivc:788-808, ivc:211).  Included by rbf_kernels.cu inside namespace rbf.
#pragma once

// ------------------------------------------------------------------------------------------
// K1: threshold + popcount.  One thread = 32 consecutive pixels = one mask word (threshold_word).
// PB = bytes per pixel (channels * sample bytes), S = sample bytes; Y is the first sample.
//   k_threshold_sweep  pairs that form a chain (consecutive frames, the benchmark's case): each frame is read from HBM once
//                      (2.87 ms per 299 4K pairs on an H100 80GB HBM3 at 400 W, 0.81 of the 3.35 TB/s data-sheet bandwidth)
//   k_threshold        any pair list: the pixel bytes of a warp are staged in shared memory (see stage_warp), 2*PB 16 B
//                      copies per lane and frame; a frame shared by two pairs is read twice (4.33 ms on the same card)
//   k_threshold_tma    k1_variant=1
// ------------------------------------------------------------------------------------------
template <int PB, int S>
__device__ __forceinline__ int absdiff_sample(uint32_t a, uint32_t b) {
    if (S == 1) {
        int d = (int)a - (int)b;
        return d < 0 ? -d : d;
    } else {                                           // numpy int16 wrap-around (ivc:801)
        int16_t x = (int16_t)(uint16_t)a, y = (int16_t)(uint16_t)b;
        int16_t d = (int16_t)(x - y);
        int16_t ad = (int16_t)(d < 0 ? -d : d);      // abs(-32768) stays -32768
        return (int)ad;
    }
}

// cv2.cvtColor(frame, cv2.COLOR_BGR2GRAY) of the reference's non-YUV colour branch (ivc:792-795): OpenCV's 15-bit
// fixed point, identical for 8- and 16-bit samples (checked against cv2 4.13 in tests/golden/make_golden.py)
__device__ __forceinline__ uint32_t bgr2gray_fixed(uint32_t b, uint32_t g, uint32_t r) {
    return (b * 3735u + g * 19235u + r * 9798u + 16384u) >> 15;
}

// one 32 B sector per thread: two 128-bit streaming loads (LDG.E.128, the widest global load on sm_90a)
__device__ __forceinline__ void ldg32B_stream(const void* p, uint32_t* r) {
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "l"(p));
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7])
                 : "l"((const uint8_t*)p + 16));
}

// Four consecutive 8-bit YUV444 pixels = three 32-bit words per frame.  Byte-SIMD:
//   nm = 4-bit mask of  |Ya - Yb| > thr  (VABSDIFF4 + per-byte compare),  nd = 4-bit "any byte differs".
// gt_or / gt_and fold the out-of-range thresholds (thr < 0: always, thr > 254: never) into the compare.
__device__ __forceinline__ void yuv8_group4(uint32_t a0, uint32_t a1, uint32_t a2, uint32_t b0, uint32_t b1, uint32_t b2,
                                            uint32_t thr4, uint32_t gt_or, uint32_t gt_and, uint32_t& nm, uint32_t& nd) {
    const uint32_t ya = __byte_perm(__byte_perm(a0, a1, 0x0630), a2, 0x5210);   // Y bytes of pixels 0..3
    const uint32_t yb = __byte_perm(__byte_perm(b0, b1, 0x0630), b2, 0x5210);
    const uint32_t gt = (__vcmpgtu4(__vabsdiffu4(ya, yb), thr4) & gt_and) | gt_or;
    nm = ((gt & 0x01010101u) * 0x01020408u) >> 24;
    const uint32_t x0 = a0 ^ b0, x1 = a1 ^ b1, x2 = a2 ^ b2;
    const uint32_t f0 = x0 & 0x00ffffffu, f1 = __funnelshift_r(x0, x1, 24) & 0x00ffffffu,
                   f2 = __funnelshift_r(x1, x2, 16) & 0x00ffffffu, f3 = x2 >> 8;
    nd = min(f0, 1u) | (min(f1, 1u) << 1) | (min(f2, 1u) << 2) | (min(f3, 1u) << 3);
}

// The 32 B of a thread come from shared memory (staged) or straight from global memory
__device__ __forceinline__ void load32B(const uint8_t* p, uint32_t* r, bool staged) {
    if (staged) {
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7]) : "r"(smem_u32(p + 16)));
    } else {
        ldg32B_stream(p, r);
    }
}

// Without a 256-bit load, a thread's 32 B sector takes two 128-bit loads, and at a lane stride of 32*PB bytes each of them
// fetches every sector from L2.  So a warp whose 1024 pixels all lie in the frame first copies them, from both frames, with
// coalesced 16 B cp.async (cached in L2 only) into its slice of shared memory; the lanes then read their own 32 pixels there.
constexpr int K1_THREADS = 256;
constexpr int K1_STAGE_BYTES_PER_PB = (K1_THREADS / 32) * 2 * 1024;    // dynamic shared memory of k_threshold = this * PB

template <int PB>
__device__ __forceinline__ void stage_warp(uint8_t* dst, const uint8_t* src, uint32_t lane) {
#pragma unroll
    for (int j = 0; j < 2 * PB; j++)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst + 512 * j + 16 * lane)), "l"(src + 512 * j + 16 * lane)
                     : "memory");
}

// The threshold in the forms the per-word compare uses
struct K1Thr {
    int thr, any_mode;
    uint32_t thr4, gt_or, gt_and, any_mask;
};
__device__ __forceinline__ K1Thr k1_thr(int thr, int any_mode) {
    K1Thr t;
    t.thr = thr;
    t.any_mode = any_mode;
    t.thr4 = (uint32_t)(thr < 0 ? 0 : (thr > 254 ? 254 : thr)) * 0x01010101u;
    t.gt_or = thr < 0 ? 0xffffffffu : 0u;
    t.gt_and = thr > 254 ? 0u : 0xffffffffu;
    t.any_mask = any_mode ? 0xfu : 0u;
    return t;
}

// One mask word: the 32 whole pixels at pa (prev) and pb (curr), in shared memory (staged) or global memory, both 16 B aligned.
// m = mask bits, r = residual bits (some byte of the pixel differs, mask bit clear).
template <int PB, int S, bool GRAY>
__device__ __forceinline__ void threshold_word(const uint8_t* pa, const uint8_t* pb, bool staged, const K1Thr& t, uint32_t& m,
                                               uint32_t& r) {
    m = 0; r = 0;
    if (PB == 3 && S == 1 && !GRAY) {
        uint32_t A[24], B[24];
#pragma unroll
        for (int j = 0; j < 3; j++) load32B(pa + 32 * j, A + 8 * j, staged);
#pragma unroll
        for (int j = 0; j < 3; j++) load32B(pb + 32 * j, B + 8 * j, staged);
#pragma unroll
        for (int g = 0; g < 8; g++) {
            uint32_t nm, nd;
            yuv8_group4(A[3 * g], A[3 * g + 1], A[3 * g + 2], B[3 * g], B[3 * g + 1], B[3 * g + 2], t.thr4, t.gt_or, t.gt_and, nm, nd);
            nm |= nd & t.any_mask;
            m |= nm << (4 * g);
            r |= (nd & ~nm) << (4 * g);
        }
    } else {
        constexpr int NV = PB;                     // 32 B loads per 32 pixels
        constexpr int HV = (NV > 3) ? NV / 2 : NV; // at most 3 in flight per frame
        constexpr int HALVES = NV / HV;
        constexpr int PXH = 32 / HALVES;
#pragma unroll
        for (int hf = 0; hf < HALVES; hf++) {
            uint32_t A[8 * HV], B[8 * HV];
            const uint32_t ho = (uint32_t)(hf * PXH) * PB;
#pragma unroll
            for (int j = 0; j < HV; j++) load32B(pa + ho + 32 * j, A + 8 * j, staged);
#pragma unroll
            for (int j = 0; j < HV; j++) load32B(pb + ho + 32 * j, B + 8 * j, staged);
#pragma unroll
            for (int k = 0; k < PXH; k++) {
                const int o = k * PB;              // byte offset of the pixel (compile-time)
                const uint32_t smask = (S == 1) ? 0xffu : 0xffffu;
                uint32_t ya = (A[o >> 2] >> (8 * (o & 3))) & smask;
                uint32_t yb = (B[o >> 2] >> (8 * (o & 3))) & smask;
                if (GRAY) {                        // samples 1 and 2 of the pixel (compile-time offsets; S == 2 samples are 2-aligned)
                    const int p1 = o + S, p2 = o + 2 * S;
                    const uint32_t a1 = (A[p1 >> 2] >> (8 * (p1 & 3))) & smask, a2 = (A[p2 >> 2] >> (8 * (p2 & 3))) & smask;
                    const uint32_t b1 = (B[p1 >> 2] >> (8 * (p1 & 3))) & smask, b2 = (B[p2 >> 2] >> (8 * (p2 & 3))) & smask;
                    ya = bgr2gray_fixed(ya, a1, a2);
                    yb = bgr2gray_fixed(yb, b1, b2);
                }
                uint32_t anyd = 0;                 // any byte of the pixel differs
#pragma unroll
                for (int q = 0; q < PB; q++) {
                    const int oq = o + q;
                    anyd |= ((A[oq >> 2] ^ B[oq >> 2]) >> (8 * (oq & 3))) & 0xffu;
                }
                const uint32_t bit = ((absdiff_sample<PB, S>(ya, yb) > t.thr) || (t.any_mode && anyd != 0u)) ? 1u : 0u;
                m |= bit << (hf * PXH + k);
                r |= ((anyd != 0u && bit == 0u) ? 1u : 0u) << (hf * PXH + k);
            }
        }
    }
}

// The ragged last word of a frame: the first nvalid (< 32) pixels at a (prev) and b (curr) in global memory, scalar loads.
template <int PB, int S, bool GRAY>
__device__ __forceinline__ void threshold_word_tail(const uint8_t* pa, const uint8_t* pb, uint32_t nvalid, const K1Thr& t, uint32_t& m,
                                                    uint32_t& r) {
    m = 0; r = 0;
    for (uint32_t k = 0; k < nvalid; k++) {
        const uint8_t* a = pa + (size_t)k * PB;
        const uint8_t* b = pb + (size_t)k * PB;
        uint32_t ya = a[0], yb = b[0];
        if (S == 2) { ya |= (uint32_t)a[1] << 8; yb |= (uint32_t)b[1] << 8; }
        if (GRAY) {
            uint32_t a1 = a[S], a2 = a[2 * S], b1 = b[S], b2 = b[2 * S];
            if (S == 2) { a1 |= (uint32_t)a[3] << 8; a2 |= (uint32_t)a[5] << 8; b1 |= (uint32_t)b[3] << 8; b2 |= (uint32_t)b[5] << 8; }
            ya = bgr2gray_fixed(ya, a1, a2);
            yb = bgr2gray_fixed(yb, b1, b2);
        }
        uint32_t anyd = 0;
        for (int q = 0; q < PB; q++) anyd |= (uint32_t)(a[q] ^ b[q]);
        const uint32_t bit = ((absdiff_sample<PB, S>(ya, yb) > t.thr) || (t.any_mode && anyd != 0u)) ? 1u : 0u;
        m |= bit << k;
        r |= ((anyd != 0u && bit == 0u) ? 1u : 0u) << k;
    }
}

// K1 for any list of pairs: grid (bx, pairs), each CTA grid-strides over the mask words of its pair.
template <int PB, int S, bool GRAY = false>
__global__ void __launch_bounds__(K1_THREADS) k_threshold(const PairJob* __restrict__ pairs, uint32_t npix, int thr, int any_mode,
                                                          uint32_t* __restrict__ ones, uint32_t* __restrict__ resid) {
    static_assert(!GRAY || PB == 3 * S, "BGR->gray needs three samples per pixel");
    extern __shared__ __align__(16) uint8_t k1_stage[];               // [warp][prev, curr][1024 * PB]
    const PairJob pj = pairs[blockIdx.y];
    const uint32_t nwords = (npix + 31u) >> 5;
    uint32_t cnt_ones = 0, cnt_res = 0;
    const K1Thr t = k1_thr(thr, any_mode);
    const uint32_t lane = threadIdx.x & 31u;
    uint8_t* const sa = k1_stage + (threadIdx.x >> 5) * 2048 * PB;
    uint8_t* const sb = sa + 1024 * PB;
    for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < nwords; w += gridDim.x * blockDim.x) {
        const uint32_t px0 = w << 5;
        uint32_t m, r;
        const bool staged = (uint64_t)((w | 31u) + 1u) * 32u <= npix;          // warp-uniform: the block stride is a multiple of 32
        if (staged) {
            __syncwarp();                                                    // the lanes have read the previous iteration's slice
            const size_t off = (size_t)(w & ~31u) * 32u * PB;
            stage_warp<PB>(sa, pj.prev + off, lane);
            stage_warp<PB>(sb, pj.curr + off, lane);
            asm volatile("cp.async.wait_all;" ::: "memory");
            __syncwarp();
        }
        if (px0 + 32u <= npix)
            threshold_word<PB, S, GRAY>(staged ? sa + lane * 32u * PB : pj.prev + (size_t)px0 * PB,
                                        staged ? sb + lane * 32u * PB : pj.curr + (size_t)px0 * PB, staged, t, m, r);
        else
            threshold_word_tail<PB, S, GRAY>(pj.prev + (size_t)px0 * PB, pj.curr + (size_t)px0 * PB, npix - px0, t, m, r);
        pj.mask[w] = m;
        cnt_ones += __popc(m);
        cnt_res += __popc(r);
    }
    // block reduction -> one atomic per block
    __shared__ uint32_t s_o[8], s_r[8];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        cnt_ones += __shfl_xor_sync(0xffffffffu, cnt_ones, d);
        cnt_res += __shfl_xor_sync(0xffffffffu, cnt_res, d);
    }
    const int warp = threadIdx.x >> 5;
    if (lane == 0) { s_o[warp] = cnt_ones; s_r[warp] = cnt_res; }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t to = 0, tr = 0;
        for (int i = 0; i < (int)(blockDim.x >> 5); i++) { to += s_o[i]; tr += s_r[i]; }
        if (to) atomicAdd(ones + blockIdx.y, to);
        if (tr) atomicAdd(resid + blockIdx.y, tr);
    }
}

// ------------------------------------------------------------------------------------------
// K1 over a chain of pairs (pairs[t].curr == pairs[t+1].prev, 16 B aligned frames).  k_threshold reads every frame twice, as curr
// of pair t-1 and as prev of pair t, and only an accident of scheduling lets the second read hit L2.  Here a persistent CTA takes
// a tile of SW_TILE_PX pixels and sweeps it through the frames prev(0), curr(0), curr(1), ..., curr(P-1): each frame tile is
// copied once, by cp.async.bulk into a ring of SW_STAGES slots (one mbarrier each), and is compared as curr of pair t-1 and as
// prev of pair t.  One thread per mask word; the compare is threshold_word, as in k_threshold.
// Ragged end: the bulk copy of the last tile of a frame is rounded down to 16 B, which still holds every whole 32-pixel word of
// the tile (a word ends on a multiple of 32 B); the ragged last word of the frame (< 32 px) is read from global memory by
// threshold_word_tail.  Mask words at or beyond ceil(npix/32) are not written.
// A CTA runs blockDim.x / SW_THREADS such sweeps, each with its own ring, mbarriers, counts and named barrier, and nothing
// shared between them: sweep g of CTA b takes tiles (b * G + g) + k * (gridDim.x * G).  Over the whole GPU the launcher
// runs one sweep per CTA; beside K2 it runs wide CTAs on a few SMs (see launch_threshold_sweep_t).
// ------------------------------------------------------------------------------------------
constexpr int SW_THREADS = 128;                       // one sweep
constexpr uint32_t SW_TILE_PX = 32u * SW_THREADS;     // 4096 px: 4 / 8 / 12 / 24 KB per frame tile at 1 / 2 / 3 / 6 B per pixel
constexpr int SW_STAGES = 4;                          // frames t and t+1 are read while t+2 and t+3 are in flight
constexpr int SW_MAX_SWEEPS = 4;                      // sweeps per CTA (named barriers 1..4)
// shared memory of one sweep: its ring, then its SW_STAGES mbarriers and the per-warp counts of two frames (96 B)
template <int PB>
__host__ __device__ constexpr uint32_t sw_sweep_bytes() { return (uint32_t)SW_STAGES * SW_TILE_PX * PB + 128u; }

template <int PB, int S, bool GRAY = false>
__global__ void __launch_bounds__(SW_THREADS * SW_MAX_SWEEPS) k_threshold_sweep(const PairJob* __restrict__ pairs, uint32_t P,
                                                                                uint32_t npix, int thr, int any_mode,
                                                                                uint32_t* __restrict__ ones, uint32_t* __restrict__ resid) {
    static_assert(!GRAY || PB == 3 * S, "BGR->gray needs three samples per pixel");
    constexpr uint32_t SLOT = SW_TILE_PX * PB;
    constexpr int NWARP = SW_THREADS / 32;
    extern __shared__ __align__(128) uint8_t k1_sweeps[];             // [sweep][sw_sweep_bytes<PB>()]
    const uint32_t g = __shfl_sync(0xffffffffu, threadIdx.x / SW_THREADS, 0);   // this thread's sweep (warp-uniform for the compiler)
    const uint32_t tid = threadIdx.x % SW_THREADS, G = blockDim.x / SW_THREADS;
    uint8_t* const ring = k1_sweeps + g * sw_sweep_bytes<PB>();       // [SW_STAGES][SLOT]
    uint64_t* const full = reinterpret_cast<uint64_t*>(ring + SW_STAGES * SLOT);
    uint32_t(*const s_cnt)[NWARP][2] = reinterpret_cast<uint32_t(*)[NWARP][2]>(full + SW_STAGES);   // [2][NWARP][ones, resid]
    const uint32_t sweep = blockIdx.x * G + g, nsweeps = gridDim.x * G;
    const uint32_t nwords = (npix + 31u) >> 5;
    const uint32_t ntiles = (npix + SW_TILE_PX - 1u) / SW_TILE_PX;
    const uint32_t my_tiles = sweep < ntiles ? (ntiles - 1u - sweep) / nsweeps + 1u : 0u;
    const uint32_t nfr = P + 1u;                                       // frames of the chain
    const uint64_t total = (uint64_t)my_tiles * nfr;                   // this sweep's (tile, frame) loads, tile-major
    const K1Thr t = k1_thr(thr, any_mode);
    const uint32_t lane = tid & 31u, warp = tid >> 5;

    if (tid == 0) {
        for (int s = 0; s < SW_STAGES; s++) mbar_init(&full[s], 1);
        fence_mbar_init();
    }
    __syncthreads();

    // load i = (k-th tile of this sweep, frame j) into slot i % SW_STAGES; one thread issues
    auto issue = [&](uint64_t i) {
        const uint32_t k = (uint32_t)(i / nfr), j = (uint32_t)(i % nfr);
        const uint32_t px0 = (sweep + k * nsweeps) * SW_TILE_PX;
        const uint32_t tpx = npix - px0 < SW_TILE_PX ? npix - px0 : SW_TILE_PX;
        const uint32_t bytes = (tpx * PB) & ~15u;                      // whole 16 B units inside the frame
        const uint8_t* frame = j == 0 ? pairs[0].prev : pairs[j - 1].curr;
        uint64_t* bar = &full[i % SW_STAGES];
        mbar_expect_tx(bar, bytes);                                    // also the one arrival: a 0-byte load completes at once
        if (bytes) bulk_g2s(ring + (i % SW_STAGES) * SLOT, frame + (size_t)px0 * PB, bytes, bar);
    };
    if (tid == 0)
        for (uint64_t i = 0; i < SW_STAGES - 1 && i < total; i++) issue(i);

    uint32_t k = 0, j = 0;                                             // tile and frame of load i
    for (uint64_t i = 0; i < total; i++) {
        mbar_wait(&full[i % SW_STAGES], (uint32_t)(i / SW_STAGES) & 1u);
        if (j > 0) {                                                   // pair j-1: frame j-1 (previous slot) against frame j
            const PairJob pj = pairs[j - 1];
            const uint32_t w = (sweep + k * nsweeps) * SW_THREADS + tid;
            uint32_t m = 0, r = 0;
            if (w < nwords) {
                const uint32_t px0 = w << 5;
                if (px0 + 32u <= npix)
                    threshold_word<PB, S, GRAY>(ring + ((i - 1) % SW_STAGES) * SLOT + tid * 32u * PB,
                                                ring + (i % SW_STAGES) * SLOT + tid * 32u * PB, true, t, m, r);
                else
                    threshold_word_tail<PB, S, GRAY>(pj.prev + (size_t)px0 * PB, pj.curr + (size_t)px0 * PB, npix - px0, t, m, r);
                pj.mask[w] = m;
            }
            const uint32_t co = __reduce_add_sync(0xffffffffu, __popc(m)), cr = __reduce_add_sync(0xffffffffu, __popc(r));
            if (lane == 0) { s_cnt[i & 1][warp][0] = co; s_cnt[i & 1][warp][1] = cr; }
        }
        // the previous slot has been read by every thread of the sweep
        asm volatile("bar.sync %0, %1;" ::"r"(g + 1u), "n"(SW_THREADS) : "memory");
        if (tid == 0) {
            if (j > 0) {
                uint32_t to = 0, tr = 0;
#pragma unroll
                for (int q = 0; q < NWARP; q++) { to += s_cnt[i & 1][q][0]; tr += s_cnt[i & 1][q][1]; }
                if (to) atomicAdd(ones + j - 1, to);
                if (tr) atomicAdd(resid + j - 1, tr);
            }
            if (i + SW_STAGES - 1 < total) { fence_proxy_async(); issue(i + SW_STAGES - 1); }   // into the slot just freed
        }
        if (++j == nfr) { j = 0; k++; }
    }
}

// ------------------------------------------------------------------------------------------
// K1 (TMA variant): persistent CTAs, 4-stage mbarrier ring, one elected thread issues
// cp.async.bulk copies of a 2 x 12 KB tile (prev, curr); for 8-bit YUV444 each lane reads
// four pixels (three words, bank-conflict free) and runs the same byte-SIMD as above; the
// per-lane nibbles are OR-reduced over 8-lane groups (REDUX) into mask words.
// ------------------------------------------------------------------------------------------
constexpr int TMA_STAGES = 4;
constexpr int TMA_TILE_BYTES = 12288;                  // per frame per stage (4096 px at 3 B/px)
constexpr int TMA_THREADS = 256;

template <int PB, int S>
__global__ void __launch_bounds__(TMA_THREADS) k_threshold_tma(const PairJob* __restrict__ pairs, int F, uint32_t npix,
                                                               int thr, int any_mode, uint32_t* __restrict__ ones,
                                                               uint32_t* __restrict__ resid) {
    constexpr uint32_t TP = TMA_TILE_BYTES / PB;       // pixels per tile (multiple of 32*8)
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t full[TMA_STAGES];
    uint8_t* bufA = smem;                               // [STAGES][TILE]
    uint8_t* bufB = smem + TMA_STAGES * TMA_TILE_BYTES;
    const uint32_t tiles_per_frame = npix / TP;         // full tiles only (bulk copies need 16 B multiples)
    const uint64_t total = (uint64_t)tiles_per_frame * (uint64_t)F;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int NWARP = TMA_THREADS / 32;
    constexpr uint32_t WPW = TP / 32 / NWARP;           // mask words per warp per tile
    const uint32_t thr4 = (uint32_t)(thr < 0 ? 0 : (thr > 254 ? 254 : thr)) * 0x01010101u;
    const uint32_t gt_or = thr < 0 ? 0xffffffffu : 0u, gt_and = thr > 254 ? 0u : 0xffffffffu;
    const uint32_t any_mask = any_mode ? 0xfu : 0u;

    if (threadIdx.x == 0) {
        for (int s = 0; s < TMA_STAGES; s++) mbar_init(&full[s], 1);
        fence_mbar_init();
    }
    __syncthreads();

    auto issue = [&](uint64_t t, int slot) {
        const uint32_t f = (uint32_t)(t / tiles_per_frame), ti = (uint32_t)(t % tiles_per_frame);
        const PairJob pj = pairs[f];
        mbar_expect_tx(&full[slot], 2 * TMA_TILE_BYTES);
        bulk_g2s(bufA + slot * TMA_TILE_BYTES, pj.prev + (size_t)ti * TMA_TILE_BYTES, TMA_TILE_BYTES, &full[slot]);
        bulk_g2s(bufB + slot * TMA_TILE_BYTES, pj.curr + (size_t)ti * TMA_TILE_BYTES, TMA_TILE_BYTES, &full[slot]);
    };

    // prologue
    uint64_t t0 = blockIdx.x;
    if (threadIdx.x == 0) {
        for (int s = 0; s < TMA_STAGES - 1; s++) {
            uint64_t t = t0 + (uint64_t)s * gridDim.x;
            if (t < total) issue(t, s);
        }
    }
    uint32_t it = 0, acc_o = 0, acc_r = 0, acc_f = 0xffffffffu;     // per-thread counts of the current frame
    auto flush_counts = [&]() {
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            acc_o += __shfl_xor_sync(0xffffffffu, acc_o, d);
            acc_r += __shfl_xor_sync(0xffffffffu, acc_r, d);
        }
        if (lane == 0 && acc_f != 0xffffffffu) {
            if (acc_o) atomicAdd(ones + acc_f, acc_o);
            if (acc_r) atomicAdd(resid + acc_f, acc_r);
        }
        acc_o = 0; acc_r = 0;
    };
    for (uint64_t t = t0; t < total; t += gridDim.x, it++) {
        const int slot = it % TMA_STAGES;
        const uint32_t parity = (it / TMA_STAGES) & 1u;
        if (threadIdx.x == 0) {                         // refill the slot freed by the previous iteration
            uint64_t tn = t + (uint64_t)(TMA_STAGES - 1) * gridDim.x;
            if (tn < total) { fence_proxy_async(); issue(tn, (it + TMA_STAGES - 1) % TMA_STAGES); }
        }
        const uint32_t f = (uint32_t)(t / tiles_per_frame), ti = (uint32_t)(t % tiles_per_frame);
        if (f != acc_f) { flush_counts(); acc_f = f; }  // warp-uniform
        mbar_wait(&full[slot], parity);
        const uint8_t* a = bufA + slot * TMA_TILE_BYTES;
        const uint8_t* b = bufB + slot * TMA_TILE_BYTES;
        uint32_t* mask_out = pairs[f].mask + (size_t)ti * (TP / 32) + warp * WPW;
        if (PB == 3 && S == 1) {
            const uint32_t* a32 = reinterpret_cast<const uint32_t*>(a) + (size_t)warp * WPW * 24;   // 32 px = 24 words
            const uint32_t* b32 = reinterpret_cast<const uint32_t*>(b) + (size_t)warp * WPW * 24;
#pragma unroll 2
            for (uint32_t k = 0; k < WPW / 4; k++) {      // 128 pixels (4 mask words) per iteration
                const uint32_t o = (k * 32u + lane) * 3u;
                uint32_t nm, nd;
                yuv8_group4(a32[o], a32[o + 1], a32[o + 2], b32[o], b32[o + 1], b32[o + 2], thr4, gt_or, gt_and, nm, nd);
                nm |= nd & any_mask;
                const uint32_t nr = nd & ~nm;
                const uint32_t grp = 0xffu << (lane & 24);
                const uint32_t wm = __reduce_or_sync(grp, nm << (4 * (lane & 7)));
                const uint32_t wr = __reduce_or_sync(grp, nr << (4 * (lane & 7)));
                if ((lane & 7) == 0) { mask_out[k * 4 + (lane >> 3)] = wm; acc_o += __popc(wm); acc_r += __popc(wr); }
            }
        } else {
            uint32_t myword = 0;
#pragma unroll 4
            for (uint32_t k = 0; k < WPW; k++) {
                const uint32_t px = (warp * WPW + k) * 32u + lane;
                const uint8_t* pa = a + px * PB;
                const uint8_t* pb = b + px * PB;
                uint32_t ya, yb, anyd = 0;
                if (S == 1) { ya = pa[0]; yb = pb[0]; }
                else { ya = *reinterpret_cast<const uint16_t*>(pa); yb = *reinterpret_cast<const uint16_t*>(pb); }
#pragma unroll
                for (int q = 0; q < PB; q += S) {
                    if (S == 1) anyd |= (uint32_t)(pa[q] ^ pb[q]);
                    else anyd |= (uint32_t)(*reinterpret_cast<const uint16_t*>(pa + q) ^ *reinterpret_cast<const uint16_t*>(pb + q));
                }
                const bool bit = (absdiff_sample<PB, S>(ya, yb) > thr) || (any_mode && anyd != 0u);
                const uint32_t bm = __ballot_sync(0xffffffffu, bit);
                const uint32_t br = __ballot_sync(0xffffffffu, (!bit) && anyd != 0u);
                if (lane == (int)k) myword = bm;
                if (lane == 0) { acc_o += __popc(bm); acc_r += __popc(br); }
            }
            if (lane < (int)WPW) mask_out[lane] = myword;
        }
        __syncthreads();                                // slot may be refilled next iteration
    }
    flush_counts();
}

// remainder of each frame after the last full TMA tile: same maths with guarded scalar loads
template <int PB, int S>
__global__ void __launch_bounds__(256) k_threshold_tail(const PairJob* __restrict__ pairs, uint32_t npix, uint32_t px_begin,
                                                        int thr, int any_mode, uint32_t* __restrict__ ones, uint32_t* __restrict__ resid) {
    const PairJob pj = pairs[blockIdx.y];
    const uint32_t w0 = px_begin >> 5, nwords = (npix + 31u) >> 5;
    for (uint32_t w = w0 + blockIdx.x * blockDim.x + threadIdx.x; w < nwords; w += gridDim.x * blockDim.x) {
        uint32_t m = 0, r = 0;
        for (uint32_t k = 0; k < 32u && (w << 5) + k < npix; k++) {
            const uint8_t* a = pj.prev + (size_t)((w << 5) + k) * PB;
            const uint8_t* b = pj.curr + (size_t)((w << 5) + k) * PB;
            uint32_t ya = a[0], yb = b[0];
            if (S == 2) { ya |= (uint32_t)a[1] << 8; yb |= (uint32_t)b[1] << 8; }
            uint32_t anyd = 0;
            for (int q = 0; q < PB; q++) anyd |= (uint32_t)(a[q] ^ b[q]);
            const uint32_t bit = ((absdiff_sample<PB, S>(ya, yb) > thr) || (any_mode && anyd != 0u)) ? 1u : 0u;
            m |= bit << k;
            r |= ((anyd != 0u && bit == 0u) ? 1u : 0u) << k;
        }
        pj.mask[w] = m;
        if (m) atomicAdd(ones + blockIdx.y, __popc(m));
        if (r) atomicAdd(resid + blockIdx.y, __popc(r));
    }
}
