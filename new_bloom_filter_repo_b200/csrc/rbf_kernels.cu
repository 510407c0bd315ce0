// rbf_kernels.cu -- hand-written sm_90a kernels of the rational-Bloom hot path.
//
//   K1  k_threshold      |Y_prev - Y_curr| > thr  -> packed mask + ones count      (ivc:788-808, ivc:211)
//       k_threshold_sweep  the same over a chain of pairs, every frame read once
//   K2  k_insert         insert every set position into the frame's Bloom filter    (ivc:235-237, ivc:99-114)
//   K3  k_query          Bloom test of ALL n positions -> pass mask                 (ivc:245-253, ivc:116-138)
//   K3b k_witness        ordered witness = mask bits at passing positions           (ivc:253)
//   K4b k_expand         decode: out[i] = witness[rank(i)] for passing i            (ivc:299-304)
//   K4c k_apply_sweep    a group's decoded masks applied along the frame chain      (ivc:849-909)
//   K5  k_motion_search  16 x 16 block motion search, +-16 px (value_coding "motion")
//       k_apply_motion   a motion-compensated residual pair of a decoded group
//   N4  k_deflate_segments / k_deflate_concat   zlib streams of host or device buffers (rbf_deflate.cuh)
//       k_inflate_scan / k_inflate_segments     inflate of those streams, segment by segment (rbf_inflate.cuh)
//
// The Bloom bit array of the frame being queried is staged into shared memory with
// cp.async.bulk (TMA bulk copy, mbarrier complete_tx); whatever exceeds the 227 KB of a
// CTA is probed through L2.  Integer hashing / bit tests only: no tensor cores.
//
// One translation unit: this file holds the PTX helpers and the launchers; the kernels live in
// rbf_k1_threshold.cuh, rbf_k2_insert.cuh, rbf_k3_query.cuh, rbf_k3b_witness.cuh, rbf_aux_kernels.cuh, rbf_deflate.cuh, rbf_k4c_apply.cuh and rbf_motion.cuh.
#include <cuda_runtime.h>
#include <stdint.h>

#include <mutex>
#include <type_traits>

#include "rbf_kernels.cuh"

namespace rbf {

// ------------------------------------------------------------------------------------------
// PTX helpers: mbarrier + bulk async copy (TMA), cache-hinted loads
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!ok);
}
__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {   // read-once frame data: do not pollute L1
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

// fire-and-forget bit set in a global bit array (RED.OR, no return value -> no round trip to wait for)
__device__ __forceinline__ void red_or_global(uint32_t* addr, uint32_t v) {
    asm volatile("red.global.or.b32 [%0], %1;" ::"l"(addr), "r"(v) : "memory");
}

// ------------------------------------------------------------------------------------------
// 100-bit helpers (a "century" of positions)
// ------------------------------------------------------------------------------------------
struct Bits128 {
    uint64_t lo, hi;
};

// bits [100c, 100c+nvalid) of a naturally packed bit array (buffer padded by >= 16 B)
__device__ __forceinline__ Bits128 load_bits100(const uint32_t* __restrict__ base, uint32_t c, uint32_t nvalid) {
    uint64_t off = 100ull * c;
    uint32_t w = (uint32_t)(off >> 5), sh = (uint32_t)off & 31u;
    uint32_t a0 = __ldg(base + w), a1 = __ldg(base + w + 1), a2 = __ldg(base + w + 2), a3 = __ldg(base + w + 3);
    uint32_t b0 = __funnelshift_r(a0, a1, sh), b1 = __funnelshift_r(a1, a2, sh), b2 = __funnelshift_r(a2, a3, sh),
             b3 = a3 >> sh;
    Bits128 r;
    r.lo = (uint64_t)b0 | ((uint64_t)b1 << 32);
    r.hi = (uint64_t)b2 | ((uint64_t)b3 << 32);
    if (nvalid >= 64) {
        r.hi &= (1ull << (nvalid - 64)) - 1ull;      // nvalid <= 100
    } else {
        r.hi = 0;
        r.lo &= (1ull << nvalid) - 1ull;              // nvalid < 64
    }
    return r;
}

// OR a (<=128-bit) value into a zero-initialised bit stream at an arbitrary bit offset
__device__ __forceinline__ void or_bits128(uint32_t* __restrict__ W, uint64_t bitoff, uint64_t lo, uint64_t hi) {
    uint32_t w = (uint32_t)(bitoff >> 5), sh = (uint32_t)bitoff & 31u;
    uint32_t s0 = (uint32_t)lo, s1 = (uint32_t)(lo >> 32), s2 = (uint32_t)hi, s3 = (uint32_t)(hi >> 32);
    uint32_t o0 = s0 << sh, o1 = __funnelshift_l(s0, s1, sh), o2 = __funnelshift_l(s1, s2, sh),
             o3 = __funnelshift_l(s2, s3, sh), o4 = __funnelshift_l(s3, 0u, sh);
    if (o0) red_or_global(W + w, o0);
    if (o1) red_or_global(W + w + 1, o1);
    if (o2) red_or_global(W + w + 2, o2);
    if (o3) red_or_global(W + w + 3, o3);
    if (o4) red_or_global(W + w + 4, o4);
}

#include "rbf_k1_threshold.cuh"
#include "rbf_k2_insert.cuh"
#include "rbf_k3_query.cuh"
#include "rbf_k3b_witness.cuh"
#include "rbf_aux_kernels.cuh"
#include "rbf_deflate.cuh"
#include "rbf_inflate.cuh"
#include "rbf_k4c_apply.cuh"
#include "rbf_motion.cuh"

// ------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------
// the launch status of the `kernels` kernels just enqueued, which are added to the context's counter
static cudaError_t counted(LaunchCfg& L, int kernels = 1) {
    L.launches += kernels;
    return cudaGetLastError();
}

// The four frame formats a stream can have (1 or 3 channels of 1- or 2-byte samples, fixed by rbf_stream_create) as compile-time
// (pixel bytes, sample bytes): f(ic<PB>, ic<S>) launches that format's kernel instances.  Any other format launches nothing.
template <int N> using ic = std::integral_constant<int, N>;
template <class F> static cudaError_t by_format(uint32_t pix_bytes, uint32_t sample_bytes, F&& f) {
    if (pix_bytes == 1 && sample_bytes == 1) return f(ic<1>{}, ic<1>{});
    if (pix_bytes == 3 && sample_bytes == 1) return f(ic<3>{}, ic<1>{});
    if (pix_bytes == 2 && sample_bytes == 2) return f(ic<2>{}, ic<2>{});
    if (pix_bytes == 6 && sample_bytes == 2) return f(ic<6>{}, ic<2>{});
    return cudaErrorInvalidValue;
}

// K1 over a chain of F >= 2 pairs: persistent sweeps, each of the same number of tiles (or one fewer).
// sms == 0: the whole GPU, one sweep per CTA and at most ctas_per_sm CTAs per SM.
// sms > 0: one wide CTA on each of `sms` SMs, with as many sweeps as fit in its shared memory (SW_MAX_SWEEPS at most).  Its
// shared memory, padded to more than half an SM's 228 KB, keeps a second K1 CTA and any K2 CTA (195 KB) off the SM: the grid
// lands on exactly that many SMs, and K2 runs beside it on the others.
template <int PB, int S, bool GRAY>
static cudaError_t launch_threshold_sweep_t(LaunchCfg& L, const PairJob* d_pairs, int F, uint32_t npix, int thr, int any_mode,
                                            uint32_t* d_ones, uint32_t* d_resid, int ctas_per_sm, int sms, cudaStream_t st) {
    constexpr int sweep_smem = (int)sw_sweep_bytes<PB>();
    constexpr int max_smem = 232448;                                   // opt-in shared memory of one CTA on sm_90
    constexpr int wide = max_smem / sweep_smem < SW_MAX_SWEEPS ? max_smem / sweep_smem : SW_MAX_SWEEPS;
    constexpr int wide_smem = wide * sweep_smem > max_smem / 2 + 1024 ? wide * sweep_smem : max_smem / 2 + 1024;
    cudaError_t e = cudaFuncSetAttribute(k_threshold_sweep<PB, S, GRAY>, cudaFuncAttributeMaxDynamicSharedMemorySize, wide_smem);
    if (e != cudaSuccess) return e;
    const uint32_t ntiles = (npix + SW_TILE_PX - 1u) / SW_TILE_PX;
    uint32_t grid, sweeps = 1;
    int smem = sweep_smem;
    if (sms > 0) {
        sweeps = (uint32_t)wide;
        smem = wide_smem;
        grid = (ntiles + sweeps - 1u) / sweeps;
        if (grid > (uint32_t)sms) grid = (uint32_t)sms;
    } else {
        int per_sm = 1;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_threshold_sweep<PB, S, GRAY>, SW_THREADS, (size_t)sweep_smem);
        if (e != cudaSuccess) return e;
        const int cap = ctas_per_sm > 0 ? ctas_per_sm : 32;
        if (per_sm > cap) per_sm = cap;
        if (per_sm < 1) per_sm = 1;
        const uint32_t slots = (uint32_t)(L.sm_count > 0 ? L.sm_count : 1) * (uint32_t)per_sm;
        const uint32_t rounds = (ntiles + slots - 1u) / slots;
        grid = (ntiles + rounds - 1u) / rounds;
    }
    k_threshold_sweep<PB, S, GRAY><<<grid, SW_THREADS * sweeps, smem, st>>>(d_pairs, (uint32_t)F, npix, thr, any_mode, d_ones, d_resid);
    return counted(L);
}

// GRAY: the mask is taken on cv2.COLOR_BGR2GRAY of the three samples instead of on sample 0 (ivc:792-795); no TMA kernel for it
template <int PB, int S, bool GRAY>
static cudaError_t launch_threshold_t(LaunchCfg& L, const PairJob* d_pairs, int F, uint32_t npix, int thr, int any_mode, uint32_t* d_ones,
                                      uint32_t* d_resid, bool chain, int ctas_per_sm, int sms, cudaStream_t st) {
    const uint32_t nwords = (npix + 31u) >> 5;
    constexpr uint32_t TP = TMA_TILE_BYTES / PB;
    if constexpr (!GRAY) {
        if (L.k1_variant == 1 && npix >= TP && (TP / 32u / (TMA_THREADS / 32)) <= 32u) {
            const int smem = 2 * TMA_STAGES * TMA_TILE_BYTES;
            cudaError_t e = cudaFuncSetAttribute(k_threshold_tma<PB, S>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
            if (e != cudaSuccess) return e;
            const uint64_t total = (uint64_t)(npix / TP) * (uint64_t)F;
            int grid = (int)((total < (uint64_t)(2 * L.sm_count)) ? total : (uint64_t)(2 * L.sm_count));
            k_threshold_tma<PB, S><<<grid, TMA_THREADS, smem, st>>>(d_pairs, F, npix, thr, any_mode, d_ones, d_resid);
            e = counted(L);
            if (e != cudaSuccess) return e;
            const uint32_t px_begin = (npix / TP) * TP;
            if (px_begin < npix) {
                const uint32_t tail_words = nwords - (px_begin >> 5);
                dim3 g((tail_words + 255u) / 256u, (unsigned)F);
                k_threshold_tail<PB, S><<<g, 256, 0, st>>>(d_pairs, npix, px_begin, thr, any_mode, d_ones, d_resid);
                return counted(L);
            }
            return cudaSuccess;
        }
    }
    if (chain && F >= 2) return launch_threshold_sweep_t<PB, S, GRAY>(L, d_pairs, F, npix, thr, any_mode, d_ones, d_resid, ctas_per_sm, sms, st);
    uint32_t bx = (nwords + 255u) / 256u;
    const uint32_t cap = (uint32_t)(L.sm_count * (ctas_per_sm > 0 ? ctas_per_sm : 32));
    if ((uint64_t)bx * (uint64_t)F > cap) { bx = (cap + (uint32_t)F - 1u) / (uint32_t)F; if (bx < 1u) bx = 1u; }
    dim3 grid(bx, (unsigned)F);
    const int smem = K1_STAGE_BYTES_PER_PB * PB;
    cudaError_t e = cudaFuncSetAttribute(k_threshold<PB, S, GRAY>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    k_threshold<PB, S, GRAY><<<grid, K1_THREADS, smem, st>>>(d_pairs, npix, thr, any_mode, d_ones, d_resid);
    return counted(L);
}

cudaError_t launch_threshold(LaunchCfg& L, const PairJob* d_pairs, int F, uint32_t npix, int channels, int sample_bytes, int thr_int,
                             int any_mode, int gray_mode, uint32_t* d_ones, uint32_t* d_resid, bool chain, int sms, cudaStream_t st) {
    if (F <= 0 || npix == 0) return cudaSuccess;
    return by_format((uint32_t)(channels * sample_bytes), (uint32_t)sample_bytes, [&](auto PBc, auto Sc) -> cudaError_t {
        constexpr int PB = decltype(PBc)::value, S = decltype(Sc)::value;
        const int cap = L.k1_ctas_per_sm;
        if (!gray_mode) return launch_threshold_t<PB, S, false>(L, d_pairs, F, npix, thr_int, any_mode, d_ones, d_resid, chain, cap, sms, st);
        if constexpr (PB == 3 * S) return launch_threshold_t<PB, S, true>(L, d_pairs, F, npix, thr_int, any_mode, d_ones, d_resid, chain, cap, sms, st);
        else return cudaErrorInvalidValue;                        // gray needs three channels
    });
}

static cudaLaunchConfig_t insert_cluster_config(uint32_t cs, uint32_t units, cudaStream_t st, cudaLaunchAttribute* attr) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(cs, units);
    cfg.blockDim = dim3(K2_THREADS);
    cfg.dynamicSmemBytes = K2_SMEM_BYTES;
    cfg.stream = st;
    attr->id = cudaLaunchAttributeClusterDimension;
    attr->val.clusterDim.x = cs; attr->val.clusterDim.y = 1; attr->val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cfg;
}

// resident clusters of cs CTAs; 0 means the shape cannot be scheduled
static cudaError_t insert_cluster_occupancy(uint32_t cs, int* clusters) {
    cudaError_t e = cudaFuncSetAttribute(k_insert_cluster, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)K2_SMEM_BYTES);
    if (e != cudaSuccess) return e;
    cudaLaunchAttribute attr;
    const cudaLaunchConfig_t cfg = insert_cluster_config(cs, 1u, nullptr, &attr);
    return cudaOccupancyMaxActiveClusters(clusters, k_insert_cluster, &cfg);
}

cudaError_t launch_insert(LaunchCfg& L, const FrameJob* d_jobs, int F, uint32_t max_centuries, uint32_t max_l_bits, int sms, cudaStream_t st) {
    if (F <= 0 || max_centuries == 0) return cudaSuccess;
    const uint32_t words = (uint32_t)(((uint64_t)max_l_bits + 31u) >> 5);
    if (L.insert_variant >= 1 && words > 2u * K2_MAX_CS * K2_WORDS) {   // less than half of the array would be on chip: RED.OR into L2
        const uint32_t nslab = (max_centuries + 31u) / 32u;
        dim3 grid((nslab + I2_WARPS - 1) / I2_WARPS, (unsigned)F);
        k_insert2<<<grid, I2_WARPS * 32, 0, st>>>(d_jobs);
        return counted(L);
    }
    if (L.insert_variant >= 1) {                          // dense, warp-compacted insert into (cluster) shared memory
        uint32_t cs = (words + K2_WORDS - 1u) / K2_WORDS;
        if (cs < 1u) cs = 1u;
        if (cs > (uint32_t)K2_MAX_CS) cs = K2_MAX_CS;    // the rest of the array is set with RED.OR in L2
        // Full waves of resident clusters take one frame each; the frames of the last, partial wave (all of them when F is small)
        // get R copies each so that they still fill the `sms` SMs K2 has, with at least K2_WARPS slabs per CTA.
        if (L.k2_clusters[cs] == 0) {                       // first launch of this shape: measure it once, and refuse it if it does not fit
            cudaError_t e = insert_cluster_occupancy(cs, &L.k2_clusters[cs]);
            if (e != cudaSuccess) return e;
            if (L.k2_clusters[cs] < 1) { L.k2_clusters[cs] = 0; return cudaErrorInvalidConfiguration; }
        }
        uint32_t slots = (uint32_t)((int64_t)L.k2_clusters[cs] * (sms < L.sm_count ? sms : L.sm_count) / L.sm_count);
        if (slots < 1u) slots = 1u;
        const uint32_t full = (uint32_t)F / slots * slots, rem = (uint32_t)F - full;
        const uint32_t nslab = (max_centuries + 31u) / 32u;
        const uint32_t useful = (nslab + cs * K2_WARPS - 1u) / (cs * K2_WARPS);
        uint32_t copies = rem ? slots / rem : 1u;
        if (copies > useful) copies = useful;
        if (copies < 1u) copies = 1u;
        cudaLaunchAttribute attr;
        const cudaLaunchConfig_t cfg = insert_cluster_config(cs, full + rem * copies, st, &attr);
        const cudaError_t e = cudaLaunchKernelEx(&cfg, k_insert_cluster, d_jobs, full, copies);
        return e != cudaSuccess ? e : counted(L);
    }
    uint32_t bx = (max_centuries + 255u) / 256u;
    const uint32_t cap = (uint32_t)(L.sm_count * 16);
    if ((uint64_t)bx * (uint64_t)F > cap) { bx = (cap + (uint32_t)F - 1u) / (uint32_t)F; if (bx < 1u) bx = 1u; }
    dim3 grid(bx, (unsigned)F);
    k_insert<<<grid, 256, 0, st>>>(d_jobs);
    return counted(L);
}


int query_max_smem_bytes() { return 232448 - 1024; }    // 227 KB opt-in minus static shared memory + slack

template <bool HYBRID>
static cudaError_t launch_query2_t(LaunchCfg& L, const FrameJob* d_jobs, const uint32_t* d_cent_prefix, int F, uint32_t total_centuries,
                                   int smem, cudaStream_t st) {
    cudaError_t e = cudaFuncSetAttribute(k_query2<HYBRID>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    uint32_t grid = (uint32_t)L.sm_count;
    const uint32_t max_useful = (total_centuries + Q2_THREADS - 1) / Q2_THREADS;
    if (grid > max_useful) grid = max_useful;
    if (grid < 1u) grid = 1u;
    k_query2<HYBRID><<<grid, Q2_THREADS, smem, st>>>(d_jobs, d_cent_prefix, F, (uint32_t)((smem - Q2_WARPS * Q2_WARP_WORDS * 4) / 4));
    return counted(L);
}

// A kernel's dynamic shared memory limit (cudaFuncSetAttribute) is one value for the whole process, and the query sets it to what
// each launch needs, which depends on l.  Contexts driven from different host threads must not interleave their set and launch: a
// thread that lowers the limit in between makes the other's launch fail with "too many resources requested for launch".
static std::mutex g_query_smem_attr;

// variant: 0 per-lane kernel; 1 staged rings; 5 decade tiles (half-decade tiles for 2^23 < m <= 2^24, rings beyond); 6 half-decade
// tiles for every m <= 2^24.  (2, 3 and 4 selected earlier kernels that were measured slower and removed; the values still
// select the current default.)
cudaError_t launch_query(LaunchCfg& L, const FrameJob* d_jobs, const uint32_t* d_cent_prefix, int F, uint32_t total_centuries,
                         uint32_t max_l_bits, cudaStream_t st) {
    if (F <= 0 || total_centuries == 0) return cudaSuccess;
    std::lock_guard<std::mutex> attr_and_launch(g_query_smem_attr);
    int variant = L.query_variant, tile_warps = L.query_warps;
    if (tile_warps < 4 || tile_warps > Q4_WARPS) tile_warps = 0;                       // 0: the tile width's default
    int cap = L.query_smem_cap & ~15;
    if (cap > query_max_smem_bytes()) cap = query_max_smem_bytes() & ~15;
    const uint32_t need_words = (((max_l_bits + 31u) >> 5) + 3u) & ~3u;
    if (variant >= 2 && variant <= 4) variant = 5;
    if (variant >= 5 && max_l_bits <= (1u << 24)) {       // decade tiles (full stage-B batches with carry)
        const bool half = (variant == 6) || max_l_bits > (1u << 23);      // half-decade tiles: 24-bit record indices
        if (tile_warps == 0) tile_warps = half ? Q4_WARPS : Q4_FULL_TILE_WARPS;
        const int qbytes = 4 * (Q4_TABLE_WORDS + tile_warps * (half ? Q4Cfg<5>::WARP_WORDS : Q4Cfg<10>::WARP_WORDS));
        if (cap < qbytes + 1024) cap = qbytes + 1024;
        const int bits_cap = cap - qbytes;
        const bool fits = (size_t)need_words * 4 <= (size_t)bits_cap;
        const int smem = qbytes + (fits ? (int)(need_words * 4 < 16 ? 16 : need_words * 4) : bits_cap);
        uint32_t grid = (uint32_t)L.sm_count;
        const uint32_t max_useful = (total_centuries + 32u * tile_warps - 1) / (32u * tile_warps);
        if (grid > max_useful) grid = max_useful;
        if (grid < 1u) grid = 1u;
        const uint32_t words_cap = (uint32_t)((smem - qbytes) / 4);
#define RBF_LAUNCH_Q4(PM, TY)                                                                                         \
    do {                                                                                                              \
        cudaError_t e = cudaFuncSetAttribute(k_query4<PM, TY>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);    \
        if (e != cudaSuccess) return e;                                                                               \
        k_query4<PM, TY><<<grid, 32 * tile_warps, smem, st>>>(d_jobs, d_cent_prefix, F, words_cap);                        \
    } while (0)
        if (fits) { if (half) RBF_LAUNCH_Q4(0, 5); else RBF_LAUNCH_Q4(0, 10); }
        else      { if (half) RBF_LAUNCH_Q4(1, 5); else RBF_LAUNCH_Q4(1, 10); }
#undef RBF_LAUNCH_Q4
        return counted(L);
    }
    if (variant >= 1) {                                   // staged rings (also the home of filters beyond 2^24 bits)
        const int qbytes = Q2_WARPS * Q2_WARP_WORDS * 4;
        if (cap < qbytes + 1024) cap = qbytes + 1024;
        const int bits_cap = cap - qbytes;
        const bool fits = (size_t)need_words * 4 <= (size_t)bits_cap;
        const int smem = qbytes + (fits ? (int)(need_words * 4 < 16 ? 16 : need_words * 4) : bits_cap);
        return !fits ? launch_query2_t<true>(L, d_jobs, d_cent_prefix, F, total_centuries, smem, st)
                     : launch_query2_t<false>(L, d_jobs, d_cent_prefix, F, total_centuries, smem, st);
    }
    int smem = (size_t)need_words * 4 > (size_t)cap ? cap : (int)(need_words * 4);
    if (smem < 16) smem = 16;
    cudaError_t e = cudaFuncSetAttribute(k_query, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    int per_sm = 1;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_query, QT, (size_t)smem);
    if (e != cudaSuccess) return e;
    if (per_sm < 1) per_sm = 1;
    uint32_t grid = (uint32_t)(L.sm_count * per_sm);
    const uint32_t max_useful = (total_centuries + QT - 1) / QT;
    if (grid > max_useful) grid = max_useful;
    if (grid < 1u) grid = 1u;
    k_query<<<grid, QT, smem, st>>>(d_jobs, d_cent_prefix, F, (uint32_t)(smem / 4));
    return counted(L);
}

static uint32_t witness_chunks(int F, uint32_t max_centuries, int sm_count) {
    uint32_t ch = (uint32_t)((16 * sm_count + F - 1) / F);            // >= 8 waves of the two 1024-thread CTAs an SM holds: with few waves
                                                                      // the ragged last wave costs a large share of K3b
    const uint32_t by_size = max_centuries / 4096u;                   // at least 4096 centuries (4 rounds) per chunk
    if (ch > by_size) ch = by_size;
    if (ch > 32u) ch = 32u;
    if (ch < 1u) ch = 1u;
    return ch;
}
// K3b: d_scratch holds F*32 uint32 (pass counts per chunk)
cudaError_t launch_witness(LaunchCfg& L, const FrameJob* d_jobs, int F, uint32_t max_centuries, uint32_t* d_scratch, uint32_t* d_wlen,
                           cudaStream_t st) {
    if (F <= 0) return cudaSuccess;
    const uint32_t ch = witness_chunks(F, max_centuries, L.sm_count);
    if (ch > 1u) k_pass_count<<<dim3(ch, (unsigned)F), 256, 0, st>>>(d_jobs, ch, d_scratch);
    k_witness<<<dim3(ch, (unsigned)F), 1024, 0, st>>>(d_jobs, ch, d_scratch, d_wlen);
    k_finalize<<<dim3(32, (unsigned)F), 256, 0, st>>>(d_jobs, d_wlen);
    return counted(L, ch > 1u ? 3 : 2);
}
cudaError_t launch_expand(LaunchCfg& L, const FrameJob* d_jobs, int F, uint32_t max_centuries, uint32_t* d_scratch, uint32_t* d_consumed,
                          cudaStream_t st) {
    if (F <= 0) return cudaSuccess;
    const uint32_t ch = witness_chunks(F, max_centuries, L.sm_count);
    if (ch > 1u) k_pass_count<<<dim3(ch, (unsigned)F), 256, 0, st>>>(d_jobs, ch, d_scratch);
    k_expand<<<dim3(ch, (unsigned)F), 1024, 0, st>>>(d_jobs, ch, d_scratch, d_consumed);
    return counted(L, ch > 1u ? 2 : 1);
}
static inline unsigned grid_for(size_t n, unsigned block, int sm_count) {
    size_t g = (n + block - 1) / block;
    const size_t cap = (size_t)(sm_count > 0 ? sm_count : 1) * 16u;    // 16 CTAs per SM; the kernels stride over the rest
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (unsigned)g;
}
uint32_t gather_chunks(uint32_t npix) {
    uint32_t ch = ((npix + 31u) >> 5) / 4096u;             // >= 4 rounds of 1024 threads per chunk
    if (ch > (uint32_t)GS_MAX_CHUNKS) ch = GS_MAX_CHUNKS;
    return ch < 1u ? 1u : ch;
}
// d_counts: F * gather_chunks(npix) uint32 of scratch
cudaError_t launch_gather(LaunchCfg& L, const GatherJob* d_jobs, int F, uint32_t npix, uint32_t pix_bytes, uint32_t sample_bytes,
                          int kind, uint32_t* d_counts, cudaStream_t st) {
    if (F <= 0) return cudaSuccess;
    return by_format(pix_bytes, sample_bytes, [&](auto PBc, auto Sc) -> cudaError_t {
        constexpr int PB = decltype(PBc)::value, S = decltype(Sc)::value;
        const uint32_t ch = gather_chunks(npix);
        const dim3 grid(ch, (unsigned)F);
        k_mask_chunk_count<<<grid, 256, 0, st>>>(d_jobs, ch, d_counts);
        if (kind == 0) k_gather<PB, 0, false><<<grid, 1024, 0, st>>>(d_jobs, ch, d_counts);
        else if (kind == 1) k_gather<PB, S, false><<<grid, 1024, 0, st>>>(d_jobs, ch, d_counts);
        else k_gather<PB, S, true><<<grid, 1024, 0, st>>>(d_jobs, ch, d_counts);
        return counted(L, 2);
    });
}
cudaError_t launch_raw_masks(LaunchCfg& L, const FrameJob* d_jobs, int F, uint32_t npix, cudaStream_t st) {
    if (F <= 0 || npix == 0) return cudaSuccess;
    unsigned gx = (((npix + 31u) >> 5) + 255u) / 256u;
    if (gx > 64u) gx = 64u;
    k_raw_masks<<<dim3(gx, (unsigned)F), 256, 0, st>>>(d_jobs);
    return counted(L);
}
cudaError_t launch_mask_popcount(LaunchCfg& L, const uint32_t* d_masks, size_t stride_w, uint32_t npix, int F, uint32_t* d_out,
                                 cudaStream_t st) {
    if (F <= 0 || npix == 0) return cudaSuccess;
    const uint32_t nwords = (npix + 31u) >> 5;
    unsigned gx = grid_for(nwords, 256, L.sm_count);
    if (gx > 64u) gx = 64u;
    k_mask_popcount<<<dim3(gx, (unsigned)F), 256, 0, st>>>(d_masks, stride_w, nwords, d_out);
    return counted(L);
}
template <int PB, int RS>
static cudaError_t launch_apply_sweep_t(LaunchCfg& L, const ApplyChain& A, cudaStream_t st) {
    int per_sm = 1;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_apply_sweep<PB, RS>, AP_THREADS, 0);
    if (e != cudaSuccess) return e;
    if (per_sm < 1) per_sm = 1;
    const uint32_t slots = (uint32_t)(L.sm_count > 0 ? L.sm_count : 1) * (uint32_t)per_sm;
    const uint32_t rounds = (A.ntiles + slots - 1u) / slots;          // every CTA sweeps the same number of tiles, or one fewer
    k_apply_sweep<PB, RS><<<(A.ntiles + rounds - 1u) / rounds, AP_THREADS, 0, st>>>(A);
    return counted(L);
}
static void launch_tile_prefix(LaunchCfg& L, const ApplyChain& A, cudaStream_t st) {
    k_tile_count<<<dim3((A.ntiles + 7u) / 8u, A.count), 256, 0, st>>>(A);
    k_tile_scan<<<A.count, 1024, 0, st>>>(A);
    L.launches += 2;
}
cudaError_t launch_apply_chain(LaunchCfg& L, const ApplyChain& A, const uint8_t* h_modes, const int8_t* d_fields, uint32_t H,
                               uint32_t W, uint32_t* d_run_bad, cudaStream_t st) {
    if (A.count == 0 || A.ntiles == 0) return cudaSuccess;
    return by_format(A.pix_bytes, A.sample_bytes, [&](auto PBc, auto Sc) -> cudaError_t {
        constexpr int PB = decltype(PBc)::value, S = decltype(Sc)::value;
        auto mode = [&](uint32_t t) -> uint8_t { return h_modes ? h_modes[t] : 0; };
        launch_tile_prefix(L, A, st);
        for (uint32_t t = 0; t < A.count;) {
            if (mode(t) == 2) {
                uint32_t* next_bad = t + 1u < A.count && mode(t + 1u) != 2 ? d_run_bad + t + 1u : nullptr;
                k_apply_motion<PB, S><<<A.ntiles, AP_THREADS, 0, st>>>(A, t, d_fields, H, W, next_bad);
                if (cudaError_t e = counted(L)) return e;
                t++;
                continue;
            }
            // a run of plain / residual pairs [t, t1) is swept as a chain of its own (without a motion pair: the whole chain, A as
            // given); a run after a motion pair checks the first failing pair counted from its start, which that motion kernel stored
            uint32_t t1 = t;
            bool run_residual = false;
            for (; t1 < A.count && mode(t1) != 2; t1++) run_residual |= mode(t1) != 0;
            ApplyChain R = A;
            R.masks = A.masks + (size_t)t * A.mask_stride_w;
            R.base = A.base + t >= A.max_frames ? A.base + t - A.max_frames : A.base + t;
            R.count = t1 - t;
            R.value_off = A.value_off + t;
            R.residual = run_residual ? A.residual + t : nullptr;
            R.tile_pfx = A.tile_pfx + (size_t)t * A.ntiles;
            R.first_bad = t == 0 ? A.first_bad : d_run_bad + t;
            const cudaError_t e = run_residual ? launch_apply_sweep_t<PB, S>(L, R, st) : launch_apply_sweep_t<PB, 0>(L, R, st);
            if (e != cudaSuccess) return e;
            t = t1;
        }
        return cudaSuccess;
    });
}
cudaError_t launch_motion_search(LaunchCfg& L, const PairJob* d_pairs, int F, uint32_t H, uint32_t W, uint32_t pix_bytes, uint32_t sample_bytes,
                                 int8_t* d_fields, cudaStream_t st) {
    if (F <= 0 || H == 0 || W == 0) return cudaSuccess;
    return by_format(pix_bytes, sample_bytes, [&](auto PBc, auto Sc) -> cudaError_t {
        constexpr int PB = decltype(PBc)::value, S = decltype(Sc)::value;
        k_motion_search<PB, S><<<dim3(mv_blocks(H, W), (unsigned)F), MV_THREADS, 0, st>>>(d_pairs, H, W, d_fields);
        return counted(L);
    });
}
cudaError_t launch_median5(LaunchCfg& L, const void* d_in, uint32_t H, uint32_t W, int sample_bytes, void* d_out, cudaStream_t st) {
    if (H == 0 || W == 0) return cudaSuccess;
    dim3 grid((W + 31u) / 32u, (H + 7u) / 8u);
    if (sample_bytes == 1) k_median5<uint8_t><<<grid, 256, 0, st>>>((const uint8_t*)d_in, H, W, (uint8_t*)d_out);
    else if (sample_bytes == 2) k_median5<uint16_t><<<grid, 256, 0, st>>>((const uint16_t*)d_in, H, W, (uint16_t*)d_out);
    else return cudaErrorInvalidValue;
    return counted(L);
}
cudaError_t launch_bitrev(LaunchCfg& L, uint32_t* d_words, size_t nwords, cudaStream_t st) {
    if (nwords == 0) return cudaSuccess;
    k_bitrev<<<grid_for(nwords, 256, L.sm_count), 256, 0, st>>>(d_words, nwords);
    return counted(L);
}
cudaError_t launch_unpack_bits(LaunchCfg& L, const uint32_t* d_words, uint8_t* d_out, size_t nbits, cudaStream_t st) {
    if (nbits == 0) return cudaSuccess;
    k_unpack_bits<<<grid_for(nbits, 256, L.sm_count), 256, 0, st>>>(d_words, d_out, nbits);
    return counted(L);
}
cudaError_t launch_pack_bytes(LaunchCfg& L, const uint8_t* d_bytes, uint32_t* d_words, size_t nbits, int nonzero, cudaStream_t st) {
    if (nbits == 0) return cudaSuccess;
    k_pack_bytes<<<grid_for((nbits + 31) / 32, 256, L.sm_count), 256, 0, st>>>(d_bytes, d_words, nbits, nonzero);
    return counted(L);
}

cudaError_t launch_unpack_bits_msb(LaunchCfg& L, const uint32_t* d_words, uint8_t* d_out, size_t nbits, cudaStream_t st) {
    if (nbits == 0) return cudaSuccess;
    k_unpack_bits_msb<<<grid_for(nbits, 256, L.sm_count), 256, 0, st>>>(d_words, d_out, nbits);
    return counted(L);
}
cudaError_t launch_popcount(LaunchCfg& L, const uint32_t* d_words, size_t nwords, uint32_t* d_out, cudaStream_t st) {
    if (nwords == 0) return cudaSuccess;
    k_popcount<<<grid_for(nwords, 256, L.sm_count), 256, 0, st>>>(d_words, nwords, d_out);
    return counted(L);
}
cudaError_t launch_count_diff(LaunchCfg& L, const uint32_t* a, const uint32_t* b, size_t stride_words, size_t nwords, int F,
                              uint32_t* d_out, cudaStream_t st) {
    if (nwords == 0 || F <= 0) return cudaSuccess;
    unsigned gx = grid_for(nwords, 256, L.sm_count);
    if (gx > 64u) gx = 64u;
    dim3 g(gx, (unsigned)F);
    k_count_diff<<<g, 256, 0, st>>>(a, b, stride_words, nwords, d_out);
    return counted(L);
}
cudaError_t launch_items_u32(LaunchCfg& L, const FrameJob* d_job, const uint32_t* d_items, uint32_t count, uint8_t* d_result,
                             int insert, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    k_items_u32<<<grid_for(count, 256, L.sm_count), 256, 0, st>>>(d_job, d_items, count, d_result, insert);
    return counted(L);
}
cudaError_t launch_items_str(LaunchCfg& L, const FrameJob* d_job, const uint8_t* d_blob, const uint64_t* d_offs, uint32_t count,
                             uint8_t* d_result, int insert, int standard_k, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    k_items_str<<<grid_for(count, 128, L.sm_count), 128, 0, st>>>(d_job, d_blob, d_offs, count, d_result, insert, standard_k);
    return counted(L);
}
cudaError_t launch_hash_debug(LaunchCfg& L, const uint32_t* d_items, uint32_t count, uint64_t seed, uint64_t* d_out, int mode,
                              cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    k_hash_debug<<<grid_for(count, 256, L.sm_count), 256, 0, st>>>(d_items, count, seed, d_out, mode);
    return counted(L);
}

cudaError_t launch_push_slots(LaunchCfg& L, const uint32_t* d_bits, size_t stride_w, uint32_t slot_w, uint32_t pairs,
                              uint32_t* const* recv, uint32_t* const* flags, int nranks, int rank, size_t dst_off_w, uint32_t seq,
                              cudaStream_t st) {
    if (nranks < 1 || nranks > PEER_MAX) return cudaErrorInvalidValue;
    PeerTable pt;
    for (int r = 0; r < PEER_MAX; r++) { pt.recv[r] = r < nranks ? recv[r] : nullptr; pt.flags[r] = r < nranks ? flags[r] : nullptr; }
    if ((slot_w & 3u) || (stride_w & 3u) || (dst_off_w & 3u)) return cudaErrorInvalidValue;
    const size_t total = (size_t)pairs * (slot_w >> 2);
    size_t grid = (total + 255) / 256;
    if (grid > (size_t)L.sm_count * 8) grid = (size_t)L.sm_count * 8;
    if (grid < 1) grid = 1;
    k_push_slots<<<(unsigned)grid, 256, 0, st>>>(d_bits, stride_w, slot_w, pairs, pt, nranks, dst_off_w);
    k_peer_signal<<<1, 32, 0, st>>>(pt, nranks, rank, seq);
    return counted(L, 2);
}
cudaError_t launch_peer_wait(LaunchCfg& L, const uint32_t* d_flags, int nranks, uint32_t seq, long long timeout_cycles, uint32_t* d_err,
                             cudaStream_t st) {
    k_peer_wait<<<1, 32, 0, st>>>(d_flags, nranks, seq, timeout_cycles, d_err);
    return counted(L);
}

// N4: one CTA per segment; d_res: kDeflateSeg uint32 per segment of the launch
cudaError_t launch_deflate_segments(LaunchCfg& L, const DeflateSeg* d_segs, int count, uint32_t* d_res, uint32_t* d_sizes,
                                    uint32_t* d_adler, uint32_t* d_err, cudaStream_t st) {
    if (count <= 0) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(k_deflate_segments, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDzBytes);
    if (e != cudaSuccess) return e;
    k_deflate_segments<<<count, kDeflateThreads, kDzBytes, st>>>(d_segs, d_res, d_sizes, d_adler, d_err);
    return counted(L);
}
cudaError_t launch_deflate_concat(LaunchCfg& L, const DeflateCopy* d_jobs, int count, uint8_t* d_dst, uint64_t cap, uint32_t* d_err,
                                  cudaStream_t st) {
    if (count <= 0) return cudaSuccess;
    k_deflate_concat<<<count, 256, 0, st>>>(d_jobs, d_dst, cap, d_err);
    return counted(L);
}
int deflate_code_lengths_host(const uint32_t* freqs, uint32_t nsym, uint32_t max_bits, uint8_t* lengths) {
    HuffScratch S;
    return deflate_code_lengths(freqs, nsym, max_bits, lengths, &S);
}
cudaError_t launch_inflate_scan(LaunchCfg& L, const InflateScanJob* d_jobs, int count, const uint8_t* d_in, uint32_t* d_counts,
                                uint32_t* d_cand, cudaStream_t st) {
    if (count <= 0) return cudaSuccess;
    k_inflate_scan<<<count, 256, 0, st>>>(d_jobs, d_in, d_counts, d_cand);
    return counted(L);
}
cudaError_t launch_inflate_segments(LaunchCfg& L, const uint32_t* d_slot_stream, const InflateStream* d_streams, int nslots,
                                    const uint8_t* d_in, const uint32_t* d_cand, uint8_t* d_slots, InflateSegResult* d_res,
                                    uint32_t* d_start, cudaStream_t st) {
    if (nslots <= 0) return cudaSuccess;
    k_inflate_segments<<<nslots, 32, 0, st>>>(d_slot_stream, d_streams, d_in, d_cand, d_slots, d_res, d_start);
    return counted(L);
}
void inflate_segment_host(const uint8_t* in, uint64_t avail, uint8_t* out, InflateSegResult* res) {
    InflateScratch S;
    inflate_segment(in, avail, out, &S, res);
}

}  // namespace rbf
