// rbf_k2_insert.cuh -- Per-filter constants and K2: insert the set positions into the frame's Bloom filter (ivc:235-237, ivc:99-114).  Included by rbf_kernels.cu inside namespace rbf.
#pragma once

// ------------------------------------------------------------------------------------------
// Per-filter constants kept in registers / shared memory
// ------------------------------------------------------------------------------------------
struct FilterK {
    FastMod fm;
    uint64_t T, s1, s2, sA;
    uint32_t fk, has_act, nm;
};
__device__ __forceinline__ FilterK filter_consts(const FrameJob& J) {
    FilterK k;
    k.fm = J.fm; k.T = J.act_T; k.s1 = J.seed1; k.s2 = J.seed2; k.sA = J.seedA; k.fk = J.floor_k; k.has_act = J.has_act; k.nm = J.neg_m;
    return k;
}

// fast reductions for 2 <= m <= 2^30 (the specialised insert / query paths are only taken then)
__device__ __forceinline__ uint32_t mod_fast(uint64_t h, const FastMod& f, uint32_t neg_m) {
    const uint32_t hh = (uint32_t)(h >> 32), hl = (uint32_t)h;
    // q = hh*Mh + hi(hh*Ml) + hi(hl*Mh);  r = hl - q*m = hl + q*neg_m (neg_m = 2^32 - m from the host), with q's two parts
    // folded into two IMADs (no add, and no zeroed register pair for an accumulating IMAD.HI)
    uint32_t r;
    asm("{\n .reg .u32 a, b;\n mul.hi.u32 a, %1, %4;\n mad.lo.u32 a, %1, %3, a;\n mul.hi.u32 b, %2, %3;\n mad.lo.u32 %0, b, %5, %2;\n mad.lo.u32 %0, a, %5, %0;\n}"
        : "=&r"(r) : "r"(hh), "r"(hl), "r"(f.Mh), "r"(f.Ml), "r"(neg_m));
    r = min(r, r - 2u * f.m);
    return min(r, r - f.m);
}
__device__ __forceinline__ uint32_t addmod_fast(uint32_t a, uint32_t b, uint32_t m) {
    const uint32_t s = a + b;
    return min(s, s - m);
}

// Bit setter of an LSB-first bit array held in global memory (RED.OR into L2)
struct GlobalBits {
    uint32_t* bits;
    __device__ __forceinline__ void set(uint32_t idx) const { red_or_global(bits + (idx >> 5), 1u << (idx & 31u)); }
};

// add_index (ivc:99-114) given the three hashes; every bit goes through B.set
template <class Bits>
__device__ __forceinline__ void insert_hashes(const Bits& B, const FilterK& K, uint64_t h1, uint64_t h2, uint64_t hA) {
    uint32_t idx = mod_u64(h1, K.fm);
    const uint32_t step = mod_u64(h2, K.fm);
    for (uint32_t i = 0; i < K.fk; i++) {
        B.set(idx);
        idx = addmod(idx, step, K.fm.m);
    }
    if (K.has_act && hA < K.T) B.set(idx);
}

// ------------------------------------------------------------------------------------------
// K2: insert.  One thread owns a century (100 positions); the few set positions of the mask
// are hashed with the shared century/decade prefix states and OR-ed into the bit array in L2.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_insert(const FrameJob* __restrict__ jobs) {
    const FrameJob& J = jobs[blockIdx.y];
    if (J.l == 0) return;
    const FilterK K = filter_consts(J);
    const uint32_t ncent = (J.n + 99u) / 100u;
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < ncent; c += gridDim.x * blockDim.x) {
        const uint32_t nvalid = min(100u, J.n - 100u * c);
        Bits128 mb = load_bits100(J.mask, c, nvalid);
        if ((mb.lo | mb.hi) == 0ull) continue;
        const Century cen = make_century(c);
        const uint64_t C1 = century_state(cen, K.s1), C2 = century_state(cen, K.s2), CA = century_state(cen, K.sA);
        for (int half = 0; half < 2; half++) {
            uint64_t v = half ? mb.hi : mb.lo;
            while (v) {
                const uint32_t pos = (uint32_t)(__ffsll((long long)v) - 1) + 64u * half;
                v &= v - 1ull;
                const uint32_t x = pos / 10u, y = pos - 10u * x;
                const uint64_t h1 = finish(cen.kind, decade_state(cen, C1, K.s1, x), K.s1, y);
                const uint64_t h2 = finish(cen.kind, decade_state(cen, C2, K.s2, x), K.s2, y);
                const uint64_t hA = K.has_act ? finish(cen.kind, decade_state(cen, CA, K.sA, x), K.sA, y) : 0ull;
                insert_hashes(GlobalBits{J.bits}, K, h1, h2, hA);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// K2 (dense, the default): the same insert with all lanes busy, building each frame's array in cluster shared memory.
//
// The mask is sparse (p ~ 5 %), so a lane looping over its own set positions leaves most of the warp idle.  Here a warp
// takes a slab of 32 centuries: the set positions of the slab are compacted (count, warp scan, scatter) into a per-warp
// item list (rounds of at most I2_CAP items), and the list is consumed 32 items at a time: the owner's century states come
// by shuffle, two-character finish, the one-IMAD remainder of the query kernels, floor(k)-specialised straight-line probes.
//
// A 4K frame sets ~1.3 M bits at random.  As one RED.OR each into L2 that is bound by the L2 atomic units, so the bits
// are set in SRAM instead: cluster (f, r) of cs CTAs holds a zeroed copy of frame f's array, CTA rank j owning words
// [j*K2_WORDS, (j+1)*K2_WORDS) in its shared memory.  A bit of the own range is a shared-memory atomic, one of a peer's
// range a distributed-shared-memory RED, and a word beyond cs*K2_WORDS (filters larger than 8 CTAs hold) a RED.OR into
// L2 as before.  At the end each CTA writes its range out once: a frame with one copy as plain 16 B stores, a frame with
// R > 1 copies (the frames of a launch's last, partial wave) as one RED.OR per non-zero word -- never more REDs than the
// direct form, since every non-zero word holds at least one bit-set.
// ------------------------------------------------------------------------------------------
// Build-time shape (scripts/build_variant.py -D...).  Measured at 299 4K pairs on an H100 80GB HBM3 at 400 W, K2 per step:
// 16 warps, cs = 2: 3.6-3.8 ms; 16 warps, 2 CTAs per SM (cs = 3): 4.7-4.9 ms; 32 warps, cs = 2: 3.3-3.6 ms; 32 warps, cs = 1:
// 3.0-3.1 ms (before the last-wave split below; 2.45 ms with it).  A RED into a peer CTA's shared memory costs more than the
// 16 % of a 4K array's bit-sets that cs = 1 leaves to L2, so clusters are off by default.
#ifndef RBF_K2_CTAS_PER_SM
#define RBF_K2_CTAS_PER_SM 1
#endif
#ifndef RBF_K2_WARPS
#define RBF_K2_WARPS (32 / RBF_K2_CTAS_PER_SM)                         // 1024 threads: 63 registers, no spills
#endif
#ifndef RBF_K2_MAX_CS
#define RBF_K2_MAX_CS 1                                                // largest cluster (at most 8, the portable limit)
#endif
constexpr int I2_CAP = 512;                                           // list entries per warp and round (uint16 each)
constexpr int K2_CTAS_PER_SM = RBF_K2_CTAS_PER_SM, K2_MAX_CS = RBF_K2_MAX_CS;
constexpr int K2_WARPS = RBF_K2_WARPS, K2_THREADS = 32 * K2_WARPS;
constexpr uint32_t K2_LIST_BYTES = (uint32_t)K2_WARPS * I2_CAP * 2u;
// 228 KB of shared memory per SM, of which the runtime reserves 1 KB per CTA; a multiple of 16 words
constexpr uint32_t K2_WORDS = ((233472u / K2_CTAS_PER_SM - 1024u - K2_LIST_BYTES) / 4u) & ~15u;
constexpr uint32_t K2_SMEM_BYTES = 4u * K2_WORDS + K2_LIST_BYTES;
static_assert(K2_MAX_CS >= 1 && K2_MAX_CS <= 8, "cluster size");
static_assert(K2_SMEM_BYTES <= 232448u, "227 KB per CTA");

__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t cluster_nctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
// every thread of the cluster: what this thread wrote (shared or remote) is visible to the cluster afterwards
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}

// Bit setter of one frame's array spread over a cluster.  Every bit-set of the clustered kernel goes through it: a RED
// into L2 on a word the cluster owns would be overwritten when the cluster writes that word out.
struct ClusterBits {
    uint32_t* bits;        // the frame's array in global memory
    uint32_t s_words;      // shared-memory address of this CTA's words (the same offset in every CTA of the cluster)
    uint32_t rank, cs;
    __device__ __forceinline__ void set(uint32_t idx) const {
        const uint32_t w = idx >> 5, v = 1u << (idx & 31u), owner = w / K2_WORDS;
        const uint32_t a = s_words + 4u * (w - owner * K2_WORDS);
        if (owner == rank) {                                       // shared::cta explicitly: ATOMS (shared::cluster would be a generic ATOM)
            asm volatile("red.shared::cta.or.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
        } else if (owner < cs) {
            asm volatile("{\n\t.reg .u32 ra;\n\tmapa.shared::cluster.u32 ra, %0, %1;\n\tred.relaxed.cluster.shared::cluster.or.b32 [ra], %2;\n\t}"
                         ::"r"(a), "r"(owner), "r"(v) : "memory");
        } else {
            red_or_global(bits + w, v);
        }
    }
};

template <int KIND, int FKT, class Bits>
__device__ __forceinline__ void insert_batch(const FilterK& K, const Bits& B, uint32_t tag, bool have, uint64_t C1,
                                             uint64_t C2, uint64_t CA) {
    const uint32_t owner = (tag >> 7) & 31u, pos = tag & 127u, x = (pos * 205u) >> 11, y = pos - 10u * x;   // pos < 128: /10 exact
    const uint64_t C1o = (uint64_t)__shfl_sync(0xffffffffu, (uint32_t)C1, owner) | ((uint64_t)__shfl_sync(0xffffffffu, (uint32_t)(C1 >> 32), owner) << 32);
    const uint64_t C2o = (uint64_t)__shfl_sync(0xffffffffu, (uint32_t)C2, owner) | ((uint64_t)__shfl_sync(0xffffffffu, (uint32_t)(C2 >> 32), owner) << 32);
    uint64_t CAo = 0;
    if (K.has_act) CAo = (uint64_t)__shfl_sync(0xffffffffu, (uint32_t)CA, owner) | ((uint64_t)__shfl_sync(0xffffffffu, (uint32_t)(CA >> 32), owner) << 32);
    if (!have) return;
    uint32_t idx = mod_fast(finish_t<KIND>(decade_state_t<KIND>(C1o, K.s1, x), K.s1, y), K.fm, K.nm);
    const uint32_t step = mod_fast(finish_t<KIND>(decade_state_t<KIND>(C2o, K.s2, x), K.s2, y), K.fm, K.nm);
    if (FKT > 0) {
#pragma unroll
        for (int p = 0; p < FKT; p++) { B.set(idx); idx = addmod_fast(idx, step, K.fm.m); }
    } else {
        for (uint32_t p = 0; p < K.fk; p++) { B.set(idx); idx = addmod_fast(idx, step, K.fm.m); }
    }
    if (K.has_act && finish_t<KIND>(decade_state_t<KIND>(CAo, K.sA, x), K.sA, y) < K.T) B.set(idx);
}

template <int KIND, class Bits>
__device__ __noinline__ void insert_slab_dense(const FilterK K, const Bits B, Bits128 mb, const Century cen, uint32_t list_addr) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t C1 = century_state(cen, K.s1), C2 = century_state(cen, K.s2), CA = century_state(cen, K.sA);
    uint64_t lo = mb.lo, hi = mb.hi;
    uint32_t total;
    do {                                                             // rounds of at most I2_CAP items (one round unless p > 16 % locally)
        const uint32_t cnt = __popcll(lo) + __popcll(hi);
        uint32_t inc = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= (uint32_t)d) inc += t;
        }
        total = __shfl_sync(0xffffffffu, inc, 31);
        uint32_t off = inc - cnt;
        while (lo && off < (uint32_t)I2_CAP) {
            const uint32_t b = (uint32_t)(__ffsll((long long)lo) - 1); lo &= lo - 1ull;
            asm volatile("st.shared.u16 [%0], %1;" ::"r"(list_addr + 2u * off), "h"((uint16_t)((lane << 7) | b)) : "memory");
            off++;
        }
        while (hi && off < (uint32_t)I2_CAP) {
            const uint32_t b = (uint32_t)(__ffsll((long long)hi) + 63); hi &= hi - 1ull;
            asm volatile("st.shared.u16 [%0], %1;" ::"r"(list_addr + 2u * off), "h"((uint16_t)((lane << 7) | b)) : "memory");
            off++;
        }
        __syncwarp();
        const uint32_t ntot = min(total, (uint32_t)I2_CAP);
#pragma unroll 1
        for (uint32_t base = 0; base < ntot; base += 32u) {
            const uint32_t i = base + lane;
            uint16_t t16;
            asm volatile("ld.shared.u16 %0, [%1];" : "=h"(t16) : "r"(list_addr + 2u * min(i, (uint32_t)(I2_CAP - 1))) : "memory");
            const bool have = i < ntot;
            if (K.fk == 3u) insert_batch<KIND, 3, Bits>(K, B, t16, have, C1, C2, CA);
            else if (K.fk == 2u) insert_batch<KIND, 2, Bits>(K, B, t16, have, C1, C2, CA);
            else insert_batch<KIND, 0, Bits>(K, B, t16, have, C1, C2, CA);
        }
        __syncwarp();
    } while (total > (uint32_t)I2_CAP);
}

// slabs sl0, sl0 + stride, ... of frame J, one per warp; every bit-set goes through B.set
template <class Bits>
__device__ __forceinline__ void insert_slabs(const FrameJob& J, const FilterK& K, const Bits& B, uint32_t list_addr, uint32_t sl0, uint32_t stride) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t ncent = (J.n + 99u) / 100u;
    const uint32_t nslab = (ncent + 31u) / 32u;
    const bool fast = K.fm.fast != 0u;                               // 2 <= m <= 2^30: the specialised path
    for (uint32_t sl = sl0; sl < nslab; sl += stride) {
        const uint32_t slab = sl * 32u, c = slab + lane;
        const bool active = c < ncent;
        Bits128 mb; mb.lo = 0; mb.hi = 0;
        if (active) mb = load_bits100(J.mask, c, min(100u, J.n - 100u * c));
        if (!__any_sync(0xffffffffu, (mb.lo | mb.hi) != 0ull)) continue;
        const uint32_t last = min(slab + 31u, ncent - 1u);
        const bool uniform = fast && slab >= 1u && ndigits_u32(slab) == ndigits_u32(last);
        if (uniform) {
            const Century cen = make_century(active ? c : slab);
            switch (cen.kind) {
            case K_4B: insert_slab_dense<K_4B, Bits>(K, B, mb, cen, list_addr); break;
            case K_8B: insert_slab_dense<K_8B, Bits>(K, B, mb, cen, list_addr); break;
            case K_44: insert_slab_dense<K_44, Bits>(K, B, mb, cen, list_addr); break;
            case K_88: insert_slab_dense<K_88, Bits>(K, B, mb, cen, list_addr); break;
            default:   insert_slab_dense<K_BB, Bits>(K, B, mb, cen, list_addr); break;
            }
        } else if ((mb.lo | mb.hi) != 0ull) {             // century 0, a digit-count boundary or a huge filter: per-lane form
            const Century cen = make_century(c);
            const uint64_t C1 = century_state(cen, K.s1), C2 = century_state(cen, K.s2), CA = century_state(cen, K.sA);
            for (int half = 0; half < 2; half++) {
                uint64_t v = half ? mb.hi : mb.lo;
                while (v) {
                    const uint32_t pos = (uint32_t)(__ffsll((long long)v) - 1) + 64u * half;
                    v &= v - 1ull;
                    const uint32_t x = pos / 10u, y = pos - 10u * x;
                    insert_hashes(B, K, finish(cen.kind, decade_state(cen, C1, K.s1, x), K.s1, y),
                                  finish(cen.kind, decade_state(cen, C2, K.s2, x), K.s2, y),
                                  K.has_act ? finish(cen.kind, decade_state(cen, CA, K.sA, x), K.sA, y) : 0ull);
                }
            }
        }
    }
}

// grid (cs, units), one cluster of cs CTAs per unit: units [0, full) are frames 0..full-1 with one copy each, and every
// later frame has tail_copies consecutive units (its copies)
__global__ void __launch_bounds__(K2_THREADS, K2_CTAS_PER_SM) k_insert_cluster(const FrameJob* __restrict__ jobs, uint32_t full,
                                                                               uint32_t tail_copies) {
    uint32_t f = blockIdx.y, copy = 0u, copies = 1u;
    if (f >= full) { const uint32_t t = f - full; f = full + t / tail_copies; copy = t - (f - full) * tail_copies; copies = tail_copies; }
    const FrameJob& J = jobs[f];
    if (J.l == 0) return;                                            // the whole cluster returns: no barrier is pending
    extern __shared__ __align__(16) uint32_t s_k2[];                 // [K2_WORDS] array words, then the per-warp item lists
    const FilterK K = filter_consts(J);
    const uint32_t warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);   // warp-uniform for the compiler
    const uint32_t list_addr = smem_u32(s_k2 + K2_WORDS) + warp * (2u * I2_CAP);
    ClusterBits B;
    B.bits = J.bits; B.s_words = smem_u32(s_k2); B.rank = cluster_ctarank(); B.cs = cluster_nctarank();
    const uint32_t words = (J.l + 31u) >> 5, first = B.rank * K2_WORDS;
    const uint32_t own = words > first ? min(words - first, K2_WORDS) : 0u;
    const uint32_t own4 = (own + 3u) >> 2;                           // 16 B groups (K2_WORDS is a multiple of 4)
    for (uint32_t i = threadIdx.x; i < own4; i += K2_THREADS) reinterpret_cast<uint4*>(s_k2)[i] = make_uint4(0u, 0u, 0u, 0u);
    cluster_sync();                                                  // every copy is zeroed before any peer ORs into it

    insert_slabs(J, K, B, list_addr, (copy * B.cs + B.rank) * K2_WARPS + warp, copies * B.cs * K2_WARPS);
    cluster_sync();                                                  // all ORs have landed; no peer addresses this CTA any more

    uint32_t* dst = J.bits + first;                                  // 16 B aligned: the array is, and K2_WORDS is a multiple of 4
    if (copies == 1u) {                                              // the only writer of these words; the zero words in [own, 4*own4)
        for (uint32_t i = threadIdx.x; i < own4; i += K2_THREADS)    // lie inside the array's 16 B padding
            reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(s_k2)[i];
    } else {
        for (uint32_t i = threadIdx.x; i < own; i += K2_THREADS) {
            const uint32_t v = s_k2[i];
            if (v) red_or_global(dst + i, v);
        }
    }
}

// K2 for arrays mostly beyond shared memory (8K frames at k* = 4: 16 % of the words fit): the same slabs with every bit a
// RED.OR into L2.  One CTA per 4 slabs and no grid cap, so the frames are worked through in order and the arrays being
// written stay in L2 (a capped grid-stride form spreads over all F frames at once).
constexpr int I2_WARPS = 4;
__global__ void __launch_bounds__(I2_WARPS * 32) k_insert2(const FrameJob* __restrict__ jobs) {
    const FrameJob& J = jobs[blockIdx.y];
    if (J.l == 0) return;
    __shared__ __align__(16) uint16_t s_list[I2_WARPS][I2_CAP];
    const uint32_t warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);   // warp-uniform for the compiler
    insert_slabs(J, filter_consts(J), GlobalBits{J.bits}, smem_u32(&s_list[warp][0]), blockIdx.x * I2_WARPS + warp, gridDim.x * I2_WARPS);
}
