// rbf_k3_query.cuh -- K3: Bloom test of all n positions -> pass mask (ivc:245-253, ivc:116-138): per-lane, staged rings, decade tiles.  Included by rbf_kernels.cu inside namespace rbf.
#pragma once
#include <type_traits>

// ------------------------------------------------------------------------------------------
// K3: query.  Persistent CTAs split the batch's centuries evenly; for every frame segment the
// CTA stages the frame's bit array into shared memory with TMA bulk copies (the tail that does
// not fit is probed through L2) and tests all positions.  Output: pass mask, 128 bits/century.
// ------------------------------------------------------------------------------------------
constexpr int QT = 512;

struct BitView {
    const uint32_t* sm;      // shared-memory copy of words [0, sm_words)
    const uint32_t* gl;      // whole array in global memory
    uint32_t sm_words;
};
__device__ __forceinline__ uint32_t test_bit(const BitView& bv, uint32_t idx) {
    const uint32_t w = idx >> 5;
    const uint32_t word = (w < bv.sm_words) ? bv.sm[w] : __ldg(bv.gl + w);
    return (word >> (idx & 31u)) & 1u;
}

// check_index (ivc:116-138) for the position with decade states D1, D2, DA and units digit y
__device__ __forceinline__ uint32_t check_one(const BitView& bv, const FilterK& K, int kind, uint64_t D1, uint64_t D2,
                                              uint64_t DA, uint32_t y) {
    uint32_t idx = mod_u64(finish(kind, D1, K.s1, y), K.fm);
    uint32_t ok = 1u;
    if (K.fk >= 1u) ok = test_bit(bv, idx);
    if (ok && (K.fk >= 2u || K.has_act)) {
        const uint32_t step = mod_u64(finish(kind, D2, K.s2, y), K.fm);
        for (uint32_t i = 1; i < K.fk && ok; i++) {
            idx = addmod(idx, step, K.fm.m);
            ok = test_bit(bv, idx);
        }
        if (ok && K.has_act && finish(kind, DA, K.sA, y) < K.T) {
            if (K.fk >= 1u) idx = addmod(idx, step, K.fm.m);
            ok = test_bit(bv, idx);
        }
    }
    return ok;
}

__device__ __forceinline__ Bits128 query_century(const BitView& bv, const FilterK& K, uint32_t c, uint32_t nvalid) {
    const Century cen = make_century(c);
    const uint64_t C1 = century_state(cen, K.s1), C2 = century_state(cen, K.s2), CA = century_state(cen, K.sA);
    Bits128 res; res.lo = 0; res.hi = 0;
#pragma unroll 1
    for (uint32_t x = 0; x < 10u; x++) {
        const uint64_t D1 = decade_state(cen, C1, K.s1, x), D2 = decade_state(cen, C2, K.s2, x),
                       DA = decade_state(cen, CA, K.sA, x);
        uint32_t dres = 0;
#pragma unroll
        for (uint32_t y = 0; y < 10u; y++) dres |= check_one(bv, K, cen.kind, D1, D2, DA, y) << y;
        const uint32_t p0 = 10u * x;
        if (p0 < 64u) {
            res.lo |= (uint64_t)dres << p0;
            if (p0 > 54u) res.hi |= (uint64_t)dres >> (64u - p0);
        } else {
            res.hi |= (uint64_t)dres << (p0 - 64u);
        }
    }
    if (nvalid < 100u) {
        if (nvalid >= 64u) res.hi &= (1ull << (nvalid - 64u)) - 1ull;
        else { res.hi = 0; res.lo &= (1ull << nvalid) - 1ull; }
    }
    return res;
}

__global__ void __launch_bounds__(QT) k_query(const FrameJob* __restrict__ jobs, const uint32_t* __restrict__ cent_prefix,
                                              int F, uint32_t smem_words_cap) {
    extern __shared__ __align__(128) uint32_t sbits[];
    __shared__ __align__(8) uint64_t bar;
    const uint32_t total = cent_prefix[F];
    const uint32_t lo = (uint32_t)(((uint64_t)total * blockIdx.x) / gridDim.x);
    const uint32_t hi = (uint32_t)(((uint64_t)total * (blockIdx.x + 1)) / gridDim.x);
    if (threadIdx.x == 0) { mbar_init(&bar, 1); fence_mbar_init(); }
    __syncthreads();
    if (lo >= hi) return;
    // first frame with cent_prefix[f+1] > lo
    int f = 0;
    { int a = 0, b = F; while (a < b) { int m = (a + b) >> 1; if (cent_prefix[m + 1] > lo) b = m; else a = m + 1; } f = a; }
    uint32_t parity = 0, g = lo;
    while (g < hi) {
        while (cent_prefix[f + 1] <= g) f++;
        const FrameJob& J = jobs[f];
        const uint32_t seg_end = min(hi, cent_prefix[f + 1]);
        const uint32_t c_begin = g - cent_prefix[f], c_end = seg_end - cent_prefix[f];
        const uint32_t nwords = (J.l + 31u) >> 5;
        const uint32_t sw = min((nwords + 3u) & ~3u, smem_words_cap);     // 16 B granules; buffer is padded
        __syncthreads();                                                    // everyone done with the previous array
        if (threadIdx.x == 0) {
            fence_proxy_async();
            mbar_expect_tx(&bar, sw * 4u);
            const uint8_t* src = reinterpret_cast<const uint8_t*>(J.bits);
            uint8_t* dst = reinterpret_cast<uint8_t*>(sbits);
            for (uint32_t off = 0; off < sw * 4u; off += 32768u)
                bulk_g2s(dst + off, src + off, min(32768u, sw * 4u - off), &bar);
        }
        mbar_wait(&bar, parity);
        parity ^= 1u;
        const FilterK K = filter_consts(J);
        BitView bv; bv.sm = sbits; bv.gl = J.bits; bv.sm_words = sw;
        uint4* pass4 = reinterpret_cast<uint4*>(J.pass);
        for (uint32_t c = c_begin + threadIdx.x; c < c_end; c += QT) {
            const Bits128 r = query_century(bv, K, c, min(100u, J.n - 100u * c));
            pass4[c] = make_uint4((uint32_t)r.lo, (uint32_t)(r.lo >> 32), (uint32_t)r.hi, (uint32_t)(r.hi >> 32));
        }
        g = seg_end;
    }
}

// ------------------------------------------------------------------------------------------
// K3 (staged): the same query as a warp-synchronous pipeline of DENSE stages.
//
// check_index is a pure conjunction (ivc:127-136), so its probes may be evaluated in any order
// and abandoned at the first zero.  Lane t of a warp owns century slab+t; the warp walks the
// 100 positions of its 32 centuries in lockstep:
//   stage A  (all positions)        h1 -> probe 0.  ~1/2 survive (the Bloom fill is ~1/2).
//   stage B  (survivors of A)       h2 -> probes 1..floor_k-1.
//   stage C  (survivors of B)       activation hash -> the floor_k+1'th probe if activated.
// Survivors are compacted through per-warp shared-memory rings (ballot + popc), so stages B and C
// always run with 32 busy lanes instead of diverging per lane.  A stage-B record carries the
// owner's decade state of seed 2; stage C fetches the owner's century state of the activation
// seed with a shuffle.  Positions whose mask bit is set are known to pass (a Bloom filter has no
// false negatives) and skip the hashing.  Results are identical to the per-lane form above.
// ------------------------------------------------------------------------------------------
constexpr int Q2_WARPS = 24;
__constant__ uint64_t c_rot_digit[16] = {rot_digit_const(0), rot_digit_const(1), rot_digit_const(2), rot_digit_const(3),
                                         rot_digit_const(4), rot_digit_const(5), rot_digit_const(6), rot_digit_const(7),
                                         rot_digit_const(8), rot_digit_const(9), 0, 0, 0, 0, 0, 0};
constexpr int Q2_THREADS = Q2_WARPS * 32;
constexpr int Q2_RING = 64;                               // entries per ring (two drains' worth)
constexpr int Q2_WARP_WORDS = (Q2_RING * 16 + Q2_RING * 8 + 32 * 16 + 128) / 4;   // B ring, C ring, pass accumulators, digit table

// explicit shared-space accesses (32-bit shared addresses): no generic-pointer resolution in the hot loops
__device__ __forceinline__ void sts128_if(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d, bool p) {
    asm volatile("{\n .reg .pred q;\n setp.ne.u32 q, %5, 0;\n @q st.shared.v4.u32 [%0], {%1,%2,%3,%4};\n}" ::"r"(addr), "r"(a), "r"(b),
                 "r"(c), "r"(d), "r"((uint32_t)p)
                 : "memory");
}
__device__ __forceinline__ void sts64_if(uint32_t addr, uint32_t a, uint32_t b, bool p) {
    asm volatile("{\n .reg .pred q;\n setp.ne.u32 q, %3, 0;\n @q st.shared.v2.u32 [%0], {%1,%2};\n}" ::"r"(addr), "r"(a), "r"(b),
                 "r"((uint32_t)p)
                 : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ uint2 lds64(uint32_t addr) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void red_or_shared_if(uint32_t addr, uint32_t v, bool p) {
    asm volatile("{\n .reg .pred q;\n setp.ne.u32 q, %2, 0;\n @q red.shared.or.b32 [%0], %1;\n}" ::"r"(addr), "r"(v), "r"((uint32_t)p) : "memory");
}

// bit `idx` of the Bloom array.  PM (probe mode):
//   0  the whole array is in this CTA's shared memory
//   1  words [0, sm_words) in shared memory, the rest through L2 (read-only path)
template <int PM>
__device__ __forceinline__ uint32_t probe_bit(uint32_t sm_addr, uint32_t sm_addr1, const uint32_t* __restrict__ gl,
                                              uint32_t sm_words, uint32_t idx) {
    const uint32_t w = idx >> 5;
    uint32_t word;
    if (PM == 1) {
        // the unconditional mov makes the two predicated loads a full definition for ptxas (otherwise `word` stays live
        // across loop iterations and is spilled right behind the load, stalling on it)
        asm("{\n .reg .pred q;\n setp.lt.u32 q, %1, %2;\n mov.u32 %0, 0;\n @q ld.shared.u32 %0, [%3];\n @!q ld.global.nc.u32 %0, [%4];\n}"
            : "=r"(word)
            : "r"(w), "r"(sm_words), "r"(sm_addr + 4u * w), "l"(gl + w));
    } else {
        asm("ld.shared.u32 %0, [%1];" : "=r"(word) : "r"(sm_addr + 4u * w));
    }
    return (word >> (idx & 31u)) & 1u;
}

// mod_fast / addmod_fast (exact h mod m for 2 <= m <= 2^30) live in rbf_k2_insert.cuh

// pass bit of (owner lane, x, y) into the owner's 128-bit accumulator
__device__ __forceinline__ void deliver_pass(uint32_t pacc_addr, uint32_t tag, bool p) {
    const uint32_t owner = tag >> 8, pos = 10u * ((tag >> 4) & 15u) + (tag & 15u);
    red_or_shared_if(pacc_addr + 16u * owner + 4u * (pos >> 5), 1u << (pos & 31u), p);
}

struct RingState {                 // warp-uniform
    uint32_t qb_head, qb_cnt, qc_head, qc_cnt;
};

// stage B (32 survivors of A) and stage C (32 survivors of B); `force` drains partial batches
template <int KIND, int FKT, int PM>
__device__ __forceinline__ void drain_stages(const FilterK& K, uint32_t sm_addr, uint32_t sm_addr1, const uint32_t* __restrict__ gl,
                                             uint32_t sm_words, uint32_t qb_addr, uint32_t qc_addr, uint32_t pacc_addr,
                                             uint32_t lane, uint32_t lt, uint64_t CA, RingState& R, bool force) {
    if (R.qb_cnt >= 32u || (force && R.qb_cnt > 0u)) {               // ---- stage B
        __syncwarp();
        const uint32_t nb = min(32u, R.qb_cnt);
        const bool have = lane < nb;
        const uint4 r = lds128(qb_addr + 16u * ((R.qb_head + lane) & (Q2_RING - 1)));
        R.qb_head = (R.qb_head + nb) & (Q2_RING - 1);
        R.qb_cnt -= nb;
        const uint64_t rbB = kind_ends_in_byte<KIND>() ? ({ const uint2 t = lds64(pacc_addr + 512u + 8u * (r.y & 15u)); (uint64_t)t.x | ((uint64_t)t.y << 32); }) : 0ull;
        const uint32_t stepm = have ? mod_fast(finish_prep<KIND>((uint64_t)r.z | ((uint64_t)r.w << 32), K.s2, r.y & 15u, rbB), K.fm, K.nm) : 0u;
        uint32_t idx = have ? r.x : 0u;
        uint32_t ok = have ? 1u : 0u;
        if (FKT > 0) {                                               // floor_k known at compile time: straight-line probes
#pragma unroll
            for (int i = 1; i < FKT; i++) {
                idx = addmod_fast(idx, stepm, K.fm.m);
                ok &= probe_bit<PM>(sm_addr, sm_addr1, gl, sm_words, idx);
            }
        } else {
            for (uint32_t i = 1; i < K.fk; i++) {
                idx = addmod_fast(idx, stepm, K.fm.m);
                ok &= probe_bit<PM>(sm_addr, sm_addr1, gl, sm_words, idx);
                if (!__any_sync(0xffffffffu, ok != 0u)) break;
            }
        }
        if (K.has_act) {
            idx = addmod_fast(idx, stepm, K.fm.m);                   // index of probe floor_k
            const uint32_t b2 = __ballot_sync(0xffffffffu, ok != 0u);
            sts64_if(qc_addr + 8u * ((R.qc_head + R.qc_cnt + __popc(b2 & lt)) & (Q2_RING - 1)), idx, r.y, ok != 0u);
            R.qc_cnt += __popc(b2);
        } else {
            deliver_pass(pacc_addr, r.y, ok != 0u);
        }
    }
    if (R.qc_cnt >= 32u || (force && R.qb_cnt == 0u && R.qc_cnt > 0u)) {   // ---- stage C
        __syncwarp();
        const uint32_t nc = min(32u, R.qc_cnt);
        const bool have = lane < nc;
        const uint2 r = lds64(qc_addr + 8u * ((R.qc_head + lane) & (Q2_RING - 1)));
        R.qc_head = (R.qc_head + nc) & (Q2_RING - 1);
        R.qc_cnt -= nc;
        const uint32_t tag = have ? r.y : 0u;
        const uint32_t owner = tag >> 8;
        const uint64_t CAo = (uint64_t)__shfl_sync(0xffffffffu, (uint32_t)CA, owner) |
                             ((uint64_t)__shfl_sync(0xffffffffu, (uint32_t)(CA >> 32), owner) << 32);
        const uint64_t hA = finish_t<KIND>(decade_state_t<KIND>(CAo, K.sA, (tag >> 4) & 15u), K.sA, tag & 15u);
        const uint32_t pb = probe_bit<PM>(sm_addr, sm_addr1, gl, sm_words, have ? r.x : 0u);
        deliver_pass(pacc_addr, tag, have && (!(hA < K.T) || pb != 0u));
    }
}

template <int KIND, int FKT, int PM>
__device__ __noinline__ void query_slab_staged(const FilterK K, uint32_t sm_addr, uint32_t sm_addr1, const uint32_t* __restrict__ gl,
                                               uint32_t sm_words, const uint32_t* __restrict__ mask, uint32_t n,
                                               uint32_t slab_c0, uint32_t c_end, uint4* __restrict__ pass4,
                                               uint32_t qb_addr, uint32_t qc_addr, uint32_t pacc_addr) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t c = slab_c0 + lane;
    const bool active = c < c_end;
    const Century cen = make_century(active ? c : slab_c0);
    const uint64_t C1 = century_state(cen, K.s1), C2 = century_state(cen, K.s2), CA = century_state(cen, K.sA);
    const uint32_t nvalid = active ? min(100u, n - 100u * c) : 0u;
    // positions that need no hashing: known members (mask bit set) and positions beyond n
    uint64_t skip_lo = 0, skip_hi = 0;
    if (active && mask != nullptr) { const Bits128 mb = load_bits100(mask, c, nvalid); skip_lo = mb.lo; skip_hi = mb.hi; }
    if (lane < 10u) sts64_if(pacc_addr + 512u + 8u * lane, (uint32_t)c_rot_digit[lane], (uint32_t)(c_rot_digit[lane] >> 32), true);
    if (nvalid < 64u) { skip_hi = ~0ull; skip_lo |= ~((1ull << nvalid) - 1ull); }
    else skip_hi |= ~((1ull << (nvalid - 64u)) - 1ull);
    const uint32_t lt = (1u << lane) - 1u;
    RingState R; R.qb_head = 0; R.qb_cnt = 0; R.qc_head = 0; R.qc_cnt = 0;
#pragma unroll 1
    for (uint32_t x = 0; x < 10u; x++) {
        const uint64_t D1 = decade_prep<KIND>(decade_state_t<KIND>(C1, K.s1, x));   // rotation hoisted for byte kinds
        const uint64_t D2 = decade_prep<KIND>(decade_state_t<KIND>(C2, K.s2, x));
        const uint32_t p0 = 10u * x;                                 // bits [p0, p0+10) of the 128-bit skip set
        const uint64_t sh = (p0 < 64u) ? ((skip_lo >> p0) | (p0 ? (skip_hi << (64u - p0)) : 0ull)) : (skip_hi >> (p0 - 64u));
        const uint32_t skip10 = (uint32_t)sh & 0x3ffu;
        const uint32_t tagx = (lane << 8) | (x << 4);
#pragma unroll 1
        for (uint32_t y = 0; y < 10u; y += 2u) {                     // ---- stage A: two positions per lane (ILP)
            const uint32_t idxA = mod_fast(finish_prep<KIND>(D1, K.s1, y, c_rot_digit[y]), K.fm, K.nm);
            const uint32_t idxB = mod_fast(finish_prep<KIND>(D1, K.s1, y + 1u, c_rot_digit[y + 1u]), K.fm, K.nm);
            const uint32_t bA = probe_bit<PM>(sm_addr, sm_addr1, gl, sm_words, idxA);
            const uint32_t bB = probe_bit<PM>(sm_addr, sm_addr1, gl, sm_words, idxB);
            const bool svA = (bA & ~(skip10 >> y) & 1u) != 0u;
            const bool svB = (bB & ~(skip10 >> (y + 1u)) & 1u) != 0u;
#pragma unroll 1
            for (uint32_t j = 0; j < 2u; j++) {                      // push survivors, then run B / C when a batch is ready
                const bool sv = j ? svB : svA;
                const uint32_t b = __ballot_sync(0xffffffffu, sv);
                sts128_if(qb_addr + 16u * ((R.qb_head + R.qb_cnt + __popc(b & lt)) & (Q2_RING - 1)), j ? idxB : idxA,
                          tagx | (y + j), (uint32_t)D2, (uint32_t)(D2 >> 32), sv);
                R.qb_cnt += __popc(b);
                drain_stages<KIND, FKT, PM>(K, sm_addr, sm_addr1, gl, sm_words, qb_addr, qc_addr, pacc_addr, lane, lt, CA, R, false);
            }
        }
    }
#pragma unroll 1
    while (R.qb_cnt | R.qc_cnt)                                      // end of the slab: drain what is left
        drain_stages<KIND, FKT, PM>(K, sm_addr, sm_addr1, gl, sm_words, qb_addr, qc_addr, pacc_addr, lane, lt, CA, R, true);
    __syncwarp();
    uint4 acc = lds128(pacc_addr + 16u * lane);
    sts128_if(pacc_addr + 16u * lane, 0u, 0u, 0u, 0u, true);
    if (active) {
        if (mask != nullptr) {                                       // known members pass (no false negatives); reloaded to save registers
            const Bits128 mb = load_bits100(mask, c, nvalid);
            acc.x |= (uint32_t)mb.lo; acc.y |= (uint32_t)(mb.lo >> 32); acc.z |= (uint32_t)mb.hi; acc.w |= (uint32_t)(mb.hi >> 32);
        }
        pass4[c] = acc;
    }
    __syncwarp();
}

// ------------------------------------------------------------------------------------------
// K3 (decade tiles): compaction without a per-position ring push.  A warp evaluates stage A for a
// whole decade (or half of one) -- TY positions per lane, y a compile-time constant, TY independent
// XXH64 chains per lane (ILP) -- then ONE warp scan of the survivor counts places every survivor in a
// flat per-warp buffer of 4-byte records {idx0, lane, y}.  Stage B consumes the buffer in dense batches
// of 32 and fetches the owner's decade state of seed 2 with a shuffle.  Survivors of B go through the
// small stage-C ring.  (An earlier k_query3 had one buffer per decade; the kernel below is its successor,
// see the comment there.)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void sts32_if(uint32_t addr, uint32_t v, bool p) {
    asm volatile("{\n .reg .pred q;\n setp.ne.u32 q, %2, 0;\n @q st.shared.u32 [%0], %1;\n}" ::"r"(addr), "r"(v), "r"((uint32_t)p) : "memory");
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}

template <int KIND, int PM>
__device__ __forceinline__ void drain_c_ring(const FilterK& K, uint32_t sm_addr, uint32_t sm_addr1, const uint32_t* __restrict__ gl,
                                             uint32_t sm_words, uint32_t qc_addr, uint32_t pacc_addr, uint32_t lane, uint64_t CA,
                                             uint32_t& qc_head, uint32_t& qc_cnt) {
    __syncwarp();
    const uint32_t nc = min(32u, qc_cnt);
    const bool have = lane < nc;
    const uint2 r = lds64(qc_addr + 8u * ((qc_head + lane) & (Q2_RING - 1)));
    qc_head = (qc_head + nc) & (Q2_RING - 1);
    qc_cnt -= nc;
    const uint32_t tag = have ? r.y : 0u;
    const uint32_t owner = (tag >> 8) & 31u;
    const uint64_t CAo = (uint64_t)__shfl_sync(0xffffffffu, (uint32_t)CA, owner) |
                         ((uint64_t)__shfl_sync(0xffffffffu, (uint32_t)(CA >> 32), owner) << 32);
    const uint64_t hA = finish_t<KIND>(decade_state_t<KIND>(CAo, K.sA, (tag >> 4) & 15u), K.sA, tag & 15u);
    const uint32_t pb = probe_bit<PM>(sm_addr, sm_addr1, gl, sm_words, have ? r.x : 0u);
    deliver_pass(pacc_addr, tag, have && (!(hA < K.T) || pb != 0u));
}

template <int KIND, int PM>
__device__ __forceinline__ void query_slab_dispatch(const FilterK& K, uint32_t sm_addr, uint32_t sm_addr1, const uint32_t* __restrict__ gl,
                                                    uint32_t sm_words, const uint32_t* __restrict__ mask, uint32_t n,
                                                    uint32_t slab_c0, uint32_t c_end, uint4* __restrict__ pass4, uint32_t qb,
                                                    uint32_t qc, uint32_t pacc) {
    if (K.fk == 3u) query_slab_staged<KIND, 3, PM>(K, sm_addr, sm_addr1, gl, sm_words, mask, n, slab_c0, c_end, pass4, qb, qc, pacc);
    else if (K.fk == 2u) query_slab_staged<KIND, 2, PM>(K, sm_addr, sm_addr1, gl, sm_words, mask, n, slab_c0, c_end, pass4, qb, qc, pacc);
    else query_slab_staged<KIND, 0, PM>(K, sm_addr, sm_addr1, gl, sm_words, mask, n, slab_c0, c_end, pass4, qb, qc, pacc);
}

template <bool HYBRID>
__global__ void __launch_bounds__(Q2_THREADS, 1) k_query2(const FrameJob* __restrict__ jobs,
                                                          const uint32_t* __restrict__ cent_prefix, int F,
                                                          uint32_t smem_words_cap) {
    extern __shared__ __align__(128) uint32_t dyn[];
    __shared__ __align__(8) uint64_t bar;
    const uint32_t warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31u;   // warp-uniform for the compiler
    uint32_t* wq = dyn + warp * Q2_WARP_WORDS;
    const uint32_t qb = smem_u32(wq), qc = smem_u32(wq + Q2_RING * 4), pacc = smem_u32(wq + Q2_RING * 4 + Q2_RING * 2);
    uint32_t* sbits = dyn + Q2_WARPS * Q2_WARP_WORDS;
    const uint32_t sb_addr = smem_u32(sbits);
    sts128_if(pacc + 16u * lane, 0u, 0u, 0u, 0u, true);
    const uint32_t total = cent_prefix[F];
    const uint32_t lo = (uint32_t)(((uint64_t)total * blockIdx.x) / gridDim.x);
    const uint32_t hi = (uint32_t)(((uint64_t)total * (blockIdx.x + 1)) / gridDim.x);
    if (threadIdx.x == 0) { mbar_init(&bar, 1); fence_mbar_init(); }
    __syncthreads();
    if (lo >= hi) return;
    int f = 0;
    { int a = 0, b = F; while (a < b) { int m = (a + b) >> 1; if (cent_prefix[m + 1] > lo) b = m; else a = m + 1; } f = a; }
    uint32_t parity = 0, g = lo;
    while (g < hi) {
        while (cent_prefix[f + 1] <= g) f++;
        const FrameJob& J = jobs[f];
        const uint32_t seg_end = min(hi, cent_prefix[f + 1]);
        const uint32_t c_begin = g - cent_prefix[f], c_end = seg_end - cent_prefix[f];
        const uint32_t nwords = (J.l + 31u) >> 5;
        const uint32_t sw = min((nwords + 3u) & ~3u, smem_words_cap);
        __syncthreads();
        if (threadIdx.x == 0) {
            fence_proxy_async();
            mbar_expect_tx(&bar, sw * 4u);
            const uint8_t* src = reinterpret_cast<const uint8_t*>(J.bits);
            uint8_t* dst = reinterpret_cast<uint8_t*>(sbits);
            for (uint32_t off = 0; off < sw * 4u; off += 32768u) bulk_g2s(dst + off, src + off, min(32768u, sw * 4u - off), &bar);
        }
        mbar_wait(&bar, parity);
        parity ^= 1u;
        const FilterK K = filter_consts(J);
        uint4* pass4 = reinterpret_cast<uint4*>(J.pass);
        for (uint32_t slab = c_begin + 32u * warp; slab < c_end; slab += 32u * Q2_WARPS) {
            const uint32_t last = min(slab + 31u, c_end - 1u);
            const bool uniform = slab >= 1u && ndigits_u32(slab) == ndigits_u32(last) && K.fk >= 1u && K.fm.fast;
            if (uniform) {
                switch (make_century(slab).kind) {
                case K_4B: query_slab_dispatch<K_4B, (HYBRID ? 1 : 0)>(K, sb_addr, 0u, J.bits, sw, J.mask, J.n, slab, c_end, pass4, qb, qc, pacc); break;
                case K_8B: query_slab_dispatch<K_8B, (HYBRID ? 1 : 0)>(K, sb_addr, 0u, J.bits, sw, J.mask, J.n, slab, c_end, pass4, qb, qc, pacc); break;
                case K_44: query_slab_dispatch<K_44, (HYBRID ? 1 : 0)>(K, sb_addr, 0u, J.bits, sw, J.mask, J.n, slab, c_end, pass4, qb, qc, pacc); break;
                case K_88: query_slab_dispatch<K_88, (HYBRID ? 1 : 0)>(K, sb_addr, 0u, J.bits, sw, J.mask, J.n, slab, c_end, pass4, qb, qc, pacc); break;
                default:   query_slab_dispatch<K_BB, (HYBRID ? 1 : 0)>(K, sb_addr, 0u, J.bits, sw, J.mask, J.n, slab, c_end, pass4, qb, qc, pacc); break;
                }
            } else {                                    // century 0, a digit-count boundary, or floor_k == 0
                const uint32_t c = slab + lane;
                if (c < c_end) {
                    BitView bv; bv.sm = sbits; bv.gl = J.bits; bv.sm_words = sw;
                    const Bits128 r = query_century(bv, K, c, min(100u, J.n - 100u * c));
                    pass4[c] = make_uint4((uint32_t)r.lo, (uint32_t)(r.lo >> 32), (uint32_t)r.hi, (uint32_t)(r.hi >> 32));
                }
            }
        }
        g = seg_end;
    }
}

// ------------------------------------------------------------------------------------------
// K3 (decade tiles: `query_variant` 5, the default).  Same tiles as k_query3 with the slack taken out:
//   * stage B only runs FULL batches of 32 records; the < 32 survivors left over at the end of a tile are moved to the front of
//     the buffer and consumed together with the next tile's (they fetch the decade state of the tile they came from; a record
//     is never carried over more than one tile, and the last tile of a slab drains everything).  k_query3 ran partial
//     batches in every decade.
//   * the survivor scatter is 4 instructions per position (predicate from the survivor bit, record = LOP3, predicated STS,
//     predicated address increment) instead of the 7 the compiler made of `off += p ? 4 : 0`.
//   * TY = 5 (half-decade tiles): records {idx:24, lane:5, y:3} -- filters up to 2^24 bits (8K frames at k* = 4) stay on the
//     tile kernel; with the carry, half tiles no longer pay for half-full batches.
//   * one digit-constant table per CTA instead of one per warp.
//   * full-decade tiles run stage B two full batches at a time (two independent hash-and-probe chains per lane), so a warp
//     waits for the probes of both batches at once (with floor_k = 3, four loads in flight instead of two).
// Results are identical to every other formulation (the variant matrix in tests/test_gpu_parity.py).
// ------------------------------------------------------------------------------------------
#ifndef RBF_Q4_WARPS
#define RBF_Q4_WARPS 28
#endif
constexpr int Q4_WARPS = RBF_Q4_WARPS, Q4_THREADS = 32 * Q4_WARPS;
// Full-decade tiles launch 24 of them by default: stage B keeps two batches in flight, so fewer warps still cover its latency,
// and the scratch of the four warps left out (9.7 KB) holds more of the bit array on chip, which takes probes off the L2 tail.
// Measured faster than 20, 22 and 28 warps at 4K.  Half-decade tiles run stage B one batch deep and keep all Q4_WARPS.
constexpr int Q4_FULL_TILE_WARPS = 24;
constexpr int Q4_TABLE_WORDS = 32;                                     // 10 x uint64 digit constants, padded
template <int TY> struct Q4Cfg {
    static constexpr int BUF = 32 * TY + 32;                            // a tile's survivors (worst case) + carried records (< 32)
    static constexpr int YB = (TY == 10) ? 4 : 3;                       // bits of y inside the tile
    static constexpr int IDXB = 27 - YB;                                // 23 or 24 bits of probe index
    static constexpr int WARP_WORDS = BUF + (Q2_RING * 8 + 32 * 16) / 4;   // tile buffer, C ring, pass accumulators
};

// survivor record scatter: `if (bit) { *off = rec; off += 4; }` as two predicated instructions
__device__ __forceinline__ void scatter_if(uint32_t& off, uint32_t rec, uint32_t bit) {
    asm volatile("{\n .reg .pred q;\n setp.ne.u32 q, %2, 0;\n @q st.shared.u32 [%0], %1;\n @q add.u32 %0, %0, 4;\n}" : "+r"(off) : "r"(rec), "r"(bit) : "memory");
}

template <int KIND, int FKT, int PM, int TY>
__device__ __noinline__ void query_slab_tiled2(const FilterK K, uint32_t sm_addr, const uint32_t* __restrict__ gl, uint32_t sm_words,
                                               const uint32_t* __restrict__ mask, uint32_t n, uint32_t slab_c0, uint32_t c_end,
                                               uint4* __restrict__ pass4, uint32_t buf_addr, uint32_t rb_addr) {
    using Cfg = Q4Cfg<TY>;
    constexpr uint32_t IDXM = (1u << Cfg::IDXB) - 1u;
    const uint32_t qc_addr = buf_addr + 4u * Cfg::BUF, pacc_addr = qc_addr + 8u * Q2_RING;
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t c = slab_c0 + lane;
    const bool active = c < c_end;
    const Century cen = make_century(active ? c : slab_c0);
    const uint64_t C1 = century_state(cen, K.s1), C2 = century_state(cen, K.s2), CA = century_state(cen, K.sA);
    const uint32_t nvalid = active ? min(100u, n - 100u * c) : 0u;
    uint64_t skip_lo = 0, skip_hi = 0;                               // known members and positions beyond n need no hashing
    if (active && mask != nullptr) { const Bits128 mb = load_bits100(mask, c, nvalid); skip_lo = mb.lo; skip_hi = mb.hi; }
    if (nvalid < 64u) { skip_hi = ~0ull; skip_lo |= ~((1ull << nvalid) - 1ull); }
    else skip_hi |= ~((1ull << (nvalid - 64u)) - 1ull);
    const uint32_t lt = (1u << lane) - 1u;
    const uint32_t ltag = lane << Cfg::IDXB;
    uint32_t qc_head = 0, qc_cnt = 0;
    uint32_t rem = 0, xp = 0, yoffp = 0;                             // carried records: count, decade and y offset of their tile
    uint64_t D2p = 0;                                                // ... and that tile's (prepared) decade state of seed 2
#pragma unroll 1
    for (uint32_t x = 0; x < 10u; x++) {
        const uint64_t D1 = decade_prep<KIND>(decade_state_t<KIND>(C1, K.s1, x));
        const uint64_t D2 = decade_prep<KIND>(decade_state_t<KIND>(C2, K.s2, x));
        const uint32_t p0 = 10u * x;
        const uint64_t sh = (p0 < 64u) ? ((skip_lo >> p0) | (p0 ? (skip_hi << (64u - p0)) : 0ull)) : (skip_hi >> (p0 - 64u));
#pragma unroll
        for (int h = 0; h < 10 / TY; h++) {
            // ---- stage A: TY positions per lane, y compile-time, independent hash chains
            uint32_t idx0[TY];
            uint32_t sv = 0;
#pragma unroll
            for (int yy = 0; yy < TY; yy++) {
                const uint32_t y = (uint32_t)(h * TY + yy);
                idx0[yy] = mod_fast(finish_prep<KIND>(D1, K.s1, y, rot_digit_const(y)), K.fm, K.nm);
                sv |= probe_bit<PM>(sm_addr, 0u, gl, sm_words, idx0[yy]) << yy;
            }
            sv &= ~(uint32_t)(sh >> (h * TY)) & ((1u << TY) - 1u);
            // ---- one scan per tile places the survivors behind the carried records
            const uint32_t cnt = __popc(sv);
            uint32_t inc = cnt;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
                if (lane >= (uint32_t)d) inc += t;
            }
            const uint32_t tot2 = rem + __shfl_sync(0xffffffffu, inc, 31);
            uint32_t off = buf_addr + 4u * (rem + inc - cnt);
#pragma unroll
            for (int yy = 0; yy < TY; yy++)
                scatter_if(off, idx0[yy] | ltag | ((uint32_t)yy << (Cfg::IDXB + 5)), sv & (1u << yy));
            __syncwarp();
            // ---- stage B: full batches only (the last tile of the slab drains the rest)
            const bool last_tile = (x == 9u) && (h == 10 / TY - 1);
            uint32_t nproc = last_tile ? tot2 : (tot2 & ~31u);
            if (nproc == 0u && rem != 0u) nproc = tot2;              // a record is carried over one tile at most
            const uint32_t yoff = (uint32_t)(h * TY);
            // the owner's decade state of seed 2 for a record; the batch at b == 0 holds the carried records (g < rem), which
            // fetch the state, x and y offset of the tile they came from
            auto owner_state = [&](const uint32_t b, const uint32_t g, const uint32_t owner, uint32_t& y, uint32_t& xr) {
                uint64_t D2o = (uint64_t)__shfl_sync(0xffffffffu, (uint32_t)D2, owner) |
                               ((uint64_t)__shfl_sync(0xffffffffu, (uint32_t)(D2 >> 32), owner) << 32);
                if (b == 0u && rem != 0u) {                          // warp-uniform
                    const uint64_t D2q = (uint64_t)__shfl_sync(0xffffffffu, (uint32_t)D2p, owner) |
                                         ((uint64_t)__shfl_sync(0xffffffffu, (uint32_t)(D2p >> 32), owner) << 32);
                    if (g < rem) { D2o = D2q; y += yoffp - yoff; xr = xp; }
                }
                return D2o;
            };
            auto h2_step = [&](const uint64_t D2o, const uint32_t y) {
                uint64_t rb = 0;
                if (kind_ends_in_byte<KIND>()) { const uint2 t = lds64(rb_addr + 8u * y); rb = (uint64_t)t.x | ((uint64_t)t.y << 32); }
                return mod_fast(finish_prep<KIND>(D2o, K.s2, y, rb), K.fm, K.nm);
            };
            // a batch's survivors of probes 1..floor_k-1: through the C ring (drained as soon as it holds 32, so it never holds
            // more than 63) or straight into the pass bits
            auto push_c = [&](uint32_t idx, const uint32_t stepm, const uint32_t ok, const uint32_t tag) {
                if (K.has_act) {
                    idx = addmod_fast(idx, stepm, K.fm.m);           // index of probe floor_k
                    const uint32_t b2 = __ballot_sync(0xffffffffu, ok != 0u);
                    sts64_if(qc_addr + 8u * ((qc_head + qc_cnt + __popc(b2 & lt)) & (Q2_RING - 1)), idx, tag, ok != 0u);
                    qc_cnt += __popc(b2);
                    if (qc_cnt >= 32u) drain_c_ring<KIND, PM>(K, sm_addr, 0u, gl, sm_words, qc_addr, pacc_addr, lane, CA, qc_head, qc_cnt);
                } else {
                    deliver_pass(pacc_addr, tag, ok != 0u);
                }
            };
            // one batch of 32 records; FULL batches (all but the last of a slab) carry no per-lane validity logic
            auto stage_b = [&](const uint32_t b, auto full) {
                constexpr bool FULL = decltype(full)::value;
                const uint32_t g = b + lane;
                const bool have = FULL ? true : (g < nproc);
                const uint32_t rec = lds32(buf_addr + 4u * (FULL ? g : min(g, (uint32_t)(Cfg::BUF - 1))));
                const uint32_t owner = (rec >> Cfg::IDXB) & 31u;
                uint32_t y = (rec >> (Cfg::IDXB + 5)) + yoff, xr = x;
                const uint64_t D2o = owner_state(b, g, owner, y, xr);
                if (!have) y = 0u;
                const uint32_t stepm = have ? h2_step(D2o, y) : 0u;
                uint32_t idx = have ? (rec & IDXM) : 0u;
                uint32_t ok = have ? 1u : 0u;
                if (FKT > 0) {
#pragma unroll
                    for (int i = 1; i < FKT; i++) {
                        idx = addmod_fast(idx, stepm, K.fm.m);
                        ok &= probe_bit<PM>(sm_addr, 0u, gl, sm_words, idx);
                    }
                } else {
                    for (uint32_t i = 1; i < K.fk; i++) {
                        idx = addmod_fast(idx, stepm, K.fm.m);
                        ok &= probe_bit<PM>(sm_addr, 0u, gl, sm_words, idx);
                    }
                }
                push_c(idx, stepm, ok, (owner << 8) | (xr << 4) | y);
            };
            // two full batches (records b + lane and b + 32 + lane) as two independent chains, so that a warp waits for the
            // probes of both at once: with part of the array in L2 nearly every batch holds an L2 probe.  Only the first
            // batch can hold carried records (b == 0, g < rem < 32).
            auto stage_b2 = [&](const uint32_t b) {
                const uint32_t rec0 = lds32(buf_addr + 4u * (b + lane)), rec1 = lds32(buf_addr + 4u * (b + 32u + lane));
                const uint32_t own0 = (rec0 >> Cfg::IDXB) & 31u, own1 = (rec1 >> Cfg::IDXB) & 31u;
                uint32_t y0 = (rec0 >> (Cfg::IDXB + 5)) + yoff, x0 = x;
                const uint32_t y1 = (rec1 >> (Cfg::IDXB + 5)) + yoff;
                const uint64_t D2o0 = owner_state(b, b + lane, own0, y0, x0);
                const uint64_t D2o1 = (uint64_t)__shfl_sync(0xffffffffu, (uint32_t)D2, own1) |
                                      ((uint64_t)__shfl_sync(0xffffffffu, (uint32_t)(D2 >> 32), own1) << 32);
                const uint32_t st0 = h2_step(D2o0, y0), st1 = h2_step(D2o1, y1);
                uint32_t idx0 = rec0 & IDXM, idx1 = rec1 & IDXM, ok0 = 1u, ok1 = 1u;
#pragma unroll
                for (int i = 1; i < FKT; i++) {
                    idx0 = addmod_fast(idx0, st0, K.fm.m);
                    idx1 = addmod_fast(idx1, st1, K.fm.m);
                    ok0 &= probe_bit<PM>(sm_addr, 0u, gl, sm_words, idx0);
                    ok1 &= probe_bit<PM>(sm_addr, 0u, gl, sm_words, idx1);
                }
                push_c(idx0, st0, ok0, (own0 << 8) | (x0 << 4) | y0);
                push_c(idx1, st1, ok1, (own1 << 8) | (x << 4) | y1);
            };
            uint32_t bb = 0;
            if (FKT > 0 && TY == 10) {                               // half tiles: a second chain spills at 72 registers
#pragma unroll 1
                for (; bb + 64u <= nproc; bb += 64u) stage_b2(bb);
            }
#pragma unroll 1
            for (; bb + 32u <= nproc; bb += 32u) stage_b(bb, std::true_type{});
            if (bb < nproc) stage_b(bb, std::false_type{});
            // ---- carry the leftover (< 32 records) to the front of the buffer
            const uint32_t nrem = tot2 - nproc;
            if (nrem != 0u) {
                const uint32_t t = lds32(buf_addr + 4u * min(nproc + lane, (uint32_t)(Cfg::BUF - 1)));
                __syncwarp();
                sts32_if(buf_addr + 4u * lane, t, lane < nrem);
            }
            __syncwarp();                                            // the tile buffer is rewritten next
            rem = nrem; xp = x; yoffp = yoff; D2p = D2;
        }
    }
#pragma unroll 1
    while (qc_cnt) drain_c_ring<KIND, PM>(K, sm_addr, 0u, gl, sm_words, qc_addr, pacc_addr, lane, CA, qc_head, qc_cnt);
    __syncwarp();
    uint4 acc = lds128(pacc_addr + 16u * lane);
    sts128_if(pacc_addr + 16u * lane, 0u, 0u, 0u, 0u, true);
    if (active) {
        if (mask != nullptr) {                                       // known members pass (no false negatives)
            const Bits128 mb = load_bits100(mask, c, nvalid);
            acc.x |= (uint32_t)mb.lo; acc.y |= (uint32_t)(mb.lo >> 32); acc.z |= (uint32_t)mb.hi; acc.w |= (uint32_t)(mb.hi >> 32);
        }
        pass4[c] = acc;
    }
    __syncwarp();
}

template <int PM, int TY>
__global__ void __launch_bounds__(Q4_THREADS, 1) k_query4(const FrameJob* __restrict__ jobs, const uint32_t* __restrict__ cent_prefix,
                                                          int F, uint32_t smem_words_cap) {
    using Cfg = Q4Cfg<TY>;
    extern __shared__ __align__(128) uint32_t dyn[];
    __shared__ __align__(8) uint64_t bar;
    const uint32_t warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31u;   // warp-uniform for the compiler
    const uint32_t rb_addr = smem_u32(dyn);                                    // digit constants, one table per CTA
    const uint32_t buf = smem_u32(dyn + Q4_TABLE_WORDS + warp * Cfg::WARP_WORDS);
    const uint32_t pacc = buf + 4u * Cfg::BUF + 8u * Q2_RING;
    const uint32_t nwarps = blockDim.x >> 5;                                   // <= Q4_WARPS (register budget); Q4_FULL_TILE_WARPS by default for full tiles
    uint32_t* sbits = dyn + Q4_TABLE_WORDS + nwarps * Cfg::WARP_WORDS;
    const uint32_t sb_addr = smem_u32(sbits);
    sts128_if(pacc + 16u * lane, 0u, 0u, 0u, 0u, true);
    if (threadIdx.x < 16u) {
        const uint64_t v = threadIdx.x < 10u ? c_rot_digit[threadIdx.x] : 0ull;
        sts64_if(rb_addr + 8u * threadIdx.x, (uint32_t)v, (uint32_t)(v >> 32), true);
    }
    const uint32_t total = cent_prefix[F];
    const uint32_t lo = (uint32_t)(((uint64_t)total * blockIdx.x) / gridDim.x);
    const uint32_t hi = (uint32_t)(((uint64_t)total * (blockIdx.x + 1)) / gridDim.x);
    if (threadIdx.x == 0) { mbar_init(&bar, 1); fence_mbar_init(); }
    __syncthreads();
    if (lo >= hi) return;
    int f = 0;
    { int a = 0, b = F; while (a < b) { int m = (a + b) >> 1; if (cent_prefix[m + 1] > lo) b = m; else a = m + 1; } f = a; }
    uint32_t parity = 0, g = lo;
    while (g < hi) {
        while (cent_prefix[f + 1] <= g) f++;
        const FrameJob& J = jobs[f];
        const uint32_t seg_end = min(hi, cent_prefix[f + 1]);
        const uint32_t c_begin = g - cent_prefix[f], c_end = seg_end - cent_prefix[f];
        const uint32_t nwords = (J.l + 31u) >> 5;
        const uint32_t sw = min((nwords + 3u) & ~3u, smem_words_cap);
        __syncthreads();
        if (threadIdx.x == 0) {
            fence_proxy_async();
            mbar_expect_tx(&bar, sw * 4u);
            const uint8_t* src = reinterpret_cast<const uint8_t*>(J.bits);
            uint8_t* dst = reinterpret_cast<uint8_t*>(sbits);
            for (uint32_t off = 0; off < sw * 4u; off += 32768u) bulk_g2s(dst + off, src + off, min(32768u, sw * 4u - off), &bar);
        }
        mbar_wait(&bar, parity);
        parity ^= 1u;
        const FilterK K = filter_consts(J);
        uint4* pass4 = reinterpret_cast<uint4*>(J.pass);
        for (uint32_t slab = c_begin + 32u * warp; slab < c_end; slab += 32u * nwarps) {
            const uint32_t last = min(slab + 31u, c_end - 1u);
            const bool uniform = slab >= 1u && ndigits_u32(slab) == ndigits_u32(last) && K.fk >= 1u && K.fm.fast && K.fm.m <= (1u << Cfg::IDXB);
            if (uniform) {
#define RBF_TILED2(KD)                                                                                                              \
    if (K.fk == 3u) query_slab_tiled2<KD, 3, PM, TY>(K, sb_addr, J.bits, sw, J.mask, J.n, slab, c_end, pass4, buf, rb_addr);          \
    else if (K.fk == 2u) query_slab_tiled2<KD, 2, PM, TY>(K, sb_addr, J.bits, sw, J.mask, J.n, slab, c_end, pass4, buf, rb_addr);     \
    else query_slab_tiled2<KD, 0, PM, TY>(K, sb_addr, J.bits, sw, J.mask, J.n, slab, c_end, pass4, buf, rb_addr);
                switch (make_century(slab).kind) {
                case K_4B: { RBF_TILED2(K_4B) } break;
                case K_8B: { RBF_TILED2(K_8B) } break;
                case K_44: { RBF_TILED2(K_44) } break;
                case K_88: { RBF_TILED2(K_88) } break;
                default:   { RBF_TILED2(K_BB) } break;
                }
#undef RBF_TILED2
            } else {                                    // century 0, a digit-count boundary, floor_k == 0 or a huge filter
                const uint32_t c = slab + lane;
                if (c < c_end) {
                    BitView bv; bv.sm = sbits; bv.gl = J.bits; bv.sm_words = sw;
                    const Bits128 r = query_century(bv, K, c, min(100u, J.n - 100u * c));
                    pass4[c] = make_uint4((uint32_t)r.lo, (uint32_t)(r.lo >> 32), (uint32_t)r.hi, (uint32_t)(r.hi >> 32));
                }
            }
        }
        g = seg_end;
    }
}
