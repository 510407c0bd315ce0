// rbf_aux_kernels.cuh -- N1 gather (ivc:810-842), N3 5x5 median (ivc:738), bit packing utilities, explicit item lists (ivc:99-138, rbf:25-182).  Included by rbf_kernels.cu inside namespace rbf.
#pragma once

// ------------------------------------------------------------------------------------------
// N1 (SURVEY 8f): ordered gather of the changed pixels' values (ivc:810-842); N2, the frame rebuilt
// from them, is the K4c sweep (rbf_k4c_apply.cuh).  A pair is cut into `chunks` runs of mask words; a
// first pass counts the set bits of every chunk, then one CTA per (chunk, pair) walks its words in
// order: rank of a set pixel = set bits of the earlier chunks + block scan of the popcounts.
// ------------------------------------------------------------------------------------------
constexpr int GS_MAX_CHUNKS = 64;

__global__ void __launch_bounds__(256) k_mask_chunk_count(const GatherJob* __restrict__ jobs, uint32_t chunks, uint32_t* __restrict__ counts) {
    const GatherJob& J = jobs[blockIdx.y];
    __shared__ uint32_t s_c[8];
    const uint32_t nwords = (J.npix + 31u) >> 5;
    const uint32_t w0 = (uint32_t)(((uint64_t)nwords * blockIdx.x) / chunks), w1 = (uint32_t)(((uint64_t)nwords * (blockIdx.x + 1)) / chunks);
    uint32_t c = 0;
    for (uint32_t w = w0 + threadIdx.x; w < w1; w += blockDim.x) c += __popc(__ldg(J.mask + w));
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
    if ((threadIdx.x & 31) == 0) s_c[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int i = 0; i < 8; i++) t += s_c[i];
        counts[blockIdx.y * chunks + blockIdx.x] = t;
    }
}

template <int PB>
__device__ __forceinline__ void copy_pixel(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src) {
    if (PB == 2) { *reinterpret_cast<uint16_t*>(dst) = *reinterpret_cast<const uint16_t*>(src); return; }
    if (PB == 6) {                                         // three 2-aligned samples
        const uint16_t a = reinterpret_cast<const uint16_t*>(src)[0], b = reinterpret_cast<const uint16_t*>(src)[1], c = reinterpret_cast<const uint16_t*>(src)[2];
        reinterpret_cast<uint16_t*>(dst)[0] = a; reinterpret_cast<uint16_t*>(dst)[1] = b; reinterpret_cast<uint16_t*>(dst)[2] = c;
        return;
    }
#pragma unroll
    for (int q = 0; q < PB; q++) dst[q] = src[q];          // PB = 1 or 3: all loads first, then the stores
}

// Residual coding of the value streams: per sample of S bytes (1, or 2 little-endian), dst = (curr - prev) mod 2^(8S) on the encode
// side and dst = (dst + r) mod 2^(8S) on the decode side.  PB = channels x S; the pair (PB, S) is one of (1,1), (3,1), (2,2), (6,2).
template <int PB, int S>
__device__ __forceinline__ void resid_pixel(uint8_t* __restrict__ dst, const uint8_t* __restrict__ curr, const uint8_t* __restrict__ prev) {
    static_assert((S == 1 || S == 2) && PB % S == 0, "sample bytes");
    if constexpr (S == 2) {
#pragma unroll
        for (int q = 0; q < PB / 2; q++)
            reinterpret_cast<uint16_t*>(dst)[q] = (uint16_t)(reinterpret_cast<const uint16_t*>(curr)[q] - reinterpret_cast<const uint16_t*>(prev)[q]);
    } else {
#pragma unroll
        for (int q = 0; q < PB; q++) dst[q] = (uint8_t)(curr[q] - prev[q]);
    }
}

template <int PB, int S>
__device__ __forceinline__ void add_pixel(uint8_t* __restrict__ dst, const uint8_t* __restrict__ r) {
    static_assert((S == 1 || S == 2) && PB % S == 0, "sample bytes");
    if constexpr (S == 2) {
#pragma unroll
        for (int q = 0; q < PB / 2; q++)
            reinterpret_cast<uint16_t*>(dst)[q] = (uint16_t)(reinterpret_cast<uint16_t*>(dst)[q] + reinterpret_cast<const uint16_t*>(r)[q]);
    } else {
#pragma unroll
        for (int q = 0; q < PB; q++) dst[q] = (uint8_t)(dst[q] + r[q]);
    }
}

// Pixel index of the motion-compensated prediction of pixel px: the pixel its block's (dx, dy) points at, clamped to the frame.
__device__ __forceinline__ size_t motion_src(const int8_t* __restrict__ field, uint32_t W, uint32_t H, uint32_t px) {
    const uint32_t y = px / W, x = px - y * W;
    const uint32_t b = (y / MV_BLOCK) * mv_blocks_x(W) + x / MV_BLOCK;
    const int dx = __ldg(field + 2 * b), dy = __ldg(field + 2 * b + 1);
    const int yy = min(max((int)y + dy, 0), (int)H - 1), xx = min(max((int)x + dx, 0), (int)W - 1);
    return (size_t)yy * W + (uint32_t)xx;
}

// RS = 0: plain gather of the pixels; RS = 1 or 2: residuals against J.prev per sample of RS bytes; MC: against the
// motion-compensated J.prev (J.field, J.width) instead of the co-located pixel
template <int PB, int RS, bool MC = false>
__global__ void __launch_bounds__(1024) k_gather(const GatherJob* __restrict__ jobs, uint32_t chunks, const uint32_t* __restrict__ counts) {
    static_assert(!MC || RS != 0, "motion gathers are residual gathers");
    // set pixels before this chunk; summed before the job is loaded, so that the motion gathers fit 32 registers without spilling
    uint32_t base = 0;
    for (uint32_t i = 0; i < blockIdx.x; i++) base += counts[blockIdx.y * chunks + i];
    const GatherJob J = jobs[blockIdx.y];
    [[maybe_unused]] const uint32_t H = MC ? J.npix / J.width : 0u;
    __shared__ uint32_t s_warp[33];
    const uint32_t nwords = (J.npix + 31u) >> 5;
    const uint32_t w_begin = (uint32_t)(((uint64_t)nwords * blockIdx.x) / chunks), w_end = (uint32_t)(((uint64_t)nwords * (blockIdx.x + 1)) / chunks);
    for (uint32_t w0 = w_begin; w0 < w_end; w0 += blockDim.x) {
        const uint32_t w = w0 + threadIdx.x;
        uint32_t m = (w < w_end) ? __ldg(J.mask + w) : 0u;
        uint32_t tot;
        uint32_t rank = base + block_excl_scan(__popc(m), s_warp, tot);
        while (m) {
            const uint32_t b = __ffs(m) - 1;
            m &= m - 1u;
            const size_t px = ((size_t)w << 5) + b;
            if constexpr (MC) resid_pixel<PB, RS>(J.values + (size_t)rank * PB, J.frame + px * PB, J.prev + motion_src(J.field, J.width, H, (uint32_t)px) * PB);
            else if constexpr (RS != 0) resid_pixel<PB, RS>(J.values + (size_t)rank * PB, J.frame + px * PB, J.prev + px * PB);
            else copy_pixel<PB>(J.values + (size_t)rank * PB, J.frame + px * PB);
            rank++;
        }
        base += tot;
    }
}

// ------------------------------------------------------------------------------------------
// N3 (SURVEY 8f): the 5x5 median of cv2.medianBlur (ivc:738) -- replicated border, 13th smallest of
// the 25 samples -- of one plane.  Rank selection (25 x 25 comparisons) is
// exact for any sample type; the float32 std that follows (ivc:741-744) stays in numpy on the host so
// that the noise estimate is bit-identical to the reference's.
// ------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) k_median5(const T* __restrict__ in, uint32_t H, uint32_t W, T* __restrict__ out) {
    const uint32_t x = blockIdx.x * 32u + (threadIdx.x & 31u), y = blockIdx.y * 8u + (threadIdx.x >> 5);
    if (x >= W || y >= H) return;
    uint32_t v[25];
#pragma unroll
    for (int dy = -2; dy <= 2; dy++) {
        const uint32_t yy = (uint32_t)min(max((int)y + dy, 0), (int)H - 1);
#pragma unroll
        for (int dx = -2; dx <= 2; dx++) {
            const uint32_t xx = (uint32_t)min(max((int)x + dx, 0), (int)W - 1);
            v[(dy + 2) * 5 + (dx + 2)] = (uint32_t)__ldg(in + (size_t)yy * W + xx);
        }
    }
    uint32_t med = 0;
#pragma unroll
    for (int i = 0; i < 25; i++) {
        uint32_t rank = 0;
#pragma unroll
        for (int j = 0; j < 25; j++) rank += (v[j] < v[i] || (v[j] == v[i] && j < i)) ? 1u : 0u;
        if (rank == 12u) med = v[i];
    }
    out[(size_t)y * W + x] = (T)med;
}

// ------------------------------------------------------------------------------------------
// small utilities
// ------------------------------------------------------------------------------------------
__global__ void k_bitrev(uint32_t* __restrict__ w, size_t n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        w[i] = bitrev_bytes(w[i]);
}
// LSB-first packed bits -> one byte per bit (np.uint8 0/1)
__global__ void k_unpack_bits(const uint32_t* __restrict__ w, uint8_t* __restrict__ out, size_t nbits) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nbits; i += (size_t)gridDim.x * blockDim.x)
        out[i] = (uint8_t)((w[i >> 5] >> (i & 31)) & 1u);
}
// one byte per position -> LSB-first packed words.  nonzero = 0: a byte == 1 is set, as the mask test `binary_input[i] == 1`
// (ivc:236); nonzero = 1: any non-zero byte is set, as a Bloom bit array is read (`bit_array[idx] == 0` is unset, ivc:129,135)
__global__ void k_pack_bytes(const uint8_t* __restrict__ in, uint32_t* __restrict__ w, size_t nbits, int nonzero) {
    const size_t nwords = (nbits + 31) >> 5;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nwords; i += (size_t)gridDim.x * blockDim.x) {
        uint32_t v = 0;
        const size_t b0 = i << 5;
        for (uint32_t k = 0; k < 32u && b0 + k < nbits; k++) v |= ((nonzero ? in[b0 + k] != 0 : in[b0 + k] == 1) ? 1u : 0u) << k;
        w[i] = v;
    }
}


// MSB-first (np.packbits order) packed bits -> one byte per bit
__global__ void k_unpack_bits_msb(const uint32_t* __restrict__ w, uint8_t* __restrict__ out, size_t nbits) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nbits; i += (size_t)gridDim.x * blockDim.x)
        out[i] = (uint8_t)((w[i >> 5] >> ((i & 31) ^ 7)) & 1u);
}
__global__ void k_popcount(const uint32_t* __restrict__ w, size_t n, uint32_t* __restrict__ out) {
    uint32_t c = 0;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) c += __popc(w[i]);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}
// per frame: number of 32-bit words in which two packed bit arrays differ
__global__ void k_count_diff(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b, size_t stride_words,
                             size_t nwords, uint32_t* __restrict__ out) {
    const uint32_t* pa = a + (size_t)blockIdx.y * stride_words;
    const uint32_t* pb = b + (size_t)blockIdx.y * stride_words;
    uint32_t c = 0;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nwords; i += (size_t)gridDim.x * blockDim.x)
        c += (pa[i] != pb[i]) ? 1u : 0u;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) c += __shfl_xor_sync(0xffffffffu, c, d);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out + blockIdx.y, c);
}

// ------------------------------------------------------------------------------------------
// explicit-item kernels: RationalBloomFilter.add_index / check_index on a list of indices
// (ivc:99-138), and the string-keyed twin rbf.RationalBloomFilter / StandardBloomFilter
// (rbf:25-41, rbf:103-182).  Bit array is LSB-first in global memory.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t check_hashes_global(const uint32_t* __restrict__ bits, const FilterK& K, uint64_t h1,
                                                        uint64_t h2, uint64_t hA) {
    uint32_t idx = mod_u64(h1, K.fm);
    const uint32_t step = mod_u64(h2, K.fm);
    for (uint32_t i = 0; i < K.fk; i++) {
        if (!((bits[idx >> 5] >> (idx & 31u)) & 1u)) return 0u;
        idx = addmod(idx, step, K.fm.m);
    }
    if (K.has_act && hA < K.T) { if (!((bits[idx >> 5] >> (idx & 31u)) & 1u)) return 0u; }
    return 1u;
}

__global__ void k_items_u32(const FrameJob* __restrict__ job, const uint32_t* __restrict__ items, uint32_t count,
                            uint8_t* __restrict__ result, int insert) {
    const FrameJob& J = *job;
    const FilterK K = filter_consts(J);
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < count; t += gridDim.x * blockDim.x) {
        const uint32_t i = items[t];
        const Century cen = make_century(i / 100u);
        const uint32_t x = (i / 10u) % 10u, y = i % 10u;
        const uint64_t h1 = finish(cen.kind, decade_state(cen, century_state(cen, K.s1), K.s1, x), K.s1, y);
        const uint64_t h2 = finish(cen.kind, decade_state(cen, century_state(cen, K.s2), K.s2, x), K.s2, y);
        const uint64_t hA = K.has_act ? finish(cen.kind, decade_state(cen, century_state(cen, K.sA), K.sA, x), K.sA, y) : 0ull;
        if (insert) insert_hashes(GlobalBits{J.bits}, K, h1, h2, hA);
        else result[t] = (uint8_t)check_hashes_global(J.bits, K, h1, h2, hA);
    }
}

__global__ void k_items_str(const FrameJob* __restrict__ job, const uint8_t* __restrict__ blob,
                            const uint64_t* __restrict__ offs, uint32_t count, uint8_t* __restrict__ result, int insert,
                            int standard_k) {
    const FrameJob& J = *job;
    const FilterK K = filter_consts(J);
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < count; t += gridDim.x * blockDim.x) {
        const uint8_t* s = blob + offs[t];
        const uint32_t len = (uint32_t)(offs[t + 1] - offs[t]);
        if (standard_k > 0) {           // StandardBloomFilter: k independent hashes, seed = i (rbf:25-41)
            uint32_t ok = 1u;
            for (int i = 0; i < standard_k; i++) {
                const uint32_t idx = mod_u64(xxh64_bytes(s, len, (uint64_t)i), K.fm);
                if (insert) atomicOr(J.bits + (idx >> 5), 1u << (idx & 31u));
                else if (!((J.bits[idx >> 5] >> (idx & 31u)) & 1u)) { ok = 0u; break; }
            }
            if (!insert) result[t] = (uint8_t)ok;
        } else {
            const uint64_t h1 = xxh64_bytes(s, len, K.s1), h2 = xxh64_bytes(s, len, K.s2);
            const uint64_t hA = K.has_act ? xxh64_bytes(s, len, K.sA) : 0ull;
            if (insert) insert_hashes(GlobalBits{J.bits}, K, h1, h2, hA);
            else result[t] = (uint8_t)check_hashes_global(J.bits, K, h1, h2, hA);
        }
    }
}

// KAT / debug: mode 0 = xxh64_decimal(item), mode 1 = century/decade/finish route
__global__ void k_hash_debug(const uint32_t* __restrict__ items, uint32_t count, uint64_t seed, uint64_t* __restrict__ out,
                             int mode) {
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < count; t += gridDim.x * blockDim.x) {
        const uint32_t i = items[t];
        if (mode == 0) out[t] = xxh64_decimal(i, seed);
        else {
            const Century cen = make_century(i / 100u);
            out[t] = finish(cen.kind, decade_state(cen, century_state(cen, seed), seed, (i / 10u) % 10u), seed, i % 10u);
        }
    }
}

// ------------------------------------------------------------------------------------------
// Multi-GPU exchange over NVLink peer memory (SURVEY 8e): instead of packing the bit arrays into a send buffer
// and handing it to ncclAllGather, ONE kernel reads each pair's bit array once and stores its slot straight into
// the receive buffer of every rank (peer pointers obtained through CUDA IPC; plain st.global to a peer address is an
// NVLink write).  Completion is a per-source sequence number stored with system-scope release into each rank's flag
// array; the consumer spins on its LOCAL flags with acquire loads (bounded, so a lost peer cannot hang the GPU).
// ------------------------------------------------------------------------------------------
constexpr int PEER_MAX = 16;
struct PeerTable {
    uint32_t* recv[PEER_MAX];      // receive buffer of rank r as mapped in THIS process (own entry: the local buffer)
    uint32_t* flags[PEER_MAX];     // flag array of rank r (one uint32 per source rank)
};

__global__ void __launch_bounds__(256) k_push_slots(const uint32_t* __restrict__ bits, size_t stride_w, uint32_t slot_w, uint32_t pairs,
                                                    PeerTable pt, int nranks, size_t dst_off_w) {
    // 16-byte granules: slot_w and stride_w are multiples of 4 words and every buffer is 16 B aligned (checked by the host)
    const uint32_t slot_q = slot_w >> 2;
    const size_t total = (size_t)pairs * slot_q;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t pair = (uint32_t)(i / slot_q), q = (uint32_t)(i - (size_t)pair * slot_q);
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(bits + (size_t)pair * stride_w) + q);
#pragma unroll 1
        for (int r = 0; r < nranks; r++) reinterpret_cast<uint4*>(pt.recv[r] + dst_off_w)[i] = v;   // peer address: an NVLink write
    }
}
// after k_push_slots on the same stream: tell every rank that this rank's slots of exchange `seq` have landed
__global__ void k_peer_signal(PeerTable pt, int nranks, int rank, uint32_t seq) {
    const int r = threadIdx.x;
    if (r < nranks) {
        __threadfence_system();
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(pt.flags[r] + rank), "r"(seq) : "memory");
    }
}
// wait until every source rank has signalled exchange `seq` (sequence numbers only grow); *err = 1 on time-out
__global__ void k_peer_wait(const uint32_t* __restrict__ flags, int nranks, uint32_t seq, long long timeout_cycles, uint32_t* err) {
    const int r = threadIdx.x;
    if (r < nranks) {
        const long long t0 = clock64();
        uint32_t v;
        do {
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + r) : "memory");
            if ((int32_t)(v - seq) >= 0) break;
            if (clock64() - t0 > timeout_cycles) { *err = 1u; break; }
            __nanosleep(200);
        } while (true);
    }
    __threadfence_system();
}
