// rbf_deflate.cuh -- zlib stream encoder (RFC 1950 around RFC 1951) for sm_90a, included by rbf_kernels.cu.
//
// Stream layout (pinned; any inflate decodes it, the bytes are a pure function of the input):
//   78 9C                                       zlib header (deflate, 32 KiB window, default level)
//   per 64 KiB segment of the input (the last one may be shorter), in order:
//       one dynamic-Huffman block, or -- when that would be larger -- stored blocks (LEN <= 65535, so a full
//       segment takes two), all with BFINAL = 0; then an empty stored block (000, pad to the byte, 00 00 FF FF,
//       zlib's sync flush).  Every segment's output is therefore byte-aligned and self-contained: matches never
//       reach before the segment start, so segments are coded in parallel and joined by a byte copy.
//   03 00                                       a final, empty fixed-Huffman block
//   Adler-32 of the whole input, big-endian.
// Empty input gives 78 9C 03 00 00 00 00 01.
//
// k_deflate_segments: one CTA (512 threads, 226 KB of shared memory) per segment.
//   A  one warp builds the hash chains: prev[i] = distance to the previous position whose 3-byte prefix has the
//      same 12-bit hash (0 = none within 32 KiB); __match_any_sync resolves equal hashes inside a 32-position step,
//      so the chains do not depend on scheduling.
//   B  per 4 KiB chunk, every thread takes positions and walks at most kDeflateDepth candidates, keeping the longest
//      match (length 3..258, the nearest one on ties).
//   P  warp 0 walks the greedy parse over the chunk's matches 32 positions at a time and records token starts and
//      match starts as bitmaps.
//   H  all threads histogram the tokens; thread 0 builds length-limited codes (deflate_code_lengths, shared with the
//      host), the run-length coded tree header, and decides between the dynamic block and stored blocks.
//   E  each thread sums the bits of the tokens that start in its 128 positions; a block scan gives bit offsets and
//      every thread writes its codes with shared-memory atomicOr into a zeroed buffer.
// The Adler-32 (s1, s2) sums of each segment come out beside its size; the host combines them in order and
// k_deflate_concat joins the segments, headers and trailers into one contiguous range of streams.
// Included by rbf_kernels.cu inside namespace rbf; kDeflateSeg, deflate_seg_bound, DeflateSeg and DeflateCopy are in
// rbf_kernels.cuh, which rbf_api.cu shares.
#pragma once

static constexpr uint32_t kDeflateWindow = 32768;      // largest distance
static constexpr uint32_t kDeflateDepth = 16;          // chain candidates compared per position
static constexpr uint32_t kDeflateHashBits = 12;
static constexpr uint32_t kDeflateChunk = 4096;        // positions per match-search / parse round
static constexpr uint32_t kDeflateThreads = 512;
static constexpr uint32_t kDeflateMaxSym = 288;

// scratch of deflate_code_lengths (host: stack; device: shared memory)
struct HuffScratch {
    uint64_t key[kDeflateMaxSym];            // (freq << 9 | sym) of the used symbols, sorted ascending
    uint64_t wint[kDeflateMaxSym];           // weights of the internal nodes
    uint16_t parent[2 * kDeflateMaxSym];     // node ids: leaves 0..n-1 (sorted order), internal nodes n..2n-2
    uint8_t depth[2 * kDeflateMaxSym];
    uint32_t cnt[16], next[16];
};

RBF_HD uint32_t deflate_clz(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return (uint32_t)__clz(x);
#else
    return (uint32_t)__builtin_clz(x);
#endif
}

RBF_HD void huff_sift(uint64_t* a, uint32_t root, uint32_t n) {
    for (;;) {
        uint32_t c = 2 * root + 1;
        if (c >= n) return;
        if (c + 1 < n && a[c + 1] > a[c]) c++;
        if (a[root] >= a[c]) return;
        const uint64_t t = a[root]; a[root] = a[c]; a[c] = t;
        root = c;
    }
}

// Length-limited Huffman code lengths.  freqs[nsym] -> lengths[nsym] (0 = no code), every length <= max_bits.
//   * fewer than two used symbols: symbols are added so that exactly two codes of length 1 exist (zlib's rule:
//     stock inflate accepts an incomplete code only as a single length-1 code, and needs a distance code at all);
//   * otherwise a Huffman tree by the two-queue method, ties taken from the leaf queue (the tree of least depth
//     among the optimal ones), depths clamped to max_bits and the Kraft sum restored to exactly 1 by moving leaves
//     one level down from the deepest level that still has room; lengths then go to the symbols by frequency.
// Deterministic; returns 0, or -1 for nsym outside 2..288, max_bits outside 1..15 or more used symbols than
// 2^max_bits codes.
RBF_HD int deflate_code_lengths(const uint32_t* freqs, uint32_t nsym, uint32_t max_bits, uint8_t* lengths, HuffScratch* S) {
    if (nsym < 2 || nsym > kDeflateMaxSym || max_bits < 1 || max_bits > 15) return -1;
    uint32_t n = 0;
    for (uint32_t s = 0; s < nsym; s++) {
        lengths[s] = 0;
        if (freqs[s]) S->key[n++] = ((uint64_t)freqs[s] << 9) | s;
    }
    if (n < 2) {
        const uint32_t a = n ? (uint32_t)(S->key[0] & 511u) : 0u;
        lengths[a] = 1;
        lengths[a == 0 ? 1 : 0] = 1;
        return 0;
    }
    if (n > (1u << max_bits)) return -1;
    for (uint32_t i = n / 2; i-- > 0;) huff_sift(S->key, i, n);        // heap sort, ascending
    for (uint32_t e = n - 1; e > 0; e--) {
        const uint64_t t = S->key[0]; S->key[0] = S->key[e]; S->key[e] = t;
        huff_sift(S->key, 0, e);
    }
    uint32_t li = 0, ii = 0, k = 0;                                     // leaf queue, internal queue, internal count
    for (; k < n - 1; k++) {
        uint64_t w = 0;
        for (int pick = 0; pick < 2; pick++) {
            uint32_t node;
            if (li < n && (ii >= k || (S->key[li] >> 9) <= S->wint[ii])) { w += S->key[li] >> 9; node = li++; }
            else { w += S->wint[ii]; node = n + ii++; }
            S->parent[node] = (uint16_t)(n + k);
        }
        S->wint[k] = w;
    }
    const uint32_t root = 2 * n - 2;
    S->depth[root] = 0;
    for (uint32_t v = root; v-- > 0;) {                                 // parents have larger ids than their children
        const uint32_t d = S->depth[S->parent[v]] + 1u;
        S->depth[v] = (uint8_t)(d > 255u ? 255u : d);
    }
    uint32_t* bl_count = S->cnt;
    for (uint32_t b = 0; b < 16; b++) bl_count[b] = 0;
    uint32_t total = 0;                                                 // Kraft sum in units of 2^-max_bits
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t d = S->depth[i] > max_bits ? max_bits : S->depth[i];
        bl_count[d]++;
        total += 1u << (max_bits - d);
    }
    while (total > (1u << max_bits)) {                                  // each step lowers the sum by exactly one unit
        bl_count[max_bits]--;
        for (uint32_t b = max_bits - 1; b > 0; b--)
            if (bl_count[b]) { bl_count[b]--; bl_count[b + 1] += 2; break; }
        total--;
    }
    uint32_t b = max_bits;                                              // least frequent symbols get the longest codes
    for (uint32_t i = 0; i < n; i++) {
        while (bl_count[b] == 0) b--;
        bl_count[b]--;
        lengths[S->key[i] & 511u] = (uint8_t)b;
    }
    return 0;
}

// canonical codes, bit-reversed for deflate's LSB-first bit order
RBF_HD void deflate_canonical(const uint8_t* lengths, uint32_t nsym, uint16_t* codes, HuffScratch* S) {
    uint32_t *bl_count = S->cnt, *next = S->next;
    for (uint32_t b = 0; b < 16; b++) bl_count[b] = 0;
    for (uint32_t s = 0; s < nsym; s++) bl_count[lengths[s]]++;
    bl_count[0] = 0;
    uint32_t code = 0;
    for (uint32_t b = 1; b < 16; b++) { code = (code + bl_count[b - 1]) << 1; next[b] = code; }
    for (uint32_t s = 0; s < nsym; s++) {
        const uint32_t len = lengths[s];
        codes[s] = 0;
        if (!len) continue;
        uint32_t c = next[len]++, r = 0;
        for (uint32_t i = 0; i < len; i++) { r = (r << 1) | (c & 1u); c >>= 1; }
        codes[s] = (uint16_t)r;
    }
}

// RFC 1951 3.2.5: length 3..258 -> symbol 257..285 and extra bits; distance 1..32768 -> symbol 0..29 and extra bits
RBF_HD uint32_t deflate_len_sym(uint32_t len) {
    const uint32_t l = len - 3u;
    if (len == 258u) return 285u;
    if (l < 8u) return 257u + l;
    const uint32_t nb = 31u - deflate_clz(l) - 2u;
    return 257u + 4u * (nb + 1u) + ((l >> nb) - 4u);
}
RBF_HD uint32_t deflate_len_extra_bits(uint32_t sym) { return (sym >= 265u && sym < 285u) ? (sym - 261u) / 4u : 0u; }
RBF_HD uint32_t deflate_dist_sym(uint32_t dist) {
    const uint32_t d = dist - 1u;
    if (d < 4u) return d;
    const uint32_t nb = 31u - deflate_clz(d) - 1u;
    return 2u * (nb + 1u) + ((d >> nb) & 1u);
}
RBF_HD uint32_t deflate_dist_extra_bits(uint32_t sym) { return sym < 4u ? 0u : sym / 2u - 1u; }


// shared-memory layout of k_deflate_segments (bytes)
static constexpr uint32_t kDzIn = 0;                                  // input, + 16 B of zero padding
static constexpr uint32_t kDzPrev = kDzIn + kDeflateSeg + 16;        // uint16 prev distance per position
static constexpr uint32_t kDzRes = kDzPrev + 2 * kDeflateSeg;         // phase A: uint32 head[4096]; B/P: uint32 match per chunk position
static constexpr uint32_t kDzStart = kDzRes + 4 * kDeflateChunk;      // token-start bitmap
static constexpr uint32_t kDzMatch = kDzStart + kDeflateSeg / 8;      // match-start bitmap
static constexpr uint32_t kDzHist = kDzMatch + kDeflateSeg / 8;       // uint32 hist_ll[286] + hist_d[30]
static constexpr uint32_t kDzMisc = kDzHist + 4 * 320;                // uint64 misc[32]
static constexpr uint32_t kDzBytes = kDzMisc + 8 * 32;
// after the parse the prev region is free: output words, then the code tables
static constexpr uint32_t kDzOut = kDzPrev;
static constexpr uint32_t kDzOutBytes = kDeflateSeg + 64;
static constexpr uint32_t kDzTab = kDzPrev + kDzOutBytes;

struct DeflateTables {
    uint8_t ll_len[kDeflateMaxSym], d_len[32], cl_len[20];
    uint16_t ll_code[kDeflateMaxSym], d_code[32], cl_code[20];
    uint8_t lens[320];                    // ll lengths then distance lengths, as the header codes them
    uint8_t rle_sym[320], rle_ext[320];
    uint32_t cl_freq[20];
    HuffScratch hs;
};
static_assert(kDzTab + sizeof(DeflateTables) <= kDzRes, "deflate tables overflow the prev region");
static_assert(kDzBytes <= 232448, "deflate shared memory exceeds a CTA");

__constant__ uint8_t kDeflateClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

enum { kDmAdlA = 0, kDmAdlB = 1, kDmMode = 2, kDmHdrBits = 3, kDmBodyBits = 4, kDmBytes = 5, kDmWarp = 8 };   // misc slots

__device__ __forceinline__ uint32_t dz_ld4(const uint8_t* in, uint32_t p) {    // 4 bytes at any offset (little endian)
    const uint32_t* w = reinterpret_cast<const uint32_t*>(in);
    return __funnelshift_r(w[p >> 2], w[(p >> 2) + 1], (p & 3u) * 8u);
}

struct DzBits {                                      // LSB-first bit writer into a zeroed shared buffer
    uint32_t* out;
    uint32_t word, n;
    uint64_t acc;
    __device__ __forceinline__ DzBits(uint32_t* o, uint32_t bitpos) : out(o), word(bitpos >> 5), n(bitpos & 31u), acc(0) {}
    __device__ __forceinline__ void put(uint32_t v, uint32_t nb) {
        acc |= (uint64_t)v << n;
        n += nb;
        if (n >= 32u) { atomicOr(out + word, (uint32_t)acc); word++; acc >>= 32; n -= 32u; }
    }
    __device__ __forceinline__ void flush() { if (n) atomicOr(out + word, (uint32_t)acc); }
};

// bits of the token starting at p (match info from the search results in global memory)
__device__ __forceinline__ uint32_t dz_token_bits(const DeflateTables* T, const uint8_t* in, const uint32_t* res_g, uint32_t p,
                                                   bool match) {
    if (!match) return T->ll_len[in[p]];
    const uint32_t r = res_g[p];
    const uint32_t ls = deflate_len_sym(r & 0xffffu), ds = deflate_dist_sym(r >> 16);
    return T->ll_len[ls] + deflate_len_extra_bits(ls) + T->d_len[ds] + deflate_dist_extra_bits(ds);
}

// thread 0: trees, header and the size decision.  Returns the dynamic block's header bits; writes the header.
__device__ void dz_build_block(DeflateTables* T, const uint32_t* hist, uint64_t* misc, uint32_t* out, uint32_t L) {
    const uint32_t* hl = hist;
    const uint32_t* hd = hist + 286;
    deflate_code_lengths(hl, 286, 15, T->ll_len, &T->hs);
    deflate_code_lengths(hd, 30, 15, T->d_len, &T->hs);
    uint32_t hlit = 286, hdist = 30;
    while (hlit > 257 && !T->ll_len[hlit - 1]) hlit--;
    while (hdist > 1 && !T->d_len[hdist - 1]) hdist--;
    for (uint32_t i = 0; i < hlit; i++) T->lens[i] = T->ll_len[i];
    for (uint32_t i = 0; i < hdist; i++) T->lens[hlit + i] = T->d_len[i];
    const uint32_t total = hlit + hdist;
    uint32_t nr = 0;
    for (uint32_t i = 0; i < 20; i++) T->cl_freq[i] = 0;
    for (uint32_t i = 0; i < total;) {                                   // run-length code of the lengths (16 / 17 / 18)
        const uint32_t v = T->lens[i];
        uint32_t run = 1;
        while (i + run < total && T->lens[i + run] == v) run++;
        if (v == 0) {
            while (run >= 11) { const uint32_t r = run < 138 ? run : 138; T->rle_sym[nr] = 18; T->rle_ext[nr++] = (uint8_t)(r - 11); run -= r; i += r; }
            if (run >= 3) { T->rle_sym[nr] = 17; T->rle_ext[nr++] = (uint8_t)(run - 3); i += run; run = 0; }
        } else {
            T->rle_sym[nr] = (uint8_t)v; T->rle_ext[nr++] = 0; i++; run--;
            while (run >= 3) { const uint32_t r = run < 6 ? run : 6; T->rle_sym[nr] = 16; T->rle_ext[nr++] = (uint8_t)(r - 3); run -= r; i += r; }
        }
        while (run > 0) { T->rle_sym[nr] = (uint8_t)v; T->rle_ext[nr++] = 0; i++; run--; }
    }
    for (uint32_t i = 0; i < nr; i++) T->cl_freq[T->rle_sym[i]]++;
    deflate_code_lengths(T->cl_freq, 19, 7, T->cl_len, &T->hs);
    uint32_t hclen = 19;
    while (hclen > 4 && !T->cl_len[kDeflateClOrder[hclen - 1]]) hclen--;
    deflate_canonical(T->ll_len, 286, T->ll_code, &T->hs);
    deflate_canonical(T->d_len, 30, T->d_code, &T->hs);
    deflate_canonical(T->cl_len, 19, T->cl_code, &T->hs);
    uint64_t hdr = 3 + 5 + 5 + 4 + 3ull * hclen, body = 0;
    for (uint32_t i = 0; i < nr; i++) {
        const uint32_t s = T->rle_sym[i];
        hdr += T->cl_len[s] + (s == 16 ? 2u : s == 17 ? 3u : s == 18 ? 7u : 0u);
    }
    for (uint32_t s = 0; s < 286; s++) body += (uint64_t)hl[s] * (T->ll_len[s] + deflate_len_extra_bits(s));
    for (uint32_t s = 0; s < 30; s++) body += (uint64_t)hd[s] * (T->d_len[s] + deflate_dist_extra_bits(s));
    const uint64_t dyn_bytes = (hdr + body + 3 + 7) / 8 + 4;            // + the sync flush (000, pad, 00 00 FF FF)
    const uint32_t dynamic = dyn_bytes <= deflate_seg_bound(L) && dyn_bytes <= kDeflateSeg;
    misc[kDmMode] = dynamic;
    misc[kDmHdrBits] = hdr;
    misc[kDmBodyBits] = body;
    misc[kDmBytes] = dynamic ? dyn_bytes : deflate_seg_bound(L);
    if (!dynamic) return;
    DzBits w(out, 0);
    w.put(4u, 3);                                                        // BFINAL 0, BTYPE 10
    w.put(hlit - 257u, 5); w.put(hdist - 1u, 5); w.put(hclen - 4u, 4);
    for (uint32_t i = 0; i < hclen; i++) w.put(T->cl_len[kDeflateClOrder[i]], 3);
    for (uint32_t i = 0; i < nr; i++) {
        const uint32_t s = T->rle_sym[i];
        w.put(T->cl_code[s], T->cl_len[s]);
        if (s >= 16) w.put(T->rle_ext[i], s == 16 ? 2u : s == 17 ? 3u : 7u);
    }
    w.flush();
}

// One CTA per segment.  res_g: kDeflateSeg uint32 per CTA (match per position); sizes[b]: coded bytes;
// adler[2b], adler[2b+1]: the segment's (s1, s2) sums mod 65521 starting from (0, 0); *err |= 1 on a region overflow,
// |= 2 on an internal size mismatch (nothing is written past a region either way).
__global__ void __launch_bounds__(kDeflateThreads, 1)
k_deflate_segments(const DeflateSeg* __restrict__ segs, uint32_t* __restrict__ res_all, uint32_t* __restrict__ sizes,
                   uint32_t* __restrict__ adler, uint32_t* __restrict__ err) {
    extern __shared__ __align__(16) uint8_t dz_smem[];
    uint8_t* in = dz_smem + kDzIn;
    uint16_t* prev = reinterpret_cast<uint16_t*>(dz_smem + kDzPrev);
    uint32_t* res = reinterpret_cast<uint32_t*>(dz_smem + kDzRes);
    uint32_t* sbits = reinterpret_cast<uint32_t*>(dz_smem + kDzStart);
    uint32_t* mbits = reinterpret_cast<uint32_t*>(dz_smem + kDzMatch);
    uint32_t* hist = reinterpret_cast<uint32_t*>(dz_smem + kDzHist);
    unsigned long long* misc = reinterpret_cast<unsigned long long*>(dz_smem + kDzMisc);
    uint32_t* outw = reinterpret_cast<uint32_t*>(dz_smem + kDzOut);
    DeflateTables* T = reinterpret_cast<DeflateTables*>(dz_smem + kDzTab);
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const DeflateSeg sg = segs[blockIdx.x];
    const uint32_t L = sg.len;
    uint32_t* res_g = res_all + (size_t)blockIdx.x * kDeflateSeg;
    if (L == 0) {
        if (tid == 0) { sizes[blockIdx.x] = 0; adler[2 * blockIdx.x] = 0; adler[2 * blockIdx.x + 1] = 0; }
        return;
    }

    // ---- load, Adler sums, initialise
    if ((reinterpret_cast<uintptr_t>(sg.src) & 15u) == 0) {
        const uint4* s4 = reinterpret_cast<const uint4*>(sg.src);
        for (uint32_t q = tid; q < L / 16u; q += kDeflateThreads) reinterpret_cast<uint4*>(in)[q] = s4[q];
        for (uint32_t i = (L & ~15u) + tid; i < L; i += kDeflateThreads) in[i] = sg.src[i];
    } else {
        for (uint32_t i = tid; i < L; i += kDeflateThreads) in[i] = sg.src[i];
    }
    for (uint32_t i = L + tid; i < L + 16u; i += kDeflateThreads) in[i] = 0;
    for (uint32_t h = tid; h < (1u << kDeflateHashBits); h += kDeflateThreads) res[h] = 0xffffffffu;
    for (uint32_t w = tid; w < kDeflateSeg / 32u; w += kDeflateThreads) { sbits[w] = 0; mbits[w] = 0; }
    for (uint32_t s = tid; s < 320u; s += kDeflateThreads) hist[s] = (s == 256u);   // end-of-block code
    if (tid < 32u) misc[tid] = 0;
    __syncthreads();
    {
        unsigned long long a = 0, b = 0;
        for (uint32_t i = tid; i < L; i += kDeflateThreads) { a += in[i]; b += (unsigned long long)(L - i) * in[i]; }
        for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
        if (lane == 0) { atomicAdd(&misc[kDmAdlA], a); atomicAdd(&misc[kDmAdlB], b); }
    }

    // ---- A: hash chains (one warp, 32 positions per step)
    if (warp == 0) {
        const uint32_t lt = (1u << lane) - 1u, gt = ~lt & ~(1u << lane);
        for (uint32_t base = 0; base < L; base += 32u) {
            const uint32_t i = base + lane;
            const bool valid = i + 2u < L;
            const uint32_t h = valid ? (((dz_ld4(in, i) & 0xffffffu) * 2654435761u) >> (32 - kDeflateHashBits)) : (0x10000u + lane);
            const uint32_t m = __match_any_sync(0xffffffffu, h);
            const uint32_t hv = valid ? res[h] : 0xffffffffu;
            __syncwarp();
            if (i < L) {
                uint32_t pd = 0;
                if (valid) {
                    const uint32_t low = m & lt;
                    if (low) pd = lane - (31u - __clz(low));
                    else if (hv != 0xffffffffu && i - hv <= kDeflateWindow) pd = i - hv;
                }
                prev[i] = (uint16_t)pd;
                if (valid && !(m & gt)) res[h] = i;
            }
            __syncwarp();
        }
    }
    __syncthreads();

    // ---- B + P per chunk
    uint32_t pos = 0;                                                    // parse position (warp 0, uniform)
    for (uint32_t cb = 0; cb < L; cb += kDeflateChunk) {
        for (uint32_t q = tid; q < kDeflateChunk; q += kDeflateThreads) {
            const uint32_t i = cb + q;
            uint32_t best = 0, blen = 0;
            if (i < L) {
                const uint32_t maxlen = (L - i) < 258u ? (L - i) : 258u;
                uint32_t d = maxlen >= 3u ? prev[i] : 0u, j = i - d;
                for (uint32_t step = 0; d != 0 && i - j <= kDeflateWindow && step < kDeflateDepth; step++) {
                    if (blen == 0 || in[j + blen] == in[i + blen]) {
                        uint32_t len = 0;
                        while (len < maxlen) {
                            const uint32_t x = dz_ld4(in, i + len) ^ dz_ld4(in, j + len);
                            if (x) { len += (uint32_t)(__ffs(x) - 1) >> 3; break; }
                            len += 4u;
                        }
                        if (len > maxlen) len = maxlen;
                        if (len >= 3u && len > blen) { blen = len; best = len | ((i - j) << 16); if (len == maxlen) break; }
                    }
                    d = prev[j];
                    j -= d;
                }
                res_g[i] = best;
            }
            res[q] = best;
        }
        __syncthreads();
        if (warp == 0) {
            const uint32_t wend = ((cb + kDeflateChunk < L ? cb + kDeflateChunk : L) + 31u) >> 5;
            for (uint32_t w = cb >> 5; w < wend; w++) {
                const uint32_t base = w << 5;
                const uint32_t r = res[base - cb + lane];
                const uint32_t has = __ballot_sync(0xffffffffu, r != 0u);
                uint32_t sb = 0, mb = 0, p = pos;
                while (p < base + 32u) {
                    const uint32_t off = p - base;
                    const uint32_t cand = has & (0xffffffffu << off);
                    if (!cand) { sb |= 0xffffffffu << off; p = base + 32u; break; }
                    const uint32_t mo = (uint32_t)__ffs(cand) - 1u;
                    sb |= (0xffffffffu << off) & (0xffffffffu >> (31u - mo));
                    mb |= 1u << mo;
                    p = base + mo + (__shfl_sync(0xffffffffu, r, mo) & 0xffffu);
                }
                if (base + 32u > L) sb &= (1u << (L - base)) - 1u;
                pos = p;
                if (lane == 0) { sbits[w] = sb; mbits[w] = mb; }
            }
        }
        __syncthreads();
    }

    // ---- H: histogram of the tokens starting in this thread's 128 positions
    const uint32_t w0 = tid * (kDeflateSeg / 32u / kDeflateThreads), w1 = w0 + kDeflateSeg / 32u / kDeflateThreads;
    for (uint32_t w = w0; w < w1 && (w << 5) < L; w++) {
        uint32_t sb = sbits[w];
        const uint32_t mb = mbits[w];
        while (sb) {
            const uint32_t b = (uint32_t)__ffs(sb) - 1u, p = (w << 5) + b;
            sb &= sb - 1u;
            if ((mb >> b) & 1u) {
                const uint32_t r = res_g[p];
                atomicAdd(&hist[deflate_len_sym(r & 0xffffu)], 1u);
                atomicAdd(&hist[286u + deflate_dist_sym(r >> 16)], 1u);
            } else {
                atomicAdd(&hist[in[p]], 1u);
            }
        }
    }
    for (uint32_t q = tid; q < kDzOutBytes / 4u; q += kDeflateThreads) outw[q] = 0;
    __syncthreads();
    if (tid == 0) dz_build_block(T, hist, reinterpret_cast<uint64_t*>(misc), outw, L);
    __syncthreads();

    const uint32_t bytes = (uint32_t)misc[kDmBytes];
    uint8_t* dst = sg.out;
    if (misc[kDmMode]) {
        // ---- E: bits per thread, block scan, emit
        uint32_t mybits = 0;
        for (uint32_t w = w0; w < w1 && (w << 5) < L; w++) {
            uint32_t sb = sbits[w];
            const uint32_t mb = mbits[w];
            while (sb) {
                const uint32_t b = (uint32_t)__ffs(sb) - 1u;
                sb &= sb - 1u;
                mybits += dz_token_bits(T, in, res_g, (w << 5) + b, (mb >> b) & 1u);
            }
        }
        uint32_t incl = mybits;
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= (uint32_t)o) incl += v;
        }
        if (lane == 31u) misc[kDmWarp + warp] = incl;
        __syncthreads();
        uint32_t before = 0;
        for (uint32_t v = 0; v < warp; v++) before += (uint32_t)misc[kDmWarp + v];
        const uint32_t hdr = (uint32_t)misc[kDmHdrBits];
        DzBits bw(outw, hdr + before + incl - mybits);
        for (uint32_t w = w0; w < w1 && (w << 5) < L; w++) {
            uint32_t sb = sbits[w];
            const uint32_t mb = mbits[w];
            while (sb) {
                const uint32_t b = (uint32_t)__ffs(sb) - 1u, p = (w << 5) + b;
                sb &= sb - 1u;
                if ((mb >> b) & 1u) {
                    const uint32_t r = res_g[p];
                    const uint32_t len = r & 0xffffu, dist = r >> 16;
                    const uint32_t ls = deflate_len_sym(len), ds = deflate_dist_sym(dist);
                    const uint32_t le = deflate_len_extra_bits(ls), de = deflate_dist_extra_bits(ds);
                    bw.put(T->ll_code[ls], T->ll_len[ls]);
                    if (le) bw.put((len - 3u) & ((1u << le) - 1u), le);
                    bw.put(T->d_code[ds], T->d_len[ds]);
                    if (de) bw.put((dist - 1u) & ((1u << de) - 1u), de);
                } else {
                    const uint32_t s = in[p];
                    bw.put(T->ll_code[s], T->ll_len[s]);
                }
            }
        }
        bw.flush();
        if (tid == kDeflateThreads - 1u) {
            const uint32_t end = hdr + before + incl;                   // every thread's bits, in order
            if ((uint64_t)end != misc[kDmHdrBits] + misc[kDmBodyBits] - T->ll_len[256]) atomicOr(err, 2u);
            DzBits ew(outw, end);
            ew.put(T->ll_code[256], T->ll_len[256]);                     // end of block
            ew.put(0u, 3);                                               // empty stored block, BFINAL 0
            ew.flush();
            const uint32_t fb = (end + T->ll_len[256] + 3u + 7u) >> 3;
            if (fb + 4u != bytes) atomicOr(err, 2u);
            else {                                                       // 00 00 FF FF
                atomicOr(outw + ((fb + 2u) >> 2), 0xffu << (((fb + 2u) & 3u) * 8u));
                atomicOr(outw + ((fb + 3u) >> 2), 0xffu << (((fb + 3u) & 3u) * 8u));
            }
        }
        __syncthreads();
        if (bytes > sg.cap || ((bytes + 3u) & ~3u) > sg.cap) {
            if (tid == 0) atomicOr(err, 1u);
        } else {
            for (uint32_t q = tid; q < (bytes + 3u) / 4u; q += kDeflateThreads) reinterpret_cast<uint32_t*>(dst)[q] = outw[q];
        }
    } else if (bytes > sg.cap) {
        if (tid == 0) atomicOr(err, 1u);
    } else {
        // ---- stored blocks: at most 65535 bytes each, then the sync flush
        const uint32_t first = L > 65535u ? 65535u : L;
        for (uint32_t i = tid; i < L; i += kDeflateThreads) dst[i < first ? 5u + i : 10u + i] = in[i];
        if (tid == 0) {
            auto hdr = [&](uint8_t* h, uint32_t n) { h[0] = 0; h[1] = n & 255u; h[2] = n >> 8; h[3] = ~n & 255u; h[4] = (~n >> 8) & 255u; };
            hdr(dst, first);
            if (L > first) hdr(dst + 5u + first, L - first);
            hdr(dst + bytes - 5u, 0);
        }
    }
    if (tid == 0) {
        sizes[blockIdx.x] = bytes;
        adler[2 * blockIdx.x] = (uint32_t)(misc[kDmAdlA] % 65521ull);
        adler[2 * blockIdx.x + 1] = (uint32_t)(misc[kDmAdlB] % 65521ull);
    }
}

// joins coded segments into consecutive zlib streams: one CTA per segment; headers and trailers as the jobs say
__global__ void __launch_bounds__(256) k_deflate_concat(const DeflateCopy* __restrict__ jobs, uint8_t* __restrict__ dst,
                                                        uint64_t cap, uint32_t* __restrict__ err) {
    const DeflateCopy J = jobs[blockIdx.x];
    const uint64_t hi = J.dst + J.len + ((J.flags & 2u) ? 6u : 0u);
    if (J.dst < ((J.flags & 1u) ? 2u : 0u) || hi > cap) {
        if (threadIdx.x == 0) atomicOr(err, 1u);
        return;
    }
    for (uint32_t i = threadIdx.x; i < J.len; i += blockDim.x) dst[J.dst + i] = J.src[i];
    if (threadIdx.x == 0) {
        if (J.flags & 1u) { dst[J.dst - 2] = 0x78; dst[J.dst - 1] = 0x9c; }
        if (J.flags & 2u) {
            uint8_t* t = dst + J.dst + J.len;
            t[0] = 0x03; t[1] = 0x00;
            t[2] = (uint8_t)(J.adler >> 24); t[3] = (uint8_t)(J.adler >> 16); t[4] = (uint8_t)(J.adler >> 8); t[5] = (uint8_t)J.adler;
        }
    }
}
