// rbf_inflate.cuh -- inflate of the zlib streams rbf_deflate.cuh writes, included by rbf_kernels.cu after rbf_deflate.cuh.
//
// The device coder's layout (rbf_deflate.cuh) makes every 64 KiB segment self-contained and ends each one with an empty stored
// block, 00 00 FF FF.  So every segment start is offset 2 or an offset that follows 00 00 FF FF, and segments inflate
// independently once their starts are known:
//   k_inflate_scan      every candidate start of each stream: offset 2 and each offset after 00 00 FF FF, below the trailer
//   k_inflate_segments  inflate_segment once per candidate, each into its own 64 KiB slot (one thread per candidate: lane 0 of
//                       a one-warp CTA, so that candidates never share a warp and diverge against each other)
// The host then follows the chain from offset 2 through the accepted candidates' end offsets, checks the trailer and the Adler-32,
// and k_deflate_concat copies the chain's slots into place.  A candidate whose data merely contains 00 00 FF FF (a stored
// segment) is decoded and ignored.  Streams outside the layout are declined and inflated by the caller on the host.
// InflateScanJob, InflateSegResult and the status codes are in rbf_kernels.cuh, which rbf_api.cu shares.
#pragma once

static constexpr uint32_t kInflateLitRoot = 9;         // first-level lookup bits of the literal/length code
static constexpr uint32_t kInflateDistRoot = 8;        // and of the distance code

// decode tables of one segment (host: stack; device: shared memory).  fast[] holds (symbol << 4 | length) of every code of at most
// root bits, replicated over the unused high bits; 0 sends the decode to the canonical walk over count[] / sym[] (longer codes,
// and the unused codes of an incomplete one, which the walk rejects)
struct InflateScratch {
    uint16_t lit_fast[1u << kInflateLitRoot];
    uint16_t dist_fast[1u << kInflateDistRoot];
    uint16_t lit_count[16], dist_count[16], cl_count[16];
    uint16_t lit_sym[288], dist_sym[32], cl_sym[19];
    uint8_t lens[320];
};

struct InflateBits {                                   // LSB-first bit reader; never reads at or past in[n]
    const uint8_t* in;
    uint32_t n, pos, cnt;
    uint64_t buf;
};

RBF_HD void ib_fill(InflateBits& B) {
    while (B.cnt <= 56u && B.pos < B.n) { B.buf |= (uint64_t)B.in[B.pos++] << B.cnt; B.cnt += 8u; }
}
RBF_HD bool ib_need(InflateBits& B, uint32_t k) {
    if (B.cnt < k) ib_fill(B);
    return B.cnt >= k;
}
RBF_HD uint32_t ib_take(InflateBits& B, uint32_t k) {
    const uint32_t v = (uint32_t)(B.buf & ((1ull << k) - 1ull));
    B.buf >>= k;
    B.cnt -= k;
    return v;
}

// Canonical code of n symbols with lengths lens[0..n) -> count / sym (and fast[1 << root] when fast != NULL).  Judged as zlib's
// inflate_table judges: an over-subscribed set is refused; an incomplete one is refused unless it is a single code of length 1
// and the set is not the code-length code (complete == false allows that).  A set without any code is accepted only when
// complete == false (a block may have no distance codes); decoding from it then fails.  Returns 0 or -1.
RBF_HD int inflate_build(const uint8_t* lens, uint32_t n, uint16_t* count, uint16_t* sym, uint16_t* fast, uint32_t root,
                         bool complete) {
    for (uint32_t b = 0; b < 16; b++) count[b] = 0;
    for (uint32_t s = 0; s < n; s++) count[lens[s]]++;
    count[0] = 0;
    uint32_t maxlen = 0;
    for (uint32_t b = 1; b < 16; b++) if (count[b]) maxlen = b;
    if (fast) for (uint32_t i = 0; i < (1u << root); i++) fast[i] = 0;
    if (maxlen == 0) return complete ? -1 : 0;
    int left = 1;
    for (uint32_t b = 1; b < 16; b++) {
        left <<= 1;
        left -= count[b];
        if (left < 0) return -1;
    }
    if (left > 0 && (complete || maxlen != 1)) return -1;
    uint16_t offs[16];
    offs[1] = 0;
    for (uint32_t b = 1; b < 15; b++) offs[b + 1] = (uint16_t)(offs[b] + count[b]);
    for (uint32_t s = 0; s < n; s++) if (lens[s]) sym[offs[lens[s]]++] = (uint16_t)s;
    if (!fast) return 0;
    uint32_t code = 0, idx = 0;                        // canonical codes in sym order, bit-reversed into the table
    for (uint32_t b = 1; b <= root && b <= maxlen; b++) {
        for (uint32_t k = 0; k < count[b]; k++, idx++, code++) {
            uint32_t r = 0;
            for (uint32_t i = 0; i < b; i++) r |= ((code >> i) & 1u) << (b - 1u - i);
            for (uint32_t f = r; f < (1u << root); f += 1u << b) fast[f] = (uint16_t)((sym[idx] << 4) | b);
        }
        code <<= 1;
    }
    return 0;
}

// One symbol: -1 when the input ends inside the code, -2 for a bit pattern that is not a code
RBF_HD int inflate_decode(InflateBits& B, const uint16_t* count, const uint16_t* sym, const uint16_t* fast, uint32_t root) {
    ib_fill(B);
    if (fast) {
        const uint32_t e = fast[B.buf & ((1u << root) - 1u)];
        if (e) {
            if ((e & 15u) > B.cnt) return -1;
            ib_take(B, e & 15u);
            return (int)(e >> 4);
        }
    }
    int code = 0, first = 0, index = 0;
    for (uint32_t len = 1; len < 16; len++) {
        if (len > B.cnt) return -1;
        code |= (int)((B.buf >> (len - 1u)) & 1u);
        const int c = count[len];
        if (code - c < first) { ib_take(B, len); return (int)sym[index + (code - first)]; }
        index += c;
        first = (first + c) << 1;
        code <<= 1;
    }
    return -2;
}

// Inflates one segment of the device layout starting at in[0], with `avail` bytes of the stream left, into out[0..65536).
// Accepted: blocks with BFINAL 0 (dynamic Huffman or stored), ended by the first empty stored block.  Everything else is refused
// with a status, without reading past in[avail) or writing past out[65536).  res: status, bytes consumed (through the closing
// 00 00 FF FF), bytes produced and the Adler-32 sums (s2 << 16 | s1) of the output, from (0, 0), as k_deflate_segments gives them.
RBF_HD void inflate_segment(const uint8_t* in, uint64_t avail, uint8_t* out, InflateScratch* S, InflateSegResult* res) {
    const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    InflateBits B;
    B.in = in; B.n = avail > 0xfffffff0ull ? 0xfffffff0u : (uint32_t)avail; B.pos = 0; B.cnt = 0; B.buf = 0;
    uint32_t p = 0, a = 0, status = kInflateOk;
    uint64_t b = 0;
    for (;;) {
        if (!ib_need(B, 3)) { status = kInflateTruncated; break; }
        const uint32_t h = ib_take(B, 3);
        if (h & 1u) { status = kInflateFinal; break; }
        const uint32_t type = h >> 1;
        if (type == 0) {                                                      // stored: to the byte, LEN, NLEN, data
            ib_take(B, B.cnt & 7u);
            B.pos -= B.cnt >> 3; B.cnt = 0; B.buf = 0;
            if (B.n - B.pos < 4u) { status = kInflateTruncated; break; }
            const uint32_t len = in[B.pos] | (uint32_t)in[B.pos + 1] << 8, nlen = in[B.pos + 2] | (uint32_t)in[B.pos + 3] << 8;
            B.pos += 4;
            if (len != (~nlen & 0xffffu)) { status = kInflateStoredLen; break; }
            if (len == 0) break;                                              // the segment's end
            if (len > B.n - B.pos) { status = kInflateTruncated; break; }
            if (len > kDeflateSeg - p) { status = kInflateOutputFull; break; }
            for (uint32_t i = 0; i < len; i++) { const uint8_t v = in[B.pos + i]; out[p + i] = v; a += v; b += a; }
            B.pos += len; p += len;
            continue;
        }
        if (type != 2) { status = kInflateBlockType; break; }
        // dynamic block header (RFC 1951 3.2.7)
        if (!ib_need(B, 14)) { status = kInflateTruncated; break; }
        const uint32_t hlit = ib_take(B, 5) + 257u, hdist = ib_take(B, 5) + 1u, hclen = ib_take(B, 4) + 4u;
        if (hlit > 286u || hdist > 30u) { status = kInflateHeader; break; }
        uint8_t cl[19];
        for (uint32_t i = 0; i < 19; i++) cl[i] = 0;
        uint32_t i = 0;
        for (; i < hclen; i++) {
            if (!ib_need(B, 3)) break;
            cl[order[i]] = (uint8_t)ib_take(B, 3);
        }
        if (i < hclen) { status = kInflateTruncated; break; }
        if (inflate_build(cl, 19, S->cl_count, S->cl_sym, nullptr, 0, true)) { status = kInflateCodeLengths; break; }
        const uint32_t total = hlit + hdist;
        for (i = 0; i < total && status == kInflateOk;) {
            const int sym = inflate_decode(B, S->cl_count, S->cl_sym, nullptr, 0);
            if (sym < 0) { status = sym == -1 ? kInflateTruncated : kInflateCodeLengths; break; }
            if (sym < 16) { S->lens[i++] = (uint8_t)sym; continue; }
            uint32_t rep = 0, nrep;
            if (sym == 16) {
                if (i == 0) { status = kInflateRepeat; break; }
                rep = S->lens[i - 1];
                if (!ib_need(B, 2)) { status = kInflateTruncated; break; }
                nrep = 3u + ib_take(B, 2);
            } else if (sym == 17) {
                if (!ib_need(B, 3)) { status = kInflateTruncated; break; }
                nrep = 3u + ib_take(B, 3);
            } else {
                if (!ib_need(B, 7)) { status = kInflateTruncated; break; }
                nrep = 11u + ib_take(B, 7);
            }
            if (nrep > total - i) { status = kInflateRepeat; break; }
            while (nrep--) S->lens[i++] = (uint8_t)rep;
        }
        if (status != kInflateOk) break;
        if (S->lens[256] == 0) { status = kInflateNoEnd; break; }
        if (inflate_build(S->lens, hlit, S->lit_count, S->lit_sym, S->lit_fast, kInflateLitRoot, false)) { status = kInflateLitCode; break; }
        if (inflate_build(S->lens + hlit, hdist, S->dist_count, S->dist_sym, S->dist_fast, kInflateDistRoot, false)) {
            status = kInflateDistCode; break;
        }
        for (;;) {                                                            // the block's symbols
            const int sym = inflate_decode(B, S->lit_count, S->lit_sym, S->lit_fast, kInflateLitRoot);
            if (sym < 0) { status = sym == -1 ? kInflateTruncated : kInflateBadSymbol; break; }
            if (sym < 256) {
                if (p >= kDeflateSeg) { status = kInflateOutputFull; break; }
                out[p++] = (uint8_t)sym; a += (uint32_t)sym; b += a;
                continue;
            }
            if (sym == 256) break;
            if (sym > 285) { status = kInflateBadSymbol; break; }
            const uint32_t li = (uint32_t)sym - 257u, le = deflate_len_extra_bits((uint32_t)sym);
            uint32_t len = sym == 285 ? 258u : li < 8u ? 3u + li : ((4u + (li & 3u)) << le) + 3u;
            if (le) {
                if (!ib_need(B, le)) { status = kInflateTruncated; break; }
                len += ib_take(B, le);
            }
            const int ds = inflate_decode(B, S->dist_count, S->dist_sym, S->dist_fast, kInflateDistRoot);
            if (ds < 0) { status = ds == -1 ? kInflateTruncated : kInflateBadDistance; break; }
            if (ds > 29) { status = kInflateBadDistance; break; }
            const uint32_t de = deflate_dist_extra_bits((uint32_t)ds);
            uint32_t dist = ds < 4 ? (uint32_t)ds + 1u : ((2u + ((uint32_t)ds & 1u)) << de) + 1u;
            if (de) {
                if (!ib_need(B, de)) { status = kInflateTruncated; break; }
                dist += ib_take(B, de);
            }
            if (dist > p) { status = kInflateTooFar; break; }
            if (len > kDeflateSeg - p) { status = kInflateOutputFull; break; }
            for (uint32_t k = 0; k < len; k++) { const uint8_t v = out[p - dist + k]; out[p + k] = v; a += v; b += a; }
            p += len;
        }
        if (status != kInflateOk) break;
    }
    res->status = status;
    res->consumed = status == kInflateOk ? B.pos - (B.cnt >> 3) : 0u;
    res->produced = p;
    res->adler = (uint32_t)(b % 65521ull) << 16 | (a % 65521u);
}

// k_inflate_scan: one CTA per job (a range of positions of one stream).  Position q is a candidate when q == 2 or the four bytes
// before it are 00 00 FF FF; the k-th one found in stream s goes to cand[job.cand0 + k] while k < job.cap, counts[s] counts them
// all.  Candidates of a stream land in any order.
__global__ void __launch_bounds__(256) k_inflate_scan(const InflateScanJob* __restrict__ jobs, const uint8_t* __restrict__ in,
                                                      uint32_t* __restrict__ counts, uint32_t* __restrict__ cand) {
    const InflateScanJob J = jobs[blockIdx.x];
    const uint8_t* s = in + J.base;
    for (uint32_t q = J.begin + threadIdx.x; q < J.end; q += blockDim.x) {
        const bool hit = q == 2u || (q >= 6u && s[q - 4] == 0 && s[q - 3] == 0 && s[q - 2] == 0xff && s[q - 1] == 0xff);
        if (hit) {
            const uint32_t k = atomicAdd(counts + J.stream, 1u);
            if (k < J.cap) cand[J.cand0 + k] = q;
        }
    }
}

// k_inflate_segments: one one-warp CTA per slot; lane 0 inflates candidate slot - slot0 of the slot's stream into the slot
__global__ void __launch_bounds__(32) k_inflate_segments(const uint32_t* __restrict__ slot_stream, const InflateStream* __restrict__ streams,
                                                         const uint8_t* __restrict__ in, const uint32_t* __restrict__ cand,
                                                         uint8_t* __restrict__ slots, InflateSegResult* __restrict__ res,
                                                         uint32_t* __restrict__ start) {
    __shared__ InflateScratch S;
    if (threadIdx.x != 0) return;
    const uint32_t slot = blockIdx.x;
    const InflateStream st = streams[slot_stream[slot]];
    const uint32_t q = cand[st.cand0 + (slot - st.slot0)];
    InflateSegResult r;
    inflate_segment(in + st.base + q, st.len - q, slots + (size_t)slot * kDeflateSeg, &S, &r);
    res[slot] = r;
    start[slot] = q;
}
