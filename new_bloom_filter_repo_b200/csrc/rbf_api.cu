// rbf_api.cu -- the C ABI (include/rbf_b200.h) and the host side of the pipeline.
// Host code mirrors the reference's float expressions exactly (compile with -ffp-contract=off).
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <utility>
#include <vector>

#include "../../include/rbf_b200.h"
#include "rbf_kernels.cuh"

using namespace rbf;

// ------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";

struct rbf_ctx {
    int device = -1;
    cudaStream_t st = nullptr;
    cudaStream_t st_copy = nullptr;   // H2D of frame chunks in rbf_stream_encode_host
    cudaStream_t st_comm = nullptr;   // slot packing + ncclAllGather of rbf_stream_allgather_bitmaps (overlaps the next encode)
    cudaEvent_t ev_enc = nullptr, ev_pack = nullptr, ev_comm = nullptr;
    bool pack_pending = false, comm_pending = false;
    // exchange over NVLink peer memory (rbf_peer_gather_init): receive buffers / flag arrays of all ranks as mapped here
    int peer_nranks = 0, peer_rank = 0;
    uint32_t* peer_recv[16] = {nullptr};
    uint32_t* peer_flags[16] = {nullptr};
    uint32_t peer_seq = 0;
    bool peer_wait_pending = false;
    uint32_t* peer_err = nullptr;     // mapped pinned word, set by k_peer_wait on time-out
    int host_chunk_frames = 32;
    cudaStream_t st_k1 = nullptr;     // pipelined encode: K1 of the later ranges + the witness memset run here, beside K2 on `st`
    cudaStream_t st_d2h = nullptr;    // rbf_stream_encode_host: result copies of chunk i overlap the kernels of chunk i+1
    cudaEvent_t ev_fork = nullptr, ev_wit = nullptr, ev_k1[8] = {nullptr}, ev_d2h = nullptr;
    int encode_ranges = 2;            // rbf_stream_encode: K1/K2 pipelined over this many ranges of pairs (1 = serial; see
                                      // stream_encode_pipelined)
    int pipe_k1_sms = 66;             // the SMs K1 of ranges 1.. runs on; K2 of the range before runs on the others
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    cudaDeviceProp prop;
    LaunchCfg L;            // launcher options and the kernel counter
    int k1_only = 0;        // stop after K1 (mask + counts): VideoFrameCompressor._calculate_frame_diff
    int mask_mode = 0;      // 0: |dY| > thr (ivc:808); 1: additionally any byte of the pixel differs
    int kq_ranges = 1;      // > 1: K2 of range r+1 runs beside K3 of range r (see stream_encode_pipelined)
    char err[512];
    int64_t h2d = 0, d2h = 0, d2d = 0;   // d2d: rbf_stream_copy_frames into caller device memory
    cudaEvent_t ev_wait = nullptr;        // rbf_stream_copy_frames: the caller's stream, recorded before the copy
    std::vector<void*> scratch;
    std::vector<size_t> scratch_sz;
    // NCCL (dlopen'ed)
    void* nccl_lib = nullptr;
    void* nccl_comm = nullptr;
    int nranks = 1, rank = 0;
};

static int set_err(rbf_ctx* c, int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    snprintf(g_err, sizeof g_err, "%s", buf);
    if (c) snprintf(c->err, sizeof c->err, "%s", buf);
    return code;
}
#define CK(ctx, call)                                                                                           \
    do {                                                                                                        \
        cudaError_t e__ = (call);                                                                               \
        if (e__ != cudaSuccess)                                                                                 \
            return set_err(ctx, e__ == cudaErrorMemoryAllocation ? RBF_ERR_OOM : RBF_ERR_CUDA, "%s:%d %s: %s", \
                           __FILE__, __LINE__, #call, cudaGetErrorString(e__));                               \
    } while (0)

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Scratch slots of a context (scratch_get).  Entry points that name the same slot overwrite each other's contents: nothing in a
// slot outlives the call that wrote it.
enum ScratchSlot {
    kScrBytes, kScrResult, kScrOffsets,           // byte per item / bit, check results, string offsets (filters, single-mask coder)
    kScrMask, kScrBits, kScrPass, kScrWit,        // the single-mask coder's FrameJob buffers
    kScrSmall,                                    // its counts, prefix and job; decode_verify's mismatch counts
    kScrValues,                                   // changed values: gather_changed, zlib_changed, apply_diff, apply_chain
    kScrGatherJobs, kScrApplyMask, kScrMedianIn, kScrMedianOut,   // the gather's jobs, apply_diff's mask, median5 planes
    kScrGatherCounts,                             // per-chunk set-bit counts of the gather
    kScrZlibRes, kScrZlibOut, kScrZlibStage, kScrZlibSegs, kScrZlibCopies, kScrZlibSmall, kScrZlibIn,
    kScrDecodeCounts, kScrChainSmall, kScrChainTiles,   // decode_masks' counts; apply_chain's offsets + flags + totals, tile prefix
    kScrInflateIn, kScrInflateSmall, kScrInflateSlots, kScrInflateRes, kScrInflateOut,   // inflate_streams / inflate_place
};

static int scratch_get(rbf_ctx* c, int slot, size_t bytes, void** out) {
    if ((int)c->scratch.size() <= slot) { c->scratch.resize(slot + 1, nullptr); c->scratch_sz.resize(slot + 1, 0); }
    if (c->scratch_sz[slot] < bytes) {
        if (c->scratch[slot]) CK(c, cudaFree(c->scratch[slot]));
        c->scratch[slot] = nullptr; c->scratch_sz[slot] = 0;
        size_t nb = align_up(bytes + (bytes >> 2), 256);
        CK(c, cudaMalloc(&c->scratch[slot], nb));
        c->scratch_sz[slot] = nb;
    }
    *out = c->scratch[slot];
    return RBF_OK;
}
// ------------------------------------------------------------------------------------------
// exact host-side scalars
// ------------------------------------------------------------------------------------------
// correctly rounded double of h / (2^64 - 1): Python int/int true division (ivc:95).  The exact
// quotient is h*2^-64*(1 + 2^-64 + ...), a hair above h*2^-64, so round h to 53 bits, ties up.
static double unit_div(uint64_t h) {
    if (h == 0) return 0.0;
    const int bl = 64 - __builtin_clzll(h);
    if (bl <= 53) return ldexp((double)h, -64);
    const int sh = bl - 53;
    uint64_t top = h >> sh;
    const uint64_t rem = h & ((1ULL << sh) - 1), half = 1ULL << (sh - 1);
    if (rem >= half) top += 1;
    return ldexp((double)top, sh - 64);
}

extern "C" uint64_t rbf_activation_threshold(double p_act) {
    if (!(p_act > 0.0)) return 0;                       // also NaN
    if (unit_div(UINT64_MAX) < p_act) return UINT64_MAX;
    uint64_t lo = 0, hi = UINT64_MAX;                   // smallest h with unit_div(h) >= p_act
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo) / 2;
        if (unit_div(mid) < p_act) lo = mid + 1; else hi = mid;
    }
    return lo;
}

static const double kPStar = 0.32453;                  // ivc:150

// _calculate_optimal_params (ivc:161-196); returns l (0 => the (0, 0) result)
static uint64_t optimal_kl(uint64_t n, double p, double* k_out) {
    *k_out = 0.0;
    if (p <= 0.0001) return 0;
    if (p >= kPStar) return 0;
    const double q = 1 - p;
    const double L = log(2.0);
    const double k = log2(q * pow(L, 2.0) / p);         // ivc:185
    if (isnan(k) || k <= 0) return 0;
    const double gamma = 1 / L;
    const double lf = p * (double)n * k * gamma;        // ivc:193, evaluated left to right
    const uint64_t l = (uint64_t)lf;
    *k_out = k > 0.1 ? k : 0.1;
    return l > 1 ? l : 1;
}

extern "C" int rbf_optimal_params(uint64_t n, uint64_t ones, double* p_out, double* k_out, uint64_t* l_out) {
    const double p = (double)ones / (double)n;          // ivc:212
    double k = 0.0;
    uint64_t l = 0;
    int coded = 0;
    if (!(p >= kPStar)) {                               // ivc:215
        l = optimal_kl(n, p, &k);
        if (!(l == 0 || l >= n)) coded = 1;             // ivc:223
    }
    if (!coded) { k = 0.0; l = 0; }
    if (p_out) *p_out = p;
    if (k_out) *k_out = k;
    if (l_out) *l_out = l;
    return coded;
}

extern "C" uint64_t rbf_xxh64(const void* data, uint64_t len, uint64_t seed) {
    return xxh64_bytes((const uint8_t*)data, (uint32_t)len, seed);
}
extern "C" uint64_t rbf_hash_decimal(uint32_t item, uint64_t seed) { return xxh64_decimal(item, seed); }
extern "C" uint64_t rbf_hash_decimal_century(uint32_t item, uint64_t seed) {
    const Century c = make_century(item / 100u);
    return finish(c.kind, decade_state(c, century_state(c, seed), seed, (item / 10u) % 10u), seed, item % 10u);
}
extern "C" uint32_t rbf_probe_index(uint64_t h1, uint64_t h2, uint32_t i, uint32_t size) {
    if (size == 0) return 0;
    return probe_index(h1, h2, i, make_fastmod(size));
}
extern "C" int rbf_abi_version(void) { return RBF_ABI_VERSION; }
extern "C" const char* rbf_last_global_error(void) { return g_err; }

// fill the filter part of a job from (size, k*)  (ivc:47-63)
static void job_set_filter(FrameJob& J, uint64_t size, double k_star, const rbf_seeds& sd) {
    J.l = (uint32_t)size;
    const double fl = floor(k_star);
    J.floor_k = (uint32_t)(fl < 0 ? 0 : fl);
    const double p_act = k_star - fl;                   // ivc:58
    J.has_act = p_act > 0.0 ? 1u : 0u;
    J.act_T = rbf_activation_threshold(p_act);
    J.seed1 = sd.h1; J.seed2 = sd.h2; J.seedA = sd.act;
    J.fm = make_fastmod((uint32_t)size);
    J.neg_m = 0u - (uint32_t)size;
}

// ------------------------------------------------------------------------------------------
// context
// ------------------------------------------------------------------------------------------
extern "C" int rbf_ctx_create(int device, rbf_ctx** out) {
    if (!out) return set_err(nullptr, RBF_ERR_INVALID, "rbf_ctx_create: out is NULL");
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return set_err(nullptr, RBF_ERR_NO_DEVICE, "no CUDA device available (%s); this library has no CPU fallback",
                       e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    if (device < 0 || device >= ndev) return set_err(nullptr, RBF_ERR_INVALID, "device %d out of range [0,%d)", device, ndev);
    rbf_ctx* c = new rbf_ctx();
    c->err[0] = 0;
    c->device = device;
    if ((e = cudaSetDevice(device)) != cudaSuccess || (e = cudaGetDeviceProperties(&c->prop, device)) != cudaSuccess) {
        delete c;
        return set_err(nullptr, RBF_ERR_CUDA, "cudaSetDevice/GetDeviceProperties: %s", cudaGetErrorString(e));
    }
    if (c->prop.major != 9 || c->prop.minor != 0) {      // sm_90a code loads on compute capability 9.0 only
        int maj = c->prop.major, mn = c->prop.minor;
        delete c;
        return set_err(nullptr, RBF_ERR_NO_DEVICE, "device is sm_%d%d; this library is built for sm_90a only", maj, mn);
    }
    c->L.sm_count = c->prop.multiProcessorCount;
    c->L.query_smem_cap = query_max_smem_bytes();
    if ((e = cudaStreamCreateWithFlags(&c->st, cudaStreamNonBlocking)) != cudaSuccess ||
        (e = cudaEventCreate(&c->ev0)) != cudaSuccess || (e = cudaEventCreate(&c->ev1)) != cudaSuccess) {
        delete c;
        return set_err(nullptr, RBF_ERR_CUDA, "stream/event create: %s", cudaGetErrorString(e));
    }
    *out = c;
    return RBF_OK;
}

extern "C" void rbf_ctx_destroy(rbf_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    rbf_nccl_destroy(c);
    for (void* p : c->scratch) if (p) cudaFree(p);
    if (c->ev0) cudaEventDestroy(c->ev0);
    if (c->ev1) cudaEventDestroy(c->ev1);
    if (c->ev_wait) cudaEventDestroy(c->ev_wait);
    if (c->st) cudaStreamDestroy(c->st);
    if (c->st_k1) cudaStreamDestroy(c->st_k1);
    if (c->st_d2h) cudaStreamDestroy(c->st_d2h);
    if (c->ev_fork) cudaEventDestroy(c->ev_fork);
    if (c->ev_wit) cudaEventDestroy(c->ev_wit);
    if (c->ev_d2h) cudaEventDestroy(c->ev_d2h);
    for (auto& e : c->ev_k1) if (e) cudaEventDestroy(e);
    if (c->st_copy) cudaStreamDestroy(c->st_copy);
    if (c->st_comm) { cudaStreamSynchronize(c->st_comm); cudaStreamDestroy(c->st_comm); }
    if (c->ev_enc) cudaEventDestroy(c->ev_enc);
    if (c->ev_pack) cudaEventDestroy(c->ev_pack);
    if (c->ev_comm) cudaEventDestroy(c->ev_comm);
    if (c->peer_err) cudaFreeHost(c->peer_err);
    delete c;
}
extern "C" const char* rbf_last_error(const rbf_ctx* c) { return c ? c->err : g_err; }

extern "C" int rbf_device_info(rbf_ctx* c, char* name, int name_len, int* sm_count, int* cc_major, int* cc_minor,
                               uint64_t* total_mem) {
    if (!c) return set_err(nullptr, RBF_ERR_INVALID, "ctx is NULL");
    if (name && name_len > 0) snprintf(name, name_len, "%s", c->prop.name);
    if (sm_count) *sm_count = c->L.sm_count;
    if (cc_major) *cc_major = c->prop.major;
    if (cc_minor) *cc_minor = c->prop.minor;
    if (total_mem) *total_mem = c->prop.totalGlobalMem;
    return RBF_OK;
}
extern "C" int rbf_set_option(rbf_ctx* c, const char* key, int64_t v) {
    if (!c || !key) return set_err(c, RBF_ERR_INVALID, "rbf_set_option: NULL");
    if (!strcmp(key, "k1_variant")) { c->L.k1_variant = (int)v; return RBF_OK; }
    if (!strcmp(key, "query_variant")) { c->L.query_variant = (int)(v < 0 ? 0 : (v > 6 ? 6 : v)); return RBF_OK; }
    if (!strcmp(key, "insert_variant")) { c->L.insert_variant = v ? 1 : 0; return RBF_OK; }
    if (!strcmp(key, "host_chunk_frames")) { c->host_chunk_frames = (int)v; return RBF_OK; }
    if (!strcmp(key, "k1_only")) { c->k1_only = v ? 1 : 0; return RBF_OK; }        // default of streams created afterwards
    if (!strcmp(key, "mask_mode")) { c->mask_mode = v ? 1 : 0; return RBF_OK; }    // (per-stream: rbf_stream_set_option)
    if (!strcmp(key, "query_warps")) { c->L.query_warps = (int)v; return RBF_OK; }
    if (!strcmp(key, "kq_ranges")) { c->kq_ranges = (int)(v < 1 ? 1 : (v > 8 ? 8 : v)); return RBF_OK; }
    if (!strcmp(key, "encode_ranges")) { c->encode_ranges = (int)(v < 1 ? 1 : (v > 8 ? 8 : v)); return RBF_OK; }
    if (!strcmp(key, "k1_ctas_per_sm")) { c->L.k1_ctas_per_sm = (int)(v < 1 ? 1 : (v > 64 ? 64 : v)); return RBF_OK; }
    if (!strcmp(key, "pipe_k1_sms")) { c->pipe_k1_sms = (int)(v < 1 ? 1 : (v > 1024 ? 1024 : v)); return RBF_OK; }
    if (!strcmp(key, "query_smem_bytes")) {
        c->L.query_smem_cap = (int)((v <= 0 || v > query_max_smem_bytes()) ? query_max_smem_bytes() : v);
        return RBF_OK;
    }
    return set_err(c, RBF_ERR_INVALID, "unknown option %s", key);
}
extern "C" int64_t rbf_get_counter(rbf_ctx* c, const char* key) {
    if (!c || !key) return -1;
    if (!strcmp(key, "kernel_launches")) return c->L.launches;
    if (!strcmp(key, "h2d_bytes")) return c->h2d;
    if (!strcmp(key, "d2h_bytes")) return c->d2h;
    if (!strcmp(key, "d2d_bytes")) return c->d2d;
    return -1;
}
extern "C" int rbf_reset_counters(rbf_ctx* c) { if (!c) return RBF_ERR_INVALID; c->L.launches = c->h2d = c->d2h = c->d2d = 0; return RBF_OK; }
// before the bit arrays are overwritten: the slot packing of a pending all-gather must have read them
static int wait_pack(rbf_ctx* c) {
    if (c->pack_pending) { CK(c, cudaStreamWaitEvent(c->st, c->ev_pack, 0)); c->pack_pending = false; }
    return RBF_OK;
}
// make the context's stream wait for an all-gather still running on the communication stream
static const long long kPeerTimeoutCycles = 6000000000LL;    // ~3 s of SM clocks: a lost peer must not hang the GPU
static int join_comm(rbf_ctx* c) {
    if (c->comm_pending) { CK(c, cudaStreamWaitEvent(c->st, c->ev_comm, 0)); c->comm_pending = false; c->pack_pending = false; }
    if (c->peer_wait_pending) {                                // the other ranks' slots of the last exchange
        CK(c, launch_peer_wait(c->L, c->peer_flags[c->peer_rank], c->peer_nranks, c->peer_seq, kPeerTimeoutCycles, c->peer_err, c->st));
        c->peer_wait_pending = false;
    }
    return RBF_OK;
}
static int check_peer_err(rbf_ctx* c) {                        // call after the stream has been synchronised
    if (c->peer_err && *(volatile uint32_t*)c->peer_err) {
        *(volatile uint32_t*)c->peer_err = 0;
        return set_err(c, RBF_ERR_NCCL, "peer exchange timed out: a rank did not deliver its slots");
    }
    return RBF_OK;
}
extern "C" int rbf_sync(rbf_ctx* c) {
    if (!c) return RBF_ERR_INVALID;
    if (int r = join_comm(c)) return r;
    CK(c, cudaStreamSynchronize(c->st));
    return check_peer_err(c);
}
extern "C" int rbf_timer_start(rbf_ctx* c) { if (!c) return RBF_ERR_INVALID; CK(c, cudaEventRecord(c->ev0, c->st)); return RBF_OK; }
extern "C" int rbf_timer_stop_ms(rbf_ctx* c, double* ms) {
    if (!c || !ms) return RBF_ERR_INVALID;
    if (int r = join_comm(c)) return r;
    CK(c, cudaEventRecord(c->ev1, c->st));
    CK(c, cudaEventSynchronize(c->ev1));
    float f = 0;
    CK(c, cudaEventElapsedTime(&f, c->ev0, c->ev1));
    *ms = f;
    return check_peer_err(c);
}

// memory
extern "C" int rbf_malloc(rbf_ctx* c, size_t bytes, void** d) { if (!c || !d) return RBF_ERR_INVALID; CK(c, cudaSetDevice(c->device)); CK(c, cudaMalloc(d, bytes ? bytes : 1)); return RBF_OK; }
extern "C" int rbf_free(rbf_ctx* c, void* d) { if (!c) return RBF_ERR_INVALID; if (d) CK(c, cudaFree(d)); return RBF_OK; }
extern "C" int rbf_malloc_host(rbf_ctx* c, size_t bytes, void** h) { if (!c || !h) return RBF_ERR_INVALID; CK(c, cudaMallocHost(h, bytes ? bytes : 1)); return RBF_OK; }
extern "C" int rbf_free_host(rbf_ctx* c, void* h) { if (!c) return RBF_ERR_INVALID; if (h) CK(c, cudaFreeHost(h)); return RBF_OK; }
extern "C" int rbf_memcpy_d2h(rbf_ctx* c, void* h, const void* d, size_t n) {
    if (!c) return RBF_ERR_INVALID;
    if (int r = join_comm(c)) return r;
    CK(c, cudaMemcpyAsync(h, d, n, cudaMemcpyDeviceToHost, c->st)); CK(c, cudaStreamSynchronize(c->st)); c->d2h += n;
    return check_peer_err(c);
}
extern "C" int rbf_memset(rbf_ctx* c, void* d, int v, size_t n) { if (!c) return RBF_ERR_INVALID; CK(c, cudaMemsetAsync(d, v, n, c->st)); return RBF_OK; }

// ------------------------------------------------------------------------------------------
// one filter
// ------------------------------------------------------------------------------------------
struct rbf_filter {
    rbf_ctx* c;
    uint64_t size;
    FrameJob job;          // host copy
    FrameJob* d_job;
    uint32_t* d_bits;      // LSB-first
    size_t words;
};

extern "C" int rbf_filter_create(rbf_ctx* c, uint64_t size, double k_star, const rbf_seeds* sd, rbf_filter** out) {
    if (!c || !sd || !out) return set_err(c, RBF_ERR_INVALID, "rbf_filter_create: NULL argument");
    if (size == 0 || size > 0xffffffffULL) return set_err(c, RBF_ERR_INVALID, "filter size %llu outside [1, 2^32)", (unsigned long long)size);
    if (!(k_star >= 0.0) || k_star > 1e6) return set_err(c, RBF_ERR_INVALID, "k_star %g not supported", k_star);
    CK(c, cudaSetDevice(c->device));
    rbf_filter* f = new rbf_filter();
    f->c = c; f->size = size; f->words = align_up((size + 31) / 32 + 8, 32);
    memset(&f->job, 0, sizeof f->job);
    job_set_filter(f->job, size, k_star, *sd);
    f->job.n = 0;
    cudaError_t e = cudaMalloc(&f->d_bits, f->words * 4);
    if (e == cudaSuccess) e = cudaMalloc(&f->d_job, sizeof(FrameJob));
    if (e != cudaSuccess) { delete f; return set_err(c, RBF_ERR_OOM, "rbf_filter_create: %s", cudaGetErrorString(e)); }
    f->job.bits = f->d_bits;
    CK(c, cudaMemsetAsync(f->d_bits, 0, f->words * 4, c->st));
    CK(c, cudaMemcpyAsync(f->d_job, &f->job, sizeof(FrameJob), cudaMemcpyHostToDevice, c->st));
    CK(c, cudaStreamSynchronize(c->st));
    *out = f;
    return RBF_OK;
}
extern "C" void rbf_filter_destroy(rbf_filter* f) {
    if (!f) return;
    cudaFree(f->d_bits); cudaFree(f->d_job);
    delete f;
}
static int filter_items_u32(rbf_filter* f, const uint32_t* items, uint32_t count, uint8_t* out, int insert) {
    rbf_ctx* c = f->c;
    if (count == 0) return RBF_OK;
    void *d_items, *d_res;
    int rc;
    if ((rc = scratch_get(c, kScrBytes, (size_t)count * 4, &d_items))) return rc;
    if ((rc = scratch_get(c, kScrResult, (size_t)count, &d_res))) return rc;
    CK(c, cudaMemcpyAsync(d_items, items, (size_t)count * 4, cudaMemcpyHostToDevice, c->st)); c->h2d += (size_t)count * 4;
    CK(c, launch_items_u32(c->L, f->d_job, (const uint32_t*)d_items, count, (uint8_t*)d_res, insert, c->st));
    if (!insert) { CK(c, cudaMemcpyAsync(out, d_res, count, cudaMemcpyDeviceToHost, c->st)); c->d2h += count; }
    CK(c, cudaStreamSynchronize(c->st));
    return RBF_OK;
}
extern "C" int rbf_filter_add_indices(rbf_filter* f, const uint32_t* items, uint32_t count) {
    if (!f || (!items && count)) return set_err(f ? f->c : nullptr, RBF_ERR_INVALID, "rbf_filter_add_indices: NULL");
    return filter_items_u32(f, items, count, nullptr, 1);
}
extern "C" int rbf_filter_check_indices(rbf_filter* f, const uint32_t* items, uint32_t count, uint8_t* out) {
    if (!f || ((!items || !out) && count)) return set_err(f ? f->c : nullptr, RBF_ERR_INVALID, "rbf_filter_check_indices: NULL");
    return filter_items_u32(f, items, count, out, 0);
}
static int filter_items_str(rbf_filter* f, const uint8_t* blob, const uint64_t* offs, uint32_t count, int standard_k,
                            uint8_t* out, int insert) {
    rbf_ctx* c = f->c;
    if (count == 0) return RBF_OK;
    const size_t blob_bytes = (size_t)offs[count];
    void *d_blob, *d_offs, *d_res;
    int rc;
    if ((rc = scratch_get(c, kScrBytes, blob_bytes + 16, &d_blob))) return rc;
    if ((rc = scratch_get(c, kScrResult, (size_t)count, &d_res))) return rc;
    if ((rc = scratch_get(c, kScrOffsets, ((size_t)count + 1) * 8, &d_offs))) return rc;
    if (blob_bytes) { CK(c, cudaMemcpyAsync(d_blob, blob, blob_bytes, cudaMemcpyHostToDevice, c->st)); }
    CK(c, cudaMemcpyAsync(d_offs, offs, ((size_t)count + 1) * 8, cudaMemcpyHostToDevice, c->st));
    c->h2d += blob_bytes + ((size_t)count + 1) * 8;
    CK(c, launch_items_str(c->L, f->d_job, (const uint8_t*)d_blob, (const uint64_t*)d_offs, count, (uint8_t*)d_res, insert,
                               standard_k, c->st));
    if (!insert) { CK(c, cudaMemcpyAsync(out, d_res, count, cudaMemcpyDeviceToHost, c->st)); c->d2h += count; }
    CK(c, cudaStreamSynchronize(c->st));
    return RBF_OK;
}
extern "C" int rbf_filter_add_strings(rbf_filter* f, const uint8_t* blob, const uint64_t* offs, uint32_t count, int standard_k) {
    if (!f || (!offs && count)) return set_err(f ? f->c : nullptr, RBF_ERR_INVALID, "rbf_filter_add_strings: NULL");
    return filter_items_str(f, blob, offs, count, standard_k, nullptr, 1);
}
extern "C" int rbf_filter_check_strings(rbf_filter* f, const uint8_t* blob, const uint64_t* offs, uint32_t count,
                                        int standard_k, uint8_t* out) {
    if (!f || ((!offs || !out) && count)) return set_err(f ? f->c : nullptr, RBF_ERR_INVALID, "rbf_filter_check_strings: NULL");
    return filter_items_str(f, blob, offs, count, standard_k, out, 0);
}
extern "C" int rbf_filter_get_bits(rbf_filter* f, uint8_t* out) {
    if (!f || !out) return set_err(f ? f->c : nullptr, RBF_ERR_INVALID, "rbf_filter_get_bits: NULL");
    rbf_ctx* c = f->c;
    void* d_bytes; int rc;
    if ((rc = scratch_get(c, kScrBytes, f->size, &d_bytes))) return rc;
    CK(c, launch_unpack_bits(c->L, f->d_bits, (uint8_t*)d_bytes, f->size, c->st));
    CK(c, cudaMemcpyAsync(out, d_bytes, f->size, cudaMemcpyDeviceToHost, c->st)); c->d2h += f->size;
    CK(c, cudaStreamSynchronize(c->st));
    return RBF_OK;
}
extern "C" int rbf_filter_set_bits(rbf_filter* f, const uint8_t* in) {
    if (!f || !in) return set_err(f ? f->c : nullptr, RBF_ERR_INVALID, "rbf_filter_set_bits: NULL");
    rbf_ctx* c = f->c;
    void* d_bytes; int rc;
    if ((rc = scratch_get(c, kScrBytes, f->size, &d_bytes))) return rc;
    CK(c, cudaMemcpyAsync(d_bytes, in, f->size, cudaMemcpyHostToDevice, c->st)); c->h2d += f->size;
    CK(c, cudaMemsetAsync(f->d_bits, 0, f->words * 4, c->st));
    CK(c, launch_pack_bytes(c->L, (const uint8_t*)d_bytes, f->d_bits, f->size, 1, c->st));     // any non-zero byte is set (ivc:129,135)
    CK(c, cudaStreamSynchronize(c->st));
    return RBF_OK;
}

// ------------------------------------------------------------------------------------------
// mask coder (host buffers)
// ------------------------------------------------------------------------------------------

static size_t bit_words_padded(uint64_t nbits) { return align_up((nbits + 31) / 32 + 8, 32); }   // >= 32 B of padding, 128 B multiple
static size_t pass_words(uint64_t n) { return align_up(((n + 99) / 100) * 4, 32); }

// A FrameJob of n positions over the given bit array, witness and pass mask, with the filter of (l, k*) when l > 0 (l == 0: raw
// passthrough).  The caller adds the mask it encodes (mask) or decodes into (out_mask, wlen_in).
static FrameJob frame_job(uint64_t n, uint64_t l, double k_star, const rbf_seeds& sd, uint32_t* bits, uint32_t* witness, uint32_t* pass) {
    FrameJob J;
    memset(&J, 0, sizeof J);
    J.n = (uint32_t)n;
    if (l) job_set_filter(J, l, k_star, sd);
    J.bits = bits; J.witness = witness; J.pass = pass;
    return J;
}

// Decode (K3 + K4b) of F jobs on the context's stream: the jobs and their century prefix (F + 1 entries) go to the device, every
// coded job's mask lands in its out_mask and its consumed witness bits in d_consumed.  d_scratch: F * 32 words.
static int decode_enqueue(rbf_ctx* c, const FrameJob* h_jobs, FrameJob* d_jobs, const uint32_t* h_prefix, uint32_t* d_prefix, int F,
                          uint32_t max_l, uint32_t ncent, uint32_t* d_scratch, uint32_t* d_consumed) {
    CK(c, cudaMemcpyAsync(d_jobs, h_jobs, sizeof(FrameJob) * F, cudaMemcpyHostToDevice, c->st));
    CK(c, cudaMemcpyAsync(d_prefix, h_prefix, 4 * ((size_t)F + 1), cudaMemcpyHostToDevice, c->st));
    CK(c, launch_query(c->L, d_jobs, d_prefix, F, h_prefix[F], max_l, c->st));
    CK(c, launch_expand(c->L, d_jobs, F, ncent, d_scratch, d_consumed, c->st));
    return RBF_OK;
}

extern "C" int rbf_compress_mask(rbf_ctx* c, const uint8_t* mask, uint64_t n, const rbf_seeds* sd, double k_override,
                                 uint64_t l_override, rbf_mask_info* info, uint8_t* bitmap_out, uint8_t* witness_out) {
    if (!c || !mask || !sd || !info) return set_err(c, RBF_ERR_INVALID, "rbf_compress_mask: NULL argument");
    if (n == 0 || n > 0xffffff00ULL) return set_err(c, RBF_ERR_INVALID, "n = %llu outside [1, 2^32-256]", (unsigned long long)n);
    CK(c, cudaSetDevice(c->device));
    memset(info, 0, sizeof *info);
    info->n = n;
    const size_t mw = bit_words_padded(n), pw = pass_words(n);
    void *d_bytes, *d_mask, *d_bits, *d_pass, *d_wit, *d_small;
    int rc;
    if ((rc = scratch_get(c, kScrBytes, n, &d_bytes)) || (rc = scratch_get(c, kScrMask, mw * 4, &d_mask)) ||
        (rc = scratch_get(c, kScrBits, mw * 4, &d_bits)) || (rc = scratch_get(c, kScrPass, pw * 4, &d_pass)) ||
        (rc = scratch_get(c, kScrWit, mw * 4, &d_wit)) || (rc = scratch_get(c, kScrSmall, 4096, &d_small)))
        return rc;
    uint32_t* d_cnt = (uint32_t*)d_small;                         // [0] ones, [1] wlen
    uint32_t* d_prefix = d_cnt + 4;                               // [2] cent_prefix
    FrameJob* d_job = (FrameJob*)((uint8_t*)d_small + 256);
    CK(c, cudaMemcpyAsync(d_bytes, mask, n, cudaMemcpyHostToDevice, c->st)); c->h2d += n;
    CK(c, cudaMemsetAsync(d_mask, 0, mw * 4, c->st));
    CK(c, cudaMemsetAsync(d_cnt, 0, 16, c->st));
    CK(c, launch_pack_bytes(c->L, (const uint8_t*)d_bytes, (uint32_t*)d_mask, n, 0, c->st));    // `binary_input[i] == 1`, ivc:236
    CK(c, launch_popcount(c->L, (const uint32_t*)d_mask, (n + 31) / 32, d_cnt, c->st));
    uint32_t h_cnt[4] = {0, 0, 0, 0};
    CK(c, cudaMemcpyAsync(h_cnt, d_cnt, 16, cudaMemcpyDeviceToHost, c->st)); c->d2h += 16;
    CK(c, cudaStreamSynchronize(c->st));
    info->ones = h_cnt[0];
    double p, k; uint64_t l;
    int coded = rbf_optimal_params(n, info->ones, &p, &k, &l);
    info->p = p;
    if (k_override > 0.0 && !(p >= kPStar)) { k = k_override; l = l_override; coded = !(l == 0 || l >= n); }
    if (!coded) { info->raw = 1; return RBF_OK; }
    info->k = k; info->l = l;
    FrameJob J = frame_job(n, l, k, *sd, (uint32_t*)d_bits, (uint32_t*)d_wit, (uint32_t*)d_pass);
    J.mask = (const uint32_t*)d_mask;
    info->floor_k = J.floor_k; info->act_T = J.act_T;
    const uint32_t ncent = (uint32_t)((n + 99) / 100);
    uint32_t h_prefix[2] = {0, ncent};
    CK(c, cudaMemcpyAsync(d_job, &J, sizeof J, cudaMemcpyHostToDevice, c->st));
    CK(c, cudaMemcpyAsync(d_prefix, h_prefix, 8, cudaMemcpyHostToDevice, c->st));
    CK(c, cudaMemsetAsync(d_bits, 0, bit_words_padded(l) * 4, c->st));
    CK(c, cudaMemsetAsync(d_wit, 0, mw * 4, c->st));
    CK(c, launch_insert(c->L, d_job, 1, ncent, (uint32_t)l, c->L.sm_count, c->st));
    CK(c, launch_query(c->L, d_job, d_prefix, 1, ncent, (uint32_t)l, c->st));
    CK(c, launch_witness(c->L, d_job, 1, ncent, (uint32_t*)((uint8_t*)d_small + 1024), d_cnt + 1, c->st));
    CK(c, cudaMemcpyAsync(h_cnt, d_cnt, 16, cudaMemcpyDeviceToHost, c->st)); c->d2h += 16;
    CK(c, cudaStreamSynchronize(c->st));
    info->wlen = h_cnt[1];
    // after K3b both streams are in packbits order; hand them back unpacked (ivc:266 returns bit_array, witness)
    if (bitmap_out) {
        CK(c, launch_unpack_bits_msb(c->L, (const uint32_t*)d_bits, (uint8_t*)d_bytes, l, c->st));
        CK(c, cudaMemcpyAsync(bitmap_out, d_bytes, l, cudaMemcpyDeviceToHost, c->st)); c->d2h += l;
        CK(c, cudaStreamSynchronize(c->st));
    }
    if (witness_out && info->wlen) {
        CK(c, launch_unpack_bits_msb(c->L, (const uint32_t*)d_wit, (uint8_t*)d_bytes, info->wlen, c->st));
        CK(c, cudaMemcpyAsync(witness_out, d_bytes, info->wlen, cudaMemcpyDeviceToHost, c->st)); c->d2h += info->wlen;
        CK(c, cudaStreamSynchronize(c->st));
    }
    return RBF_OK;
}

extern "C" int rbf_decompress_mask(rbf_ctx* c, const uint8_t* bitmap, uint64_t l, const uint8_t* witness, uint64_t wlen,
                                   uint64_t n, double k, const rbf_seeds* sd, uint8_t* out, uint64_t* consumed) {
    if (!c || !bitmap || !sd || !out || (!witness && wlen)) return set_err(c, RBF_ERR_INVALID, "rbf_decompress_mask: NULL argument");
    if (n == 0 || n > 0xffffff00ULL || l == 0 || l > 0xffffffffULL) return set_err(c, RBF_ERR_INVALID, "bad n/l");
    if (!(k >= 0.0)) return set_err(c, RBF_ERR_INVALID, "bad k");
    CK(c, cudaSetDevice(c->device));
    const size_t mw = bit_words_padded(n), lw = bit_words_padded(l), ww = bit_words_padded(wlen), pw = pass_words(n);
    const size_t big = n > l ? (n > wlen ? n : wlen) : (l > wlen ? l : wlen);
    void *d_bytes, *d_out, *d_bits, *d_pass, *d_wit, *d_small;
    int rc;
    if ((rc = scratch_get(c, kScrBytes, big, &d_bytes)) || (rc = scratch_get(c, kScrMask, mw * 4, &d_out)) ||
        (rc = scratch_get(c, kScrBits, lw * 4, &d_bits)) || (rc = scratch_get(c, kScrPass, pw * 4, &d_pass)) ||
        (rc = scratch_get(c, kScrWit, ww * 4, &d_wit)) || (rc = scratch_get(c, kScrSmall, 4096, &d_small)))
        return rc;
    uint32_t* d_cnt = (uint32_t*)d_small;
    uint32_t* d_prefix = d_cnt + 4;
    FrameJob* d_job = (FrameJob*)((uint8_t*)d_small + 256);
    CK(c, cudaMemsetAsync(d_bits, 0, lw * 4, c->st));
    CK(c, cudaMemsetAsync(d_wit, 0, ww * 4, c->st));
    CK(c, cudaMemsetAsync(d_out, 0, mw * 4, c->st));
    CK(c, cudaMemcpyAsync(d_bytes, bitmap, l, cudaMemcpyHostToDevice, c->st)); c->h2d += l;
    CK(c, launch_pack_bytes(c->L, (const uint8_t*)d_bytes, (uint32_t*)d_bits, l, 1, c->st));     // the filter's bit array: non-zero is set
    if (wlen) {
        CK(c, cudaMemcpyAsync(d_bytes, witness, wlen, cudaMemcpyHostToDevice, c->st)); c->h2d += wlen;
        // witness values are used as bits: any non-zero byte other than 1 is not representable; the reference
        // stores whatever the list holds (ivc:303); np.unpackbits output is 0/1 (ivc:1001-1002)
        CK(c, launch_pack_bytes(c->L, (const uint8_t*)d_bytes, (uint32_t*)d_wit, wlen, 0, c->st));
    }
    FrameJob J = frame_job(n, l, k, *sd, (uint32_t*)d_bits, (uint32_t*)d_wit, (uint32_t*)d_pass);
    J.out_mask = (uint32_t*)d_out;
    J.wlen_in = (uint32_t)wlen;
    const uint32_t ncent = (uint32_t)((n + 99) / 100);
    const uint32_t h_prefix[2] = {0, ncent};
    if (int r = decode_enqueue(c, &J, d_job, h_prefix, d_prefix, 1, (uint32_t)l, ncent, (uint32_t*)((uint8_t*)d_small + 1024), d_cnt)) return r;
    CK(c, launch_unpack_bits(c->L, (const uint32_t*)d_out, (uint8_t*)d_bytes, n, c->st));
    uint32_t h_cnt = 0;
    CK(c, cudaMemcpyAsync(out, d_bytes, n, cudaMemcpyDeviceToHost, c->st)); c->d2h += n;
    CK(c, cudaMemcpyAsync(&h_cnt, d_cnt, 4, cudaMemcpyDeviceToHost, c->st));
    CK(c, cudaStreamSynchronize(c->st));
    if (consumed) *consumed = h_cnt;
    return RBF_OK;
}

// ------------------------------------------------------------------------------------------
// frame stream
// ------------------------------------------------------------------------------------------
struct rbf_stream {
    rbf_ctx* c;
    uint32_t H, W, C, S, max_frames, max_pairs;
    uint64_t npix, frame_bytes, frame_stride;
    uint8_t* d_frames = nullptr;
    size_t mask_stride_w = 0, pass_stride_w = 0;     // words per pair
    uint32_t *d_mask = nullptr, *d_bits = nullptr, *d_wit = nullptr, *d_pass = nullptr, *d_dec = nullptr;
    FrameJob* d_jobs = nullptr;
    PairJob* d_pairs = nullptr;
    uint32_t *d_prefix = nullptr, *d_ones = nullptr, *d_resid = nullptr, *d_wlen = nullptr, *d_chunkcnt = nullptr;
    // pinned host mirrors
    FrameJob* h_jobs = nullptr;
    PairJob* h_pairs = nullptr;
    uint32_t *h_prefix = nullptr, *h_ones = nullptr, *h_resid = nullptr, *h_wlen = nullptr;
    uint32_t last_pairs = 0, last_max_l = 0;
    cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    bool staged = false;
    // per-stream options (rbf_stream_set_option); defaults come from the context at creation
    int k1_only = 0;        // stop after K1 (mask + counts): VideoFrameCompressor._calculate_frame_diff
    int mask_mode = 0;      // 0: |dY| > thr (ivc:808); 1: additionally any byte of the pixel differs
    int gray_mode = 0;      // 1: the mask is taken on cv2.COLOR_BGR2GRAY of the pixel (ivc:792-795) instead of on sample 0
    int value_mode = 0;     // changed-value gathers: 0 the current samples; 1 residuals (curr - prev) mod 2^(8 S) per sample
    int motion_values = 0;  // 1: the gathers return residuals against the motion-compensated previous frame of the last search
    int8_t* d_fields = nullptr;             // [max_pairs][mv_blocks(H, W)][2] block vectors of rbf_stream_motion_search
    uint32_t motion_pairs = 0;              // pairs searched since the last encode (0: none, or a decode_masks overwrote the slots)
    uint8_t* d_inflated = nullptr;          // rbf_stream_inflate_values: the group's values back to back, read by apply_chain (values NULL)
    size_t inflated_cap = 0;
    uint64_t inflated_bytes = 0;            // bytes the last rbf_stream_inflate_values placed (cleared by apply_chain with values NULL)
    bool last_k1_only = false;
    rbf_seeds last_sd = {};                 // seeds of the last encode (decode_verify rebuilds its jobs from them and last_infos)
    size_t bits_hwm = 0, wit_hwm = 0;   // bytes per slot that may hold set bits (see enc_stage_jobs)
    bool wit_dirty_full = false;
    std::vector<cudaEvent_t> ev_copy;
    std::vector<rbf_mask_info> last_infos;
};

extern "C" void rbf_stream_destroy(rbf_stream* s) {
    if (!s) return;
    cudaSetDevice(s->c->device);
    cudaFree(s->d_frames); cudaFree(s->d_mask); cudaFree(s->d_bits); cudaFree(s->d_wit); cudaFree(s->d_pass); cudaFree(s->d_dec);
    cudaFree(s->d_jobs); cudaFree(s->d_pairs); cudaFree(s->d_prefix); cudaFree(s->d_ones); cudaFree(s->d_resid); cudaFree(s->d_wlen); cudaFree(s->d_chunkcnt);
    cudaFree(s->d_fields); cudaFree(s->d_inflated);
    for (auto& e : s->ev) if (e) cudaEventDestroy(e);
    for (auto& e : s->ev_copy) if (e) cudaEventDestroy(e);
    cudaFreeHost(s->h_jobs); cudaFreeHost(s->h_pairs); cudaFreeHost(s->h_prefix); cudaFreeHost(s->h_ones); cudaFreeHost(s->h_resid); cudaFreeHost(s->h_wlen);
    delete s;
}

extern "C" int rbf_stream_create(rbf_ctx* c, uint32_t H, uint32_t W, uint32_t C, uint32_t S, uint32_t max_frames,
                                 uint32_t max_pairs, rbf_stream** out) {
    if (!c || !out) return set_err(c, RBF_ERR_INVALID, "rbf_stream_create: NULL");
    if (!(S == 1 || S == 2) || !(C == 1 || C == 3) || H == 0 || W == 0 || max_frames < 2 || max_pairs < 1)
        return set_err(c, RBF_ERR_INVALID, "unsupported frame format H=%u W=%u C=%u sample_bytes=%u", H, W, C, S);
    const uint64_t npix = (uint64_t)H * W;
    if (npix > 0xffffff00ULL) return set_err(c, RBF_ERR_INVALID, "frame too large");
    CK(c, cudaSetDevice(c->device));
    rbf_stream* s = new rbf_stream();
    s->c = c; s->H = H; s->W = W; s->C = C; s->S = S; s->max_frames = max_frames; s->max_pairs = max_pairs;
    s->npix = npix; s->frame_bytes = npix * C * S; s->frame_stride = align_up(s->frame_bytes + 64, 256);
    s->mask_stride_w = bit_words_padded(npix);
    s->pass_stride_w = pass_words(npix);
    cudaError_t e = cudaSuccess;
    auto dalloc = [&](void** p, size_t bytes) { if (e == cudaSuccess) e = cudaMalloc(p, bytes); };
    auto halloc = [&](void** p, size_t bytes) { if (e == cudaSuccess) e = cudaMallocHost(p, bytes); };
    dalloc((void**)&s->d_frames, s->frame_stride * max_frames);
    dalloc((void**)&s->d_mask, s->mask_stride_w * 4 * max_pairs);
    dalloc((void**)&s->d_bits, s->mask_stride_w * 4 * max_pairs);
    dalloc((void**)&s->d_wit, s->mask_stride_w * 4 * max_pairs);
    dalloc((void**)&s->d_pass, s->pass_stride_w * 4 * max_pairs);
    dalloc((void**)&s->d_jobs, sizeof(FrameJob) * max_pairs);
    dalloc((void**)&s->d_pairs, sizeof(PairJob) * max_pairs);
    dalloc((void**)&s->d_prefix, 4 * (3 * (size_t)max_pairs + 32));
    dalloc((void**)&s->d_ones, 4 * (size_t)max_pairs);
    dalloc((void**)&s->d_resid, 4 * (size_t)max_pairs);
    dalloc((void**)&s->d_wlen, 4 * (size_t)max_pairs);
    dalloc((void**)&s->d_chunkcnt, 4 * 32 * (size_t)max_pairs);
    halloc((void**)&s->h_jobs, sizeof(FrameJob) * max_pairs);
    halloc((void**)&s->h_pairs, sizeof(PairJob) * max_pairs);
    halloc((void**)&s->h_prefix, 4 * (3 * (size_t)max_pairs + 32));
    halloc((void**)&s->h_ones, 4 * (size_t)max_pairs);
    halloc((void**)&s->h_resid, 4 * (size_t)max_pairs);
    halloc((void**)&s->h_wlen, 4 * (size_t)max_pairs);
    if (e != cudaSuccess) {
        rbf_stream_destroy(s);
        return set_err(c, e == cudaErrorMemoryAllocation ? RBF_ERR_OOM : RBF_ERR_CUDA, "rbf_stream_create: %s", cudaGetErrorString(e));
    }
    for (auto& ev : s->ev) CK(c, cudaEventCreate(&ev));
    memset(s->h_ones, 0, 4 * (size_t)max_pairs); memset(s->h_resid, 0, 4 * (size_t)max_pairs); memset(s->h_wlen, 0, 4 * (size_t)max_pairs);
    s->k1_only = c->k1_only; s->mask_mode = c->mask_mode;
    CK(c, cudaMemsetAsync(s->d_wlen, 0, 4 * (size_t)max_pairs, c->st));
    CK(c, cudaMemsetAsync(s->d_bits, 0, s->mask_stride_w * 4 * max_pairs, c->st));
    CK(c, cudaMemsetAsync(s->d_wit, 0, s->mask_stride_w * 4 * max_pairs, c->st));
    CK(c, cudaMemsetAsync(s->d_mask, 0, s->mask_stride_w * 4 * max_pairs, c->st));   // zero padding once
    CK(c, cudaStreamSynchronize(c->st));
    *out = s;
    return RBF_OK;
}

extern "C" int rbf_stream_set_option(rbf_stream* s, const char* key, int64_t v) {
    if (!s || !key) return set_err(s ? s->c : nullptr, RBF_ERR_INVALID, "rbf_stream_set_option: NULL");
    if (!strcmp(key, "k1_only")) { s->k1_only = v ? 1 : 0; return RBF_OK; }
    if (!strcmp(key, "mask_mode")) { s->mask_mode = v ? 1 : 0; return RBF_OK; }
    if (!strcmp(key, "gray_mode")) {
        if (v && s->C != 3) return set_err(s->c, RBF_ERR_INVALID, "gray_mode needs 3-channel frames");
        s->gray_mode = v ? 1 : 0;
        return RBF_OK;
    }
    if (!strcmp(key, "value_mode")) {
        if (v != 0 && v != 1) return set_err(s->c, RBF_ERR_INVALID, "value_mode must be 0 (values) or 1 (residuals), not %lld", (long long)v);
        if (v && s->motion_values) return set_err(s->c, RBF_ERR_INVALID, "value_mode 1 and motion_values 1 exclude each other");
        s->value_mode = (int)v;
        return RBF_OK;
    }
    if (!strcmp(key, "motion_values")) {
        if (v != 0 && v != 1) return set_err(s->c, RBF_ERR_INVALID, "motion_values must be 0 or 1, not %lld", (long long)v);
        if (v && s->value_mode) return set_err(s->c, RBF_ERR_INVALID, "value_mode 1 and motion_values 1 exclude each other");
        if (v && s->motion_pairs == 0) return set_err(s->c, RBF_ERR_INVALID, "motion_values needs a motion search since the last encode");
        s->motion_values = (int)v;
        return RBF_OK;
    }
    return set_err(s->c, RBF_ERR_INVALID, "unknown stream option %s", key);
}

extern "C" int rbf_stream_upload(rbf_stream* s, uint32_t first, uint32_t count, const void* host) {
    if (!s || !host) return set_err(s ? s->c : nullptr, RBF_ERR_INVALID, "rbf_stream_upload: NULL");
    rbf_ctx* c = s->c;
    if ((uint64_t)first + count > s->max_frames) return set_err(c, RBF_ERR_INVALID, "frames [%u,%u) exceed store of %u", first, first + count, s->max_frames);
    CK(c, cudaMemcpy2DAsync(s->d_frames + (size_t)first * s->frame_stride, s->frame_stride, host, s->frame_bytes, s->frame_bytes,
                            count, cudaMemcpyHostToDevice, c->st));
    c->h2d += (int64_t)s->frame_bytes * count;
    CK(c, cudaStreamSynchronize(c->st));
    return RBF_OK;
}
extern "C" int rbf_stream_bitmap_region(rbf_stream* s, void** dptr, uint64_t* stride) {
    if (!s) return RBF_ERR_INVALID;
    if (dptr) *dptr = s->d_bits;
    if (stride) *stride = s->mask_stride_w * 4;
    return RBF_OK;
}

// `diff > threshold` with integer diff and a Python float threshold (ivc:808)  ==  diff > floor(threshold).  The int16 abs of 16-bit
// samples can be -32768 (ivc:801), so for them a threshold below -1 keeps its exact floor (down to -40000).
static int threshold_to_int(double thr, uint32_t sample_bytes) {
    if (isnan(thr)) return 0x7fffffff;                 // every comparison with NaN is False
    if (thr < -1.0) return sample_bytes == 2 ? (thr < -40000.0 ? -40000 : (int)floor(thr)) : -1;
    if (thr > 1e9) return 0x7fffffff;
    return (int)floor(thr);
}

// ---- steps of the batched encode, shared by rbf_stream_encode and rbf_stream_encode_host ---------------------------------
// The PairJobs of pairs [first, first+count) go to the device and their K1 counts are zeroed, on the context's stream.
static int enc_stage_pairs(rbf_stream* s, uint32_t first, uint32_t count, const uint32_t* prev_idx, const uint32_t* curr_idx) {
    rbf_ctx* c = s->c;
    for (uint32_t i = 0; i < count; i++) {
        if (prev_idx[i] >= s->max_frames || curr_idx[i] >= s->max_frames)
            return set_err(c, RBF_ERR_INVALID, "pair %u references a frame outside the store", first + i);
        PairJob& P = s->h_pairs[first + i];
        P.prev = s->d_frames + (size_t)prev_idx[i] * s->frame_stride;
        P.curr = s->d_frames + (size_t)curr_idx[i] * s->frame_stride;
        P.mask = s->d_mask + (size_t)(first + i) * s->mask_stride_w;
    }
    CK(c, cudaMemcpyAsync(s->d_pairs + first, s->h_pairs + first, sizeof(PairJob) * count, cudaMemcpyHostToDevice, c->st));
    CK(c, cudaMemsetAsync(s->d_ones + first, 0, 4 * (size_t)count, c->st));
    CK(c, cudaMemsetAsync(s->d_resid + first, 0, 4 * (size_t)count, c->st));
    return RBF_OK;
}

// Pairs of a consecutive run of frames (pairs[t].curr == pairs[t+1].prev) let K1 read each frame once instead of twice; its bulk
// copies also need 16 B aligned frames, which cudaMalloc and the 256-byte frame stride give.
static bool pairs_form_chain(const PairJob* h, uint32_t count) {
    if (count < 2) return false;
    for (uint32_t i = 0; i < count; i++) {
        if (((uintptr_t)h[i].prev | (uintptr_t)h[i].curr) & 15u) return false;
        if (i + 1 < count && h[i].curr != h[i + 1].prev) return false;
    }
    return true;
}

// K1 over pairs [f, f+cnt) on `st`, then the copy of their counts to the host.  sms > 0: on that many SMs, K2 runs beside it.
static int enc_k1(rbf_stream* s, uint32_t f, uint32_t cnt, int thr_int, int sms, cudaStream_t st) {
    rbf_ctx* c = s->c;
    CK(c, launch_threshold(c->L, s->d_pairs + f, (int)cnt, (uint32_t)s->npix, (int)s->C, (int)s->S, thr_int, s->mask_mode, s->gray_mode,
                           s->d_ones + f, s->d_resid + f, pairs_form_chain(s->h_pairs + f, cnt), sms, st));
    CK(c, cudaMemcpyAsync(s->h_ones + f, s->d_ones + f, 4 * (size_t)cnt, cudaMemcpyDeviceToHost, st));
    CK(c, cudaMemcpyAsync(s->h_resid + f, s->d_resid + f, 4 * (size_t)cnt, cudaMemcpyDeviceToHost, st));
    c->d2h += 8 * (int64_t)cnt;
    return RBF_OK;
}

// The FrameJob of pair slot i in h_jobs: the slot's bit array, witness and pass mask, and the filter of (l, k*) when l > 0.
// out == NULL: an encode job over the slot's mask; otherwise a decode job writing `out` from a witness of wlen bits.
static FrameJob& slot_job(rbf_stream* s, uint32_t i, uint64_t l, double k_star, const rbf_seeds& sd, uint32_t* out, uint64_t wlen) {
    const size_t mw = (size_t)i * s->mask_stride_w;
    FrameJob& J = s->h_jobs[i];
    J = frame_job(s->npix, l, k_star, sd, s->d_bits + mw, s->d_wit + mw, s->d_pass + (size_t)i * s->pass_stride_w);
    if (out) { J.out_mask = out; J.wlen_in = l ? (uint32_t)wlen : 0u; }
    else J.mask = s->d_mask + mw;
    return J;
}

struct RangeTotals {
    uint32_t total_cent = 0, coded_pairs = 0, max_l = 0;
};

// host side of pairs [first, first+count): K1's counts -> (p, k, l, T) exactly as the reference computes them -> FrameJob.
// hp[i+1] = base_cent + centuries of the coded pairs among the first i+1 of the range (K3's work list).
static void stream_range_params(rbf_stream* s, uint32_t first, uint32_t count, const rbf_seeds* sd, const double* kov,
                                const uint64_t* lov, uint32_t* hp, uint32_t base_cent, RangeTotals* out) {
    const uint32_t n = (uint32_t)s->npix, ncent = (n + 99u) / 100u;
    if (s->last_infos.size() < (size_t)first + count) s->last_infos.resize((size_t)first + count);
    uint32_t total_cent = base_cent;
    hp[0] = base_cent;
    for (uint32_t i = 0; i < count; i++) {
        rbf_mask_info& in = s->last_infos[first + i];
        memset(&in, 0, sizeof in);
        in.n = n; in.ones = s->h_ones[first + i]; in.resid = s->h_resid[first + i];
        double p, k; uint64_t l;
        int coded = rbf_optimal_params(n, in.ones, &p, &k, &l);
        in.p = p;
        if (kov && kov[i] > 0.0 && !(p >= kPStar)) { k = kov[i]; l = lov ? lov[i] : 0; coded = !(l == 0 || l >= n); }
        const FrameJob& J = slot_job(s, first + i, coded ? l : 0, k, *sd, nullptr, 0);
        if (coded) {
            in.k = k; in.l = l; in.floor_k = J.floor_k; in.act_T = J.act_T;
            total_cent += ncent; out->coded_pairs++;
            if (l > out->max_l) out->max_l = (uint32_t)l;
        } else {
            in.raw = 1;
        }
        hp[i + 1] = total_cent;
    }
    out->total_cent = total_cent - base_cent;
}

// The FrameJobs of pairs [f, f+cnt) go to the device, with their work list hp (cnt + 1 entries inside h_prefix, or NULL), then what
// K2 / K3b will OR into is zeroed, once the slot packing of a pending all-gather has read the bit arrays.  Nothing ever writes a bit
// array at or beyond bit l, or a witness at or beyond bit wlen, and both regions are fully zeroed at creation, so clearing
// [0, high-water mark) of every slot is enough.  Keep the work list behind the jobs: uploaded ahead of them, it held K2 of
// rbf_stream_encode_host's first chunk until every frame copy of the call had landed (+20 ms per 4K call on an H100 at 700 W).
// Every range and chunk of an encode is staged, whether or not it has a coded pair, so that after any encode a raw pair's rows read
// as zero and K3b never sees a job of an earlier call.  Copies and memsets only: kernel_launches does not count this step.
static int enc_stage_jobs(rbf_stream* s, uint32_t f, uint32_t cnt, uint32_t max_l, const uint32_t* hp) {
    rbf_ctx* c = s->c;
    CK(c, cudaMemcpyAsync(s->d_jobs + f, s->h_jobs + f, sizeof(FrameJob) * cnt, cudaMemcpyHostToDevice, c->st));
    if (hp) CK(c, cudaMemcpyAsync(s->d_prefix + (hp - s->h_prefix), hp, 4 * ((size_t)cnt + 1), cudaMemcpyHostToDevice, c->st));
    if (int r = wait_pack(c)) return r;
    const size_t stride = s->mask_stride_w * 4;
    const size_t need = align_up((size_t)((max_l + 31u) / 32u) * 4 + 64, 128);
    if (need > s->bits_hwm) s->bits_hwm = need;
    const size_t wb = s->bits_hwm < stride ? s->bits_hwm : stride;
    const size_t ww = (s->wit_dirty_full || s->wit_hwm > stride) ? stride : s->wit_hwm;
    CK(c, cudaMemset2DAsync(s->d_bits + (size_t)f * s->mask_stride_w, stride, 0, wb, cnt, c->st));
    if (ww) CK(c, cudaMemset2DAsync(s->d_wit + (size_t)f * s->mask_stride_w, stride, 0, ww, cnt, c->st));
    return RBF_OK;
}

// K3b over pairs [f, f+cnt) and the copy of their witness lengths to the host.  timed: the last two stage events bracket K3b,
// which completes the stage timings of rbf_stream_stage_ms.
static int enc_witness(rbf_stream* s, uint32_t f, uint32_t cnt, bool timed) {
    rbf_ctx* c = s->c;
    if (timed) CK(c, cudaEventRecord(s->ev[4], c->st));
    s->wit_dirty_full = true;                            // until the witness lengths of this encode are known
    CK(c, launch_witness(c->L, s->d_jobs + f, (int)cnt, (uint32_t)((s->npix + 99) / 100), s->d_chunkcnt + 32 * (size_t)f, s->d_wlen + f,
                         c->st));
    if (timed) { CK(c, cudaEventRecord(s->ev[5], c->st)); s->staged = true; }
    CK(c, cudaMemcpyAsync(s->h_wlen + f, s->d_wlen + f, 4 * (size_t)cnt, cudaMemcpyDeviceToHost, c->st));
    c->d2h += 4 * (int64_t)cnt;
    return RBF_OK;
}

// An encode starts: the slots hold no complete encode (fetch, gather and decode_verify refuse) until enc_finish.
static void enc_begin(rbf_stream* s, const rbf_seeds* sd) {
    s->last_infos.clear();
    s->last_pairs = 0; s->last_max_l = 0;
    s->motion_pairs = 0;
    s->staged = false;
    s->last_sd = *sd;
}

// After the encode of pairs [0, pairs) has been synchronised: what fetch, gather and decode_verify read, the witness high-water
// mark of the next encode's clear, and the caller's infos.
static void enc_finish(rbf_stream* s, uint32_t pairs, rbf_mask_info* infos) {
    const bool coded_run = !s->k1_only;
    s->last_pairs = pairs;
    s->last_k1_only = !coded_run;
    if (coded_run) {
        for (uint32_t i = 0; i < pairs; i++) {
            const size_t nb = align_up((size_t)((s->h_wlen[i] + 31u) / 32u) * 4 + 64, 128);
            if (nb > s->wit_hwm) s->wit_hwm = nb;
        }
        s->wit_dirty_full = false;
    }
    for (uint32_t i = 0; i < pairs; i++) {
        rbf_mask_info& in = s->last_infos[i];
        if (!in.raw && in.l > s->last_max_l) s->last_max_l = (uint32_t)in.l;
        if (coded_run && !in.raw) in.wlen = s->h_wlen[i];
        if (infos) infos[i] = in;
    }
}

// Encode pairs [first, first+count) serially on the context's stream (one chunk of rbf_stream_encode_host); `pfx` is the slot of this
// range's century-prefix array (count+1 entries) inside h_prefix/d_prefix.
static int stream_encode_range(rbf_stream* s, uint32_t first, uint32_t count, uint32_t pfx, const uint32_t* prev_idx,
                               const uint32_t* curr_idx, int thr_int, const rbf_seeds* sd) {
    rbf_ctx* c = s->c;
    if (int r = enc_stage_pairs(s, first, count, prev_idx, curr_idx)) return r;
    if (int r = enc_k1(s, first, count, thr_int, 0, c->st)) return r;
    CK(c, cudaStreamSynchronize(c->st));               // the one host round trip: (p, k, l, T) need libm's log2
    RangeTotals rt;
    uint32_t* hp = s->h_prefix + pfx;
    stream_range_params(s, first, count, sd, nullptr, nullptr, hp, 0, &rt);
    if (int r = enc_stage_jobs(s, first, count, rt.max_l, hp)) return r;   // also when all raw: the caller copies these rows out
    if (rt.coded_pairs == 0) return RBF_OK;
    CK(c, launch_insert(c->L, s->d_jobs + first, (int)count, (uint32_t)((s->npix + 99) / 100), rt.max_l, c->L.sm_count, c->st));
    CK(c, launch_query(c->L, s->d_jobs + first, s->d_prefix + pfx, (int)count, rt.total_cent, rt.max_l, c->st));
    return enc_witness(s, first, count, false);
}

static int ensure_pipe_streams(rbf_ctx* c) {
    if (!c->st_k1) {
        CK(c, cudaStreamCreateWithFlags(&c->st_k1, cudaStreamNonBlocking));
        CK(c, cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
        for (auto& e : c->ev_k1) CK(c, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    }
    return RBF_OK;
}

// The resident-stream encode, pipelined over R ranges of pairs: K1 has no host dependency, so K1 of ALL ranges is enqueued up
// front on a second stream.  K1 of range 0 takes the whole GPU.  K1 of ranges 1.. runs on pipe_k1_sms SMs only, in CTAs whose
// shared memory keeps K2 off those SMs (over the whole GPU K1 is HBM-bound; 66 of 132 SMs still pull 70 % of that bandwidth,
// DESIGN §4).  As soon as range
// r's counts have landed, the host derives its (k, l, T) while K1 of range r+1 runs, and enqueues K2 of range r on the main
// stream, sized for the SMs K1 leaves free; K2 of the last range has nothing beside it and gets every SM.
// K3 and K3b are single launches over all pairs.
static int stream_encode_pipelined(rbf_stream* s, uint32_t pairs, const uint32_t* prev_idx, const uint32_t* curr_idx,
                                   double threshold, const rbf_seeds* sd, const double* kov, const uint64_t* lov) {
    rbf_ctx* c = s->c;
    const uint32_t ncent = (uint32_t)((s->npix + 99) / 100);
    const int thr_int = threshold_to_int(threshold, s->S);
    uint32_t R = (uint32_t)c->encode_ranges;
    if (R > 8u) R = 8u;
    if (pairs < 8u * R) R = 1u;                          // small jobs: nothing to hide behind
    const int k1_sms = c->pipe_k1_sms < c->L.sm_count ? c->pipe_k1_sms : c->L.sm_count - 1;   // K1 beside K2
    if (int r = ensure_pipe_streams(c)) return r;
    if (int r = enc_stage_pairs(s, 0, pairs, prev_idx, curr_idx)) return r;
    enc_begin(s, sd);
    CK(c, cudaEventRecord(s->ev[0], c->st));
    CK(c, cudaEventRecord(c->ev_fork, c->st));
    CK(c, cudaStreamWaitEvent(c->st_k1, c->ev_fork, 0));
    uint32_t lo[9];
    for (uint32_t r = 0; r <= R; r++) lo[r] = (uint32_t)(((uint64_t)pairs * r) / R);
    for (uint32_t r = 0; r < R; r++) {
        if (int e = enc_k1(s, lo[r], lo[r + 1] - lo[r], thr_int, r > 0 ? k1_sms : 0, c->st_k1)) return e;
        CK(c, cudaEventRecord(c->ev_k1[r], c->st_k1));
    }
    CK(c, cudaEventRecord(s->ev[1], c->st_k1));           // end of the last K1
    RangeTotals all;
    uint32_t base_cent = 0;
    bool first_k2 = true;
    // K2 || K3 mode (kq_ranges > 1, serial K1): K2 of range q+1 is enqueued on the second stream beside K3 of range q.  Both
    // kernels take nearly all of an SM's shared memory, so a K2 CTA only starts on an SM without a K3 CTA: the two stages
    // share the GPU by SMs, not within one.
    uint32_t Q = (R == 1u && !s->k1_only) ? (uint32_t)c->kq_ranges : 1u;
    if (Q > 8u) Q = 8u;
    if (pairs < 8u * Q) Q = 1u;
    const bool kq = Q > 1u;
    for (uint32_t r = 0; r < R; r++) {
        const uint32_t f = lo[r], cnt = lo[r + 1] - lo[r];
        CK(c, cudaEventSynchronize(c->ev_k1[r]));         // this range's counts are on the host
        RangeTotals rt;                                    // the overrides are per pair: range r reads entries [f, f+cnt)
        stream_range_params(s, f, cnt, sd, kov ? kov + f : nullptr, lov ? lov + f : nullptr, s->h_prefix + f, base_cent, &rt);
        base_cent += rt.total_cent;
        all.coded_pairs += rt.coded_pairs;
        if (rt.max_l > all.max_l) all.max_l = rt.max_l;
        if (s->k1_only) continue;
        CK(c, cudaStreamWaitEvent(c->st, c->ev_k1[r], 0)); // K2 reads the masks K1 wrote on the other stream
        // a range without a coded pair is staged too: K3b runs over every pair's job, and its raw rows must read as zero
        if (int e = enc_stage_jobs(s, f, cnt, rt.max_l, nullptr)) return e;   // the work list goes up once, for all ranges
        if (rt.coded_pairs == 0) continue;
        if (first_k2) { CK(c, cudaEventRecord(s->ev[2], c->st)); first_k2 = false; }
        if (!kq) CK(c, launch_insert(c->L, s->d_jobs + f, (int)cnt, ncent, rt.max_l, r + 1 < R ? c->L.sm_count - k1_sms : c->L.sm_count, c->st));
    }
    if (s->k1_only || all.coded_pairs == 0) {
        CK(c, cudaStreamWaitEvent(c->st, c->ev_k1[R - 1], 0));
        return RBF_OK;
    }
    CK(c, cudaMemcpyAsync(s->d_prefix, s->h_prefix, 4 * ((size_t)pairs + 1), cudaMemcpyHostToDevice, c->st));
    if (kq) {
        uint32_t qlo[9];
        for (uint32_t q = 0; q <= Q; q++) qlo[q] = (uint32_t)(((uint64_t)pairs * q) / Q);
        // per-range work lists for K3 (each starts at 0), behind the whole-encode list
        uint32_t* hp2 = s->h_prefix + pairs + 1;
        uint32_t off = 0, range_cent[8], range_off[8];
        for (uint32_t q = 0; q < Q; q++) {
            range_off[q] = off;
            const uint32_t b0 = s->h_prefix[qlo[q]];
            for (uint32_t i = qlo[q]; i <= qlo[q + 1]; i++) hp2[off++] = s->h_prefix[i] - b0;
            range_cent[q] = s->h_prefix[qlo[q + 1]] - b0;
        }
        CK(c, cudaMemcpyAsync(s->d_prefix + pairs + 1, hp2, 4 * (size_t)off, cudaMemcpyHostToDevice, c->st));
        CK(c, cudaEventRecord(c->ev_fork, c->st));            // jobs, prefix lists and cleared outputs are in place
        CK(c, cudaStreamWaitEvent(c->st_k1, c->ev_fork, 0));
        for (uint32_t q = 0; q < Q; q++) {
            const uint32_t f = qlo[q], cnt = qlo[q + 1] - qlo[q];
            CK(c, launch_insert(c->L, s->d_jobs + f, (int)cnt, ncent, all.max_l, c->L.sm_count, c->st_k1));
            CK(c, cudaEventRecord(c->ev_k1[q], c->st_k1));
            CK(c, cudaStreamWaitEvent(c->st, c->ev_k1[q], 0));
            if (q == 0) CK(c, cudaEventRecord(s->ev[3], c->st));
            CK(c, launch_query(c->L, s->d_jobs + f, s->d_prefix + pairs + 1 + range_off[q], (int)cnt, range_cent[q], all.max_l, c->st));
        }
    } else {
        CK(c, cudaEventRecord(s->ev[3], c->st));
        CK(c, launch_query(c->L, s->d_jobs, s->d_prefix, (int)pairs, base_cent, all.max_l, c->st));
    }
    return enc_witness(s, 0, pairs, true);
}

extern "C" int rbf_stream_encode(rbf_stream* s, const uint32_t* prev_idx, const uint32_t* curr_idx, uint32_t pairs,
                                 double threshold, const rbf_seeds* sd, const double* kov, const uint64_t* lov,
                                 rbf_mask_info* infos) {
    if (!s || !prev_idx || !curr_idx || !sd) return set_err(s ? s->c : nullptr, RBF_ERR_INVALID, "rbf_stream_encode: NULL");
    rbf_ctx* c = s->c;
    if (pairs == 0 || pairs > s->max_pairs) return set_err(c, RBF_ERR_INVALID, "pairs = %u outside [1, %u]", pairs, s->max_pairs);
    CK(c, cudaSetDevice(c->device));
    int rc = stream_encode_pipelined(s, pairs, prev_idx, curr_idx, threshold, sd, kov, lov);
    if (rc) { cudaStreamSynchronize(c->st_k1); cudaStreamSynchronize(c->st); return rc; }
    CK(c, cudaStreamSynchronize(c->st));
    enc_finish(s, pairs, infos);
    return RBF_OK;
}

extern "C" int rbf_stream_stage_ms(rbf_stream* s, double out[6]) {
    if (!s || !out) return RBF_ERR_INVALID;
    rbf_ctx* c = s->c;
    if (!s->staged) return set_err(c, RBF_ERR_STATE, "no fully staged encode has run");
    CK(c, cudaEventSynchronize(s->ev[5]));
    auto span = [&](int a, int b, double* o) -> cudaError_t { float f = 0; cudaError_t e = cudaEventElapsedTime(&f, s->ev[a], s->ev[b]); *o = f; return e; };
    CK(c, span(0, 1, &out[0]));     // K1: first launch .. end of the last range (runs beside K2 of the earlier ranges)
    CK(c, span(0, 3, &out[1]));     // everything in front of K3: K1 + host (k, l, T) round trips + K2, as overlapped
    CK(c, span(2, 3, &out[2]));     // K2: first launch .. end of the last range
    CK(c, span(3, 4, &out[3]));     // K3
    CK(c, span(4, 5, &out[4]));     // K3b (pass count, witness, packbits order)
    CK(c, span(0, 5, &out[5]));     // whole encode
    return RBF_OK;
}

// Pairs [first, first+count) of a per-pair device region into host rows of `slot` bytes, row 0 for pair `first` (a row takes what fits
// of its pair's slot); no copy when host is NULL or slot is 0.
static int copy_slots_d2h(rbf_stream* s, uint8_t* host, uint64_t slot, const uint32_t* region, uint32_t first, uint32_t count, cudaStream_t st) {
    if (!host || !slot) return RBF_OK;
    const size_t stride = s->mask_stride_w * 4, w = slot < stride ? (size_t)slot : stride;
    CK(s->c, cudaMemcpy2DAsync(host, slot, (const uint8_t*)region + (size_t)first * stride, stride, w, count, cudaMemcpyDeviceToHost, st));
    s->c->d2h += (int64_t)w * count;
    return RBF_OK;
}

// One strided copy per output kind for pairs [first, first+count) and ONE synchronisation (the GOP loop's batched fetch).
extern "C" int rbf_stream_fetch_batch(rbf_stream* s, uint32_t first, uint32_t count, uint8_t* bitmaps, uint64_t bitmap_slot,
                                      uint8_t* witness, uint64_t witness_slot, uint8_t* masks_little, uint64_t mask_slot) {
    if (!s) return RBF_ERR_INVALID;
    rbf_ctx* c = s->c;
    if (count == 0 || (uint64_t)first + count > s->last_pairs) return set_err(c, RBF_ERR_INVALID, "pairs [%u,%u) were not encoded", first, first + count);
    if (s->last_k1_only && (bitmaps || witness))
        return set_err(c, RBF_ERR_STATE, "the last encode stopped after K1 (k1_only): there is no bitmap / witness to fetch");
    int r;
    if ((r = copy_slots_d2h(s, bitmaps, bitmap_slot, s->d_bits, first, count, c->st)) ||
        (r = copy_slots_d2h(s, witness, witness_slot, s->d_wit, first, count, c->st)) ||
        (r = copy_slots_d2h(s, masks_little, mask_slot, s->d_mask, first, count, c->st)))
        return r;
    CK(c, cudaStreamSynchronize(c->st));
    return RBF_OK;
}

extern "C" int rbf_stream_encode_host(rbf_stream* s, const void* host_frames, uint32_t nframes, double threshold,
                                      const rbf_seeds* sd, rbf_mask_info* infos, uint8_t* bitmaps, uint64_t bitmap_slot,
                                      uint8_t* witness, uint64_t witness_slot) {
    if (!s || !host_frames || !sd || nframes < 2) return set_err(s ? s->c : nullptr, RBF_ERR_INVALID, "rbf_stream_encode_host: bad argument");
    rbf_ctx* c = s->c;
    const uint32_t pairs = nframes - 1;
    if (nframes > s->max_frames || pairs > s->max_pairs) return set_err(c, RBF_ERR_INVALID, "stream too small for %u frames", nframes);
    CK(c, cudaSetDevice(c->device));
    if (!c->st_copy) CK(c, cudaStreamCreateWithFlags(&c->st_copy, cudaStreamNonBlocking));
    if (!c->st_d2h) { CK(c, cudaStreamCreateWithFlags(&c->st_d2h, cudaStreamNonBlocking)); CK(c, cudaEventCreateWithFlags(&c->ev_d2h, cudaEventDisableTiming)); }
    if (s->k1_only) return set_err(c, RBF_ERR_STATE, "rbf_stream_encode_host on a k1_only stream");
    // chunks of frames: all H2D copies are queued on the copy stream up front (pinned source), the compute stream
    // encodes a chunk's pairs as soon as its frames have landed, so PCIe transfer and kernels overlap
    const uint32_t CH = c->host_chunk_frames > 1 ? (uint32_t)c->host_chunk_frames : 32u;
    const uint32_t nchunks = (nframes + CH - 1) / CH;
    while (s->ev_copy.size() < nchunks) { cudaEvent_t e; CK(c, cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); s->ev_copy.push_back(e); }
    const uint8_t* src = (const uint8_t*)host_frames;
    for (uint32_t k = 0; k < nchunks; k++) {
        const uint32_t f0 = k * CH, f1 = (f0 + CH < nframes) ? f0 + CH : nframes;
        CK(c, cudaMemcpy2DAsync(s->d_frames + (size_t)f0 * s->frame_stride, s->frame_stride, src + (size_t)f0 * s->frame_bytes,
                                s->frame_bytes, s->frame_bytes, f1 - f0, cudaMemcpyHostToDevice, c->st_copy));
        CK(c, cudaEventRecord(s->ev_copy[k], c->st_copy));
    }
    c->h2d += (int64_t)s->frame_bytes * nframes;
    enc_begin(s, sd);
    const int thr_int = threshold_to_int(threshold, s->S);
    std::vector<uint32_t> pi, ci;
    for (uint32_t k = 0; k < nchunks; k++) {
        const uint32_t f0 = k * CH, f1 = (f0 + CH < nframes) ? f0 + CH : nframes;
        const uint32_t p0 = f0 == 0 ? 0 : f0 - 1, p1 = f1 - 1;      // pairs (i, i+1) whose current frame is in this chunk
        if (p1 <= p0) continue;
        const uint32_t cnt = p1 - p0;
        pi.resize(cnt); ci.resize(cnt);
        for (uint32_t i = 0; i < cnt; i++) { pi[i] = p0 + i; ci[i] = p0 + i + 1; }
        CK(c, cudaStreamWaitEvent(c->st, s->ev_copy[k], 0));
        if (int rc = stream_encode_range(s, p0, cnt, p0 + k, pi.data(), ci.data(), thr_int, sd)) return rc;
        // the packed results of this chunk go back on their own stream, beside the kernels of the next chunk
        CK(c, cudaEventRecord(c->ev_d2h, c->st));
        CK(c, cudaStreamWaitEvent(c->st_d2h, c->ev_d2h, 0));
        int r;
        if ((r = copy_slots_d2h(s, bitmaps ? bitmaps + (size_t)p0 * bitmap_slot : nullptr, bitmap_slot, s->d_bits, p0, cnt, c->st_d2h)) ||
            (r = copy_slots_d2h(s, witness ? witness + (size_t)p0 * witness_slot : nullptr, witness_slot, s->d_wit, p0, cnt, c->st_d2h)))
            return r;
    }
    CK(c, cudaEventRecord(c->ev_d2h, c->st_d2h));        // the caller's timer / next call on `st` sees the copies done
    CK(c, cudaStreamWaitEvent(c->st, c->ev_d2h, 0));
    CK(c, cudaStreamSynchronize(c->st));
    enc_finish(s, pairs, infos);
    return RBF_OK;
}

extern "C" int rbf_stream_decode_verify(rbf_stream* s, uint32_t pairs, uint64_t* mismatches) {
    if (!s || !mismatches) return set_err(s ? s->c : nullptr, RBF_ERR_INVALID, "rbf_stream_decode_verify: NULL");
    rbf_ctx* c = s->c;
    if (pairs == 0 || pairs > s->last_pairs) return set_err(c, RBF_ERR_INVALID, "only %u pairs were encoded", s->last_pairs);
    CK(c, cudaSetDevice(c->device));
    const size_t stride_w = s->mask_stride_w;
    if (!s->d_dec) CK(c, cudaMalloc((void**)&s->d_dec, stride_w * 4 * s->max_pairs));
    CK(c, cudaMemsetAsync(s->d_dec, 0, stride_w * 4 * pairs, c->st));
    // bitmap and witness sit in packbits order after K3b; the kernels work LSB-first
    if (int r = wait_pack(c)) return r;
    CK(c, launch_bitrev(c->L, s->d_bits, stride_w * pairs, c->st));
    CK(c, launch_bitrev(c->L, s->d_wit, stride_w * pairs, c->st));
    // the decode jobs and their work list come from what the encode stored; a real decode knows no mask (ivc:286-304)
    const uint32_t ncent = (uint32_t)((s->npix + 99) / 100);
    s->h_prefix[0] = 0;
    for (uint32_t i = 0; i < pairs; i++) {
        const rbf_mask_info& in = s->last_infos[i];
        slot_job(s, i, in.raw ? 0 : in.l, in.k, s->last_sd, s->d_dec + (size_t)i * stride_w, in.wlen);
        s->h_prefix[i + 1] = s->h_prefix[i] + (in.raw ? 0 : ncent);
    }
    if (int r = decode_enqueue(c, s->h_jobs, s->d_jobs, s->h_prefix, s->d_prefix, (int)pairs, s->last_max_l, ncent, s->d_chunkcnt, s->d_wlen))
        return r;
    void* d_cnt; int rc;
    if ((rc = scratch_get(c, kScrSmall, 4 * (size_t)pairs + 4096, &d_cnt))) return rc;
    CK(c, cudaMemsetAsync(d_cnt, 0, 4 * (size_t)pairs, c->st));
    CK(c, launch_count_diff(c->L, s->d_mask, s->d_dec, stride_w, (s->npix + 31) / 32, (int)pairs, (uint32_t*)d_cnt, c->st));
    CK(c, launch_bitrev(c->L, s->d_bits, stride_w * pairs, c->st));
    CK(c, launch_bitrev(c->L, s->d_wit, stride_w * pairs, c->st));
    std::vector<uint32_t> h(pairs);
    CK(c, cudaMemcpyAsync(h.data(), d_cnt, 4 * (size_t)pairs, cudaMemcpyDeviceToHost, c->st));
    CK(c, cudaStreamSynchronize(c->st));
    for (uint32_t i = 0; i < pairs; i++) mismatches[i] = s->last_infos[i].raw ? 0 : h[i];
    return RBF_OK;
}


// ------------------------------------------------------------------------------------------
// N1 / N2: changed-value gather and frame reconstruction on the device
// ------------------------------------------------------------------------------------------
// byte offsets [pairs + 1] of the encoded pairs' changed values (set pixels x pixel bytes); returns the total
static uint64_t changed_offsets(const rbf_stream* s, uint32_t pairs, uint64_t* offs) {
    const uint64_t pb = (uint64_t)s->C * s->S;
    offs[0] = 0;
    for (uint32_t i = 0; i < pairs; i++) offs[i + 1] = offs[i] + s->last_infos[i].ones * pb;
    return offs[pairs];
}

// The changed values of the encoded pairs [0, pairs) gathered at offs into the values scratch slot, on the context's stream
// (value_mode 1: residuals against each pair's previous frame; motion_values 1: against its motion-compensated previous frame).
static int gather_values(rbf_stream* s, uint32_t pairs, const uint64_t* offs, uint8_t** d_values) {
    rbf_ctx* c = s->c;
    const uint32_t pb = s->C * s->S;
    if (s->motion_values && pairs > s->motion_pairs)
        return set_err(c, RBF_ERR_INVALID, "motion_values: %u pairs were searched since the last encode, %u are gathered", s->motion_pairs, pairs);
    const size_t field_bytes = (size_t)mv_blocks(s->H, s->W) * 2;
    void *d_vals = nullptr, *d_jobs = nullptr, *d_gcnt = nullptr;
    int rc;
    if ((rc = scratch_get(c, kScrValues, (size_t)offs[pairs] + 256, &d_vals)) ||
        (rc = scratch_get(c, kScrGatherJobs, sizeof(GatherJob) * pairs, &d_jobs)) ||
        (rc = scratch_get(c, kScrGatherCounts, 4 * (size_t)pairs * gather_chunks((uint32_t)s->npix) + 64, &d_gcnt)))
        return rc;
    std::vector<GatherJob> jobs(pairs);
    for (uint32_t i = 0; i < pairs; i++) {
        GatherJob& J = jobs[i];
        J.mask = s->d_mask + (size_t)i * s->mask_stride_w;
        J.frame = s->h_pairs[i].curr;
        J.prev = s->h_pairs[i].prev;
        J.values = (uint8_t*)d_vals + offs[i];
        J.npix = (uint32_t)s->npix;
        J.pix_bytes = pb;
        J.width = s->W;
        J.field = s->motion_values ? s->d_fields + i * field_bytes : nullptr;
    }
    CK(c, cudaMemcpyAsync(d_jobs, jobs.data(), sizeof(GatherJob) * pairs, cudaMemcpyHostToDevice, c->st));   // pageable: staged before return
    CK(c, launch_gather(c->L, (const GatherJob*)d_jobs, (int)pairs, (uint32_t)s->npix, pb, s->S, s->motion_values ? 2 : s->value_mode,
                        (uint32_t*)d_gcnt, c->st));
    *d_values = (uint8_t*)d_vals;
    return RBF_OK;
}

extern "C" int rbf_stream_gather_changed(rbf_stream* s, uint32_t pairs, uint8_t* values_out, uint64_t capacity,
                                         uint64_t* offsets_out) {
    if (!s || !offsets_out) return set_err(s ? s->c : nullptr, RBF_ERR_INVALID, "rbf_stream_gather_changed: NULL");
    rbf_ctx* c = s->c;
    if (pairs == 0 || pairs > s->last_pairs) return set_err(c, RBF_ERR_INVALID, "only %u pairs were encoded", s->last_pairs);
    CK(c, cudaSetDevice(c->device));
    const uint64_t total = changed_offsets(s, pairs, offsets_out);
    if (!values_out) return RBF_OK;                      // size query
    if (capacity < total) return set_err(c, RBF_ERR_INVALID, "values buffer too small: %llu < %llu", (unsigned long long)capacity, (unsigned long long)total);
    uint8_t* d_vals;
    if (int r = gather_values(s, pairs, offsets_out, &d_vals)) return r;
    if (total) { CK(c, cudaMemcpyAsync(values_out, d_vals, (size_t)total, cudaMemcpyDeviceToHost, c->st)); c->d2h += (int64_t)total; }
    CK(c, cudaStreamSynchronize(c->st));
    return RBF_OK;
}

// ------------------------------------------------------------------------------------------
// K4b / K4c batched: the inter frames of a group decoded with one query + expand and rebuilt along the chain in one sweep
// ------------------------------------------------------------------------------------------
extern "C" int rbf_stream_decode_masks(rbf_stream* s, uint32_t count, const uint8_t* bitmaps, uint64_t bitmap_slot,
                                       const uint8_t* witness, uint64_t witness_slot, const uint64_t* l, const uint64_t* wlen,
                                       const double* k, const uint8_t* raw, const rbf_seeds* sd, uint64_t* consumed_out,
                                       uint64_t* ones_out) {
    if (!s || !bitmaps || !l || !wlen || !k || !raw || !sd || !consumed_out || !ones_out || (witness_slot && !witness))
        return set_err(s ? s->c : nullptr, RBF_ERR_INVALID, "rbf_stream_decode_masks: NULL");
    rbf_ctx* c = s->c;
    const uint64_t n = s->npix, stride = s->mask_stride_w * 4;
    if (count == 0 || count > s->max_pairs) return set_err(c, RBF_ERR_INVALID, "%u pairs for a stream of %u", count, s->max_pairs);
    if (bitmap_slot == 0 || bitmap_slot > stride || witness_slot > stride)
        return set_err(c, RBF_ERR_INVALID, "slots of %llu / %llu bytes exceed the device slot of %llu", (unsigned long long)bitmap_slot,
                       (unsigned long long)witness_slot, (unsigned long long)stride);
    for (uint32_t i = 0; i < count; i++) {
        if (raw[i]) {
            if (bitmap_slot < (n + 7) / 8) return set_err(c, RBF_ERR_INVALID, "pair %u: a raw mask needs %llu bytes", i, (unsigned long long)((n + 7) / 8));
        } else if (l[i] == 0 || l[i] > 0xffffffffULL || l[i] > 8 * bitmap_slot || wlen[i] == 0 || wlen[i] > 8 * witness_slot || !(k[i] >= 0.0)) {
            return set_err(c, RBF_ERR_INVALID, "pair %u: bad l / wlen / k", i);
        }
    }
    CK(c, cudaSetDevice(c->device));
    if (int r = wait_pack(c)) return r;                  // the bit arrays are overwritten
    void* d_cnt;
    if (int r = scratch_get(c, kScrDecodeCounts, 8 * (size_t)count, &d_cnt)) return r;
    uint32_t* d_consumed = (uint32_t*)d_cnt;
    uint32_t* d_ones = d_consumed + count;
    CK(c, cudaMemcpy2DAsync(s->d_bits, stride, bitmaps, bitmap_slot, bitmap_slot, count, cudaMemcpyHostToDevice, c->st));
    c->h2d += (int64_t)(bitmap_slot * count);
    if (witness_slot) {
        CK(c, cudaMemcpy2DAsync(s->d_wit, stride, witness, witness_slot, witness_slot, count, cudaMemcpyHostToDevice, c->st));
        c->h2d += (int64_t)(witness_slot * count);
    }
    // packbits order -> LSB-first words.  k_bitrev reverses each byte in place, so whatever lies past a slot is only reordered,
    // and nothing reads a bit array at or past bit l or a witness at or past bit wlen
    CK(c, launch_bitrev(c->L, s->d_bits, s->mask_stride_w * count, c->st));
    if (witness_slot) CK(c, launch_bitrev(c->L, s->d_wit, s->mask_stride_w * count, c->st));
    CK(c, cudaMemsetAsync(s->d_mask, 0, stride * count, c->st));       // K4b ORs into the mask slots
    CK(c, cudaMemsetAsync(d_cnt, 0, 8 * (size_t)count, c->st));
    const uint32_t ncent = (uint32_t)((n + 99) / 100);
    uint32_t total_cent = 0, max_l = 0, coded = 0;
    s->h_prefix[0] = 0;
    for (uint32_t i = 0; i < count; i++) {
        const uint64_t li = raw[i] ? 0 : l[i];                // the payload's float64 k (ivc:275-279)
        slot_job(s, i, li, k[i], *sd, s->d_mask + (size_t)i * s->mask_stride_w, wlen[i]);
        if (li) { total_cent += ncent; coded++; }
        if (li > max_l) max_l = (uint32_t)li;
        s->h_prefix[i + 1] = total_cent;
    }
    if (coded) {
        if (int r = decode_enqueue(c, s->h_jobs, s->d_jobs, s->h_prefix, s->d_prefix, (int)count, max_l, ncent, s->d_chunkcnt, d_consumed))
            return r;
    } else {
        CK(c, cudaMemcpyAsync(s->d_jobs, s->h_jobs, sizeof(FrameJob) * count, cudaMemcpyHostToDevice, c->st));
    }
    if (coded < count) CK(c, launch_raw_masks(c->L, s->d_jobs, (int)count, (uint32_t)n, c->st));
    CK(c, launch_mask_popcount(c->L, s->d_mask, s->mask_stride_w, (uint32_t)n, (int)count, d_ones, c->st));
    std::vector<uint32_t> h(2 * (size_t)count);
    CK(c, cudaMemcpyAsync(h.data(), d_cnt, 8 * (size_t)count, cudaMemcpyDeviceToHost, c->st));
    c->d2h += 8 * (int64_t)count;
    CK(c, cudaStreamSynchronize(c->st));
    for (uint32_t i = 0; i < count; i++) { consumed_out[i] = raw[i] ? 0 : h[i]; ones_out[i] = h[count + i]; }
    // the slots no longer hold the outputs of an encode: refuse fetch / gather / decode_verify until the next one, and let the next
    // encode clear what was written here
    s->last_pairs = 0; s->last_max_l = 0; s->staged = false; s->motion_pairs = 0;
    const size_t bh = align_up((size_t)bitmap_slot + 64, 128), wh = align_up((size_t)witness_slot + 64, 128);
    if (bh > s->bits_hwm) s->bits_hwm = bh;
    if (witness_slot && wh > s->wit_hwm) s->wit_hwm = wh;
    return RBF_OK;
}

// K4c over pairs [0, count) from base_frame: pair i's mask at d_masks + i * mask_stride_w, its values at d_vals + value_offsets[i]
// (device), modes / fields as in rbf_stream_apply_chain, already validated (field_bytes: 0 when no field is read).  One H2D copy of
// the offsets with the modes and fields behind them, one synchronisation.  *first_bad_out (may be NULL): the first pair whose value
// count does not match its mask (ivc:882), UINT32_MAX when none.
static int stream_apply_chain(rbf_stream* s, uint32_t base_frame, uint32_t count, const uint8_t* d_vals, const uint64_t* value_offsets,
                              const uint8_t* modes, const int8_t* fields, size_t field_bytes, const uint32_t* d_masks,
                              size_t mask_stride_w, uint64_t* applied_out, uint32_t* first_bad_out) {
    rbf_ctx* c = s->c;
    const uint32_t ntiles = (uint32_t)((s->npix + AP_TILE_PX - 1) / AP_TILE_PX);
    void *d_small, *d_pfx;
    int rc;
    // d_small: the value offsets, then the modes, then the fields (one H2D copy for all three), then first_bad and the totals
    const size_t off_bytes = 8 * ((size_t)count + 1), flag_bytes = modes ? count : 0;
    const size_t res_at = align_up(off_bytes + flag_bytes + field_bytes, 16);
    const size_t small = res_at + 4 * ((size_t)count + 1) + (field_bytes ? 4 * (size_t)count : 0);   // + the runs' first_bad words
    if ((rc = scratch_get(c, kScrChainSmall, small, &d_small)) || (rc = scratch_get(c, kScrChainTiles, 4 * (size_t)count * ntiles, &d_pfx)))
        return rc;
    uint64_t* d_off = (uint64_t*)d_small;
    uint32_t* d_res = (uint32_t*)((uint8_t*)d_small + res_at);   // [0] first_bad, [1 + i] totals
    if (modes) {
        std::vector<uint8_t> head(off_bytes + flag_bytes + field_bytes);
        memcpy(head.data(), value_offsets, off_bytes);
        memcpy(head.data() + off_bytes, modes, flag_bytes);
        if (field_bytes) memcpy(head.data() + off_bytes + flag_bytes, fields, field_bytes);
        CK(c, cudaMemcpyAsync(d_off, head.data(), head.size(), cudaMemcpyHostToDevice, c->st));   // pageable: staged before return
    } else {
        CK(c, cudaMemcpyAsync(d_off, value_offsets, off_bytes, cudaMemcpyHostToDevice, c->st));
    }
    c->h2d += (int64_t)(off_bytes + flag_bytes + field_bytes);
    CK(c, cudaMemsetAsync(d_res, 0xff, 4, c->st));
    ApplyChain A;
    A.masks = d_masks; A.mask_stride_w = mask_stride_w;
    A.frames = s->d_frames; A.frame_stride = s->frame_stride;
    A.max_frames = s->max_frames; A.base = base_frame;
    A.npix = (uint32_t)s->npix; A.ntiles = ntiles; A.count = count; A.pix_bytes = s->C * s->S;
    A.values = d_vals; A.value_off = d_off;
    A.sample_bytes = s->S;
    A.tile_pfx = (uint32_t*)d_pfx; A.totals = d_res + 1; A.first_bad = d_res;
    A.residual = modes ? (const uint8_t*)d_small + off_bytes : nullptr;     // read by runs with a mode-1 or mode-2 pair only
    CK(c, launch_apply_chain(c->L, A, modes, field_bytes ? (const int8_t*)d_small + off_bytes + flag_bytes : nullptr, s->H, s->W,
                             d_res + 1 + count, c->st));
    std::vector<uint32_t> h((size_t)count + 1);
    CK(c, cudaMemcpyAsync(h.data(), d_res, 4 * ((size_t)count + 1), cudaMemcpyDeviceToHost, c->st));
    c->d2h += 4 * ((int64_t)count + 1);
    CK(c, cudaStreamSynchronize(c->st));
    for (uint32_t i = 0; i < count; i++) applied_out[i] = i < h[0] ? h[1 + i] : 0;
    if (first_bad_out) *first_bad_out = h[0];
    return RBF_OK;
}

extern "C" int rbf_stream_apply_chain(rbf_stream* s, uint32_t base_frame, uint32_t count, const uint8_t* values,
                                      const uint64_t* value_offsets, const uint8_t* modes, const int8_t* fields, uint64_t* applied_out) {
    if (!s || !value_offsets || !applied_out) return set_err(s ? s->c : nullptr, RBF_ERR_INVALID, "rbf_stream_apply_chain: NULL");
    rbf_ctx* c = s->c;
    const uint64_t vbytes = value_offsets[count];
    if (!values) {                                       // the bytes the last rbf_stream_inflate_values placed, read by one call
        if (vbytes > s->inflated_bytes)
            return set_err(c, RBF_ERR_INVALID, "rbf_stream_apply_chain: %llu value bytes, %llu inflated", (unsigned long long)vbytes,
                           (unsigned long long)s->inflated_bytes);
        s->inflated_bytes = 0;
    }
    if (count == 0 || count > s->max_pairs || count >= s->max_frames || base_frame >= s->max_frames)
        return set_err(c, RBF_ERR_INVALID, "chain of %u frames from slot %u does not fit a store of %u frames / %u pairs", count,
                       base_frame, s->max_frames, s->max_pairs);
    for (uint32_t i = 0; i < count; i++)
        if (value_offsets[i + 1] < value_offsets[i]) return set_err(c, RBF_ERR_INVALID, "value offsets decrease at pair %u", i);
    bool any_motion = false;
    for (uint32_t i = 0; modes && i < count; i++) {
        if (modes[i] > 2) return set_err(c, RBF_ERR_INVALID, "pair %u: value mode %u is not 0, 1 or 2", i, (unsigned)modes[i]);
        any_motion |= modes[i] == 2;
    }
    const size_t field_bytes = modes && fields ? (size_t)count * mv_blocks(s->H, s->W) * 2 : 0;
    if (any_motion && !fields) return set_err(c, RBF_ERR_INVALID, "rbf_stream_apply_chain: motion pairs without fields");
    for (size_t i = 0; i < field_bytes; i++)
        if (fields[i] < -MV_RANGE || fields[i] > MV_RANGE)
            return set_err(c, RBF_ERR_INVALID, "pair %llu: motion vector component %d is outside [-%d, %d]",
                           (unsigned long long)(i / (field_bytes / count)), (int)fields[i], MV_RANGE, MV_RANGE);
    CK(c, cudaSetDevice(c->device));
    void* d_vals = s->d_inflated;
    if (values || !vbytes) {                             // else the values are where rbf_stream_inflate_values left them
        if (int r = scratch_get(c, kScrValues, (size_t)vbytes + 256, &d_vals)) return r;
        if (vbytes) { CK(c, cudaMemcpyAsync(d_vals, values, (size_t)vbytes, cudaMemcpyHostToDevice, c->st)); c->h2d += (int64_t)vbytes; }
    }
    return stream_apply_chain(s, base_frame, count, (const uint8_t*)d_vals, value_offsets, modes, fields, field_bytes, s->d_mask,
                              s->mask_stride_w, applied_out, nullptr);
}

// The one-pair chain from base_frame into frame (base_frame + 1) % max_frames, with the mask and values from the host
extern "C" int rbf_stream_apply_diff(rbf_stream* s, uint32_t base_frame, const uint8_t* mask_packed_little, const uint8_t* values,
                                     uint64_t values_bytes, uint64_t* applied_pixels) {
    if (!s || !mask_packed_little || (!values && values_bytes)) return set_err(s ? s->c : nullptr, RBF_ERR_INVALID, "rbf_stream_apply_diff: NULL");
    rbf_ctx* c = s->c;
    if (base_frame >= s->max_frames) return set_err(c, RBF_ERR_INVALID, "frame index outside the store");
    CK(c, cudaSetDevice(c->device));
    const size_t mbytes = (size_t)((s->npix + 7) / 8), mwords = s->mask_stride_w;
    void *d_mask, *d_vals;
    int rc;
    if ((rc = scratch_get(c, kScrApplyMask, mwords * 4, &d_mask)) || (rc = scratch_get(c, kScrValues, (size_t)values_bytes + 256, &d_vals)))
        return rc;
    CK(c, cudaMemsetAsync(d_mask, 0, mwords * 4, c->st));
    CK(c, cudaMemcpyAsync(d_mask, mask_packed_little, mbytes, cudaMemcpyHostToDevice, c->st)); c->h2d += (int64_t)mbytes;
    if (values_bytes) { CK(c, cudaMemcpyAsync(d_vals, values, (size_t)values_bytes, cudaMemcpyHostToDevice, c->st)); c->h2d += (int64_t)values_bytes; }
    const uint64_t offs[2] = {0, values_bytes};
    uint64_t applied = 0;
    uint32_t first_bad = 0;
    if (int r = stream_apply_chain(s, base_frame, 1, (const uint8_t*)d_vals, offs, nullptr, nullptr, 0, (const uint32_t*)d_mask, mwords,
                                   &applied, &first_bad))
        return r;
    if (first_bad == 0) {                                // ivc:882: the sweep wrote nothing; the output is the base frame unchanged
        const uint32_t out = base_frame + 1 == s->max_frames ? 0 : base_frame + 1;
        CK(c, cudaMemcpyAsync(s->d_frames + (size_t)out * s->frame_stride, s->d_frames + (size_t)base_frame * s->frame_stride,
                              s->frame_bytes, cudaMemcpyDeviceToDevice, c->st));
        CK(c, cudaStreamSynchronize(c->st));
    }
    if (applied_pixels) *applied_pixels = applied;
    return RBF_OK;
}

// ------------------------------------------------------------------------------------------
// Block motion search of the encoded pairs (value_coding "motion"); the fields stay in the stream for the motion_values gathers
// ------------------------------------------------------------------------------------------
extern "C" int rbf_stream_motion_search(rbf_stream* s, uint32_t pairs, int8_t* fields_out) {
    if (!s || !fields_out) return set_err(s ? s->c : nullptr, RBF_ERR_INVALID, "rbf_stream_motion_search: NULL");
    rbf_ctx* c = s->c;
    if (pairs == 0 || pairs > s->last_pairs) return set_err(c, RBF_ERR_INVALID, "only %u pairs were encoded", s->last_pairs);
    CK(c, cudaSetDevice(c->device));
    const size_t field_bytes = (size_t)mv_blocks(s->H, s->W) * 2;
    if (!s->d_fields) CK(c, cudaMalloc((void**)&s->d_fields, field_bytes * s->max_pairs));
    // the PairJobs of the last encode are still on the device (d_pairs)
    CK(c, launch_motion_search(c->L, s->d_pairs, (int)pairs, s->H, s->W, s->C * s->S, s->S, s->d_fields, c->st));
    CK(c, cudaMemcpyAsync(fields_out, s->d_fields, field_bytes * pairs, cudaMemcpyDeviceToHost, c->st));
    c->d2h += (int64_t)(field_bytes * pairs);
    CK(c, cudaStreamSynchronize(c->st));
    s->motion_pairs = pairs;
    return RBF_OK;
}

extern "C" int rbf_stream_download_batch(rbf_stream* s, uint32_t first, uint32_t count, void* host_out) {
    if (!s || !host_out || first >= s->max_frames || count == 0 || count > s->max_frames)
        return set_err(s ? s->c : nullptr, RBF_ERR_INVALID, "rbf_stream_download_batch: bad argument");
    rbf_ctx* c = s->c;
    const uint32_t head = count < s->max_frames - first ? count : s->max_frames - first;   // slots wrap as in rbf_stream_apply_chain
    CK(c, cudaMemcpy2DAsync(host_out, s->frame_bytes, s->d_frames + (size_t)first * s->frame_stride, s->frame_stride, s->frame_bytes,
                            head, cudaMemcpyDeviceToHost, c->st));
    if (head < count)
        CK(c, cudaMemcpy2DAsync((uint8_t*)host_out + (size_t)head * s->frame_bytes, s->frame_bytes, s->d_frames, s->frame_stride,
                                s->frame_bytes, count - head, cudaMemcpyDeviceToHost, c->st));
    c->d2h += (int64_t)s->frame_bytes * count;
    CK(c, cudaStreamSynchronize(c->st));
    return RBF_OK;
}

// rbf_stream_download_batch into device memory: the caller's pending work on wait_stream (its __cuda_array_interface__ stream) is
// ordered before the copy through an event, so a buffer still being written or read there is not overwritten early.
extern "C" int rbf_stream_copy_frames(rbf_stream* s, uint32_t first, uint32_t count, void* dst_device, uint64_t dst_capacity,
                                      uint64_t wait_stream) {
    if (!s) return set_err(nullptr, RBF_ERR_INVALID, "rbf_stream_copy_frames: stream is NULL");
    rbf_ctx* c = s->c;
    if (first >= s->max_frames || count == 0 || count > s->max_frames)
        return set_err(c, RBF_ERR_INVALID, "rbf_stream_copy_frames: frames %u + %u of a store of %u", first, count, s->max_frames);
    const uint64_t bytes = s->frame_bytes * count;
    if (!dst_device || dst_capacity < bytes)
        return set_err(c, RBF_ERR_INVALID, "rbf_stream_copy_frames: %llu bytes into a buffer of %llu", (unsigned long long)bytes,
                       dst_device ? (unsigned long long)dst_capacity : 0ULL);
    CK(c, cudaSetDevice(c->device));
    cudaPointerAttributes pa;
    cudaError_t e = cudaPointerGetAttributes(&pa, dst_device);
    if (e != cudaSuccess) cudaGetLastError();                    // not a pointer the runtime knows: refused below
    if (e != cudaSuccess || !(pa.type == cudaMemoryTypeDevice || pa.type == cudaMemoryTypeManaged) || pa.device != c->device)
        return set_err(c, RBF_ERR_INVALID, "rbf_stream_copy_frames: dst is not device or managed memory of device %d", c->device);
    if (wait_stream) {
        cudaStream_t ws = wait_stream == 1 ? cudaStreamLegacy : wait_stream == 2 ? cudaStreamPerThread : (cudaStream_t)(uintptr_t)wait_stream;
        if (!c->ev_wait) CK(c, cudaEventCreateWithFlags(&c->ev_wait, cudaEventDisableTiming));
        CK(c, cudaEventRecord(c->ev_wait, ws));
        CK(c, cudaStreamWaitEvent(c->st, c->ev_wait, 0));
    }
    const uint32_t head = count < s->max_frames - first ? count : s->max_frames - first;   // slots wrap as in rbf_stream_apply_chain
    CK(c, cudaMemcpy2DAsync(dst_device, s->frame_bytes, s->d_frames + (size_t)first * s->frame_stride, s->frame_stride, s->frame_bytes,
                            head, cudaMemcpyDeviceToDevice, c->st));
    if (head < count)
        CK(c, cudaMemcpy2DAsync((uint8_t*)dst_device + (size_t)head * s->frame_bytes, s->frame_bytes, s->d_frames, s->frame_stride,
                                s->frame_bytes, count - head, cudaMemcpyDeviceToDevice, c->st));
    c->d2d += (int64_t)bytes;
    CK(c, cudaStreamSynchronize(c->st));
    return RBF_OK;
}


// ------------------------------------------------------------------------------------------
// N3: cv2.medianBlur(frame, 5) of VideoFrameCompressor._estimate_noise_level (ivc:738)
// ------------------------------------------------------------------------------------------
extern "C" int rbf_median_blur5(rbf_ctx* c, const void* plane_in, uint32_t H, uint32_t W, uint32_t sample_bytes, void* plane_out) {
    if (!c || !plane_in || !plane_out) return set_err(c, RBF_ERR_INVALID, "rbf_median_blur5: NULL");
    if (!(sample_bytes == 1 || sample_bytes == 2) || H == 0 || W == 0) return set_err(c, RBF_ERR_INVALID, "rbf_median_blur5: bad shape");
    CK(c, cudaSetDevice(c->device));
    const size_t bytes = (size_t)H * W * sample_bytes;
    void *d_in, *d_out;
    int rc;
    if ((rc = scratch_get(c, kScrMedianIn, bytes, &d_in)) || (rc = scratch_get(c, kScrMedianOut, bytes, &d_out))) return rc;
    CK(c, cudaMemcpyAsync(d_in, plane_in, bytes, cudaMemcpyHostToDevice, c->st)); c->h2d += (int64_t)bytes;
    CK(c, launch_median5(c->L, d_in, H, W, (int)sample_bytes, d_out, c->st));
    CK(c, cudaMemcpyAsync(plane_out, d_out, bytes, cudaMemcpyDeviceToHost, c->st)); c->d2h += (int64_t)bytes;
    CK(c, cudaStreamSynchronize(c->st));
    return RBF_OK;
}

// ------------------------------------------------------------------------------------------
// N4: zlib streams coded on the device (layout: rbf_deflate.cuh)
// ------------------------------------------------------------------------------------------
extern "C" uint64_t rbf_zlib_bound(uint64_t n) {
    if (n == 0) return 8;
    const uint64_t full = (n - 1) / kDeflateSeg, last = n - full * kDeflateSeg;
    return 2 + full * deflate_seg_bound(kDeflateSeg) + deflate_seg_bound((uint32_t)last) + 6;
}

extern "C" int rbf_deflate_code_lengths(const uint32_t* freqs, uint32_t nsym, uint32_t max_bits, uint8_t* lengths) {
    if (!freqs || !lengths) return set_err(nullptr, RBF_ERR_INVALID, "rbf_deflate_code_lengths: NULL");
    if (deflate_code_lengths_host(freqs, nsym, max_bits, lengths))
        return set_err(nullptr, RBF_ERR_INVALID, "rbf_deflate_code_lengths: nsym %u / max_bits %u not codable", nsym, max_bits);
    return RBF_OK;
}

// Segments are coded in waves of at most 2 per SM, so scratch is bounded whatever the input size; each wave's streams are
// joined on the device and copied to out_host with one copy.
static int zlib_batch(rbf_ctx* c, uint32_t count, const void* const* srcs, const uint64_t* lens, bool on_device, uint8_t* out_host,
                      uint64_t capacity, uint64_t* offsets) {
    CK(c, cudaSetDevice(c->device));
    offsets[0] = 0;
    if (count == 0) return RBF_OK;
    for (uint32_t b = 0; b < count; b++)
        if (lens[b] && !srcs[b]) return set_err(c, RBF_ERR_INVALID, "zlib: buffer %u is NULL", b);
    const uint32_t W = 2u * (uint32_t)(c->L.sm_count > 0 ? c->L.sm_count : 1);
    const size_t region = align_up(deflate_seg_bound(kDeflateSeg), 16), stage_cap = (size_t)W * (region + 8);
    void *d_in = nullptr, *d_res, *d_out, *d_stage, *d_segs, *d_copies, *d_small;
    int rc;
    if ((rc = scratch_get(c, kScrZlibRes, (size_t)W * kDeflateSeg * 4, &d_res)) || (rc = scratch_get(c, kScrZlibOut, (size_t)W * region, &d_out)) ||
        (rc = scratch_get(c, kScrZlibStage, stage_cap, &d_stage)) || (rc = scratch_get(c, kScrZlibSegs, (size_t)W * sizeof(DeflateSeg), &d_segs)) ||
        (rc = scratch_get(c, kScrZlibCopies, (size_t)W * sizeof(DeflateCopy), &d_copies)) ||
        (rc = scratch_get(c, kScrZlibSmall, (size_t)W * 12 + 64, &d_small)) ||
        (!on_device && (rc = scratch_get(c, kScrZlibIn, (size_t)W * kDeflateSeg, &d_in))))
        return rc;
    uint32_t* d_sizes = (uint32_t*)d_small;
    uint32_t* d_adler = d_sizes + W;
    uint32_t* d_err = d_adler + 2 * W;
    struct Ref { uint32_t buf; uint64_t off; uint32_t len; bool first, last; };
    std::vector<Ref> refs;
    std::vector<DeflateSeg> segs;
    std::vector<DeflateCopy> copies;
    std::vector<uint32_t> h_small(3 * (size_t)W + 1);
    uint32_t b = 0;
    uint64_t k = 0, pos = 0;
    uint32_t s1 = 1, s2 = 0;                                              // Adler-32 of the buffer being written
    while (b < count) {
        refs.clear(); segs.clear(); copies.clear();
        while (refs.size() < W && b < count) {
            const uint64_t nseg = lens[b] ? (lens[b] + kDeflateSeg - 1) / kDeflateSeg : 1, off = k * kDeflateSeg;
            const uint64_t left = lens[b] - (lens[b] ? off : 0);
            refs.push_back({b, off, (uint32_t)(left < kDeflateSeg ? left : kDeflateSeg), k == 0, k + 1 == nseg});
            if (++k == nseg) { b++; k = 0; }
        }
        const uint32_t n = (uint32_t)refs.size();
        for (uint32_t i = 0; i < n; i++) {
            const Ref& r = refs[i];
            DeflateSeg sg;
            sg.src = on_device ? (const uint8_t*)srcs[r.buf] + r.off : (const uint8_t*)d_in + (size_t)i * kDeflateSeg;
            sg.out = (uint8_t*)d_out + (size_t)i * region;
            sg.len = r.len;
            sg.cap = (uint32_t)region;
            segs.push_back(sg);
            if (!on_device && r.len && (i == 0 || refs[i - 1].buf != r.buf)) {   // the wave's part of one buffer is contiguous
                uint64_t bytes = 0;
                for (uint32_t j = i; j < n && refs[j].buf == r.buf; j++) bytes += refs[j].len;
                CK(c, cudaMemcpyAsync((uint8_t*)d_in + (size_t)i * kDeflateSeg, (const uint8_t*)srcs[r.buf] + r.off, bytes,
                                      cudaMemcpyHostToDevice, c->st));
                c->h2d += (int64_t)bytes;
            }
        }
        CK(c, cudaMemsetAsync(d_err, 0, 4, c->st));
        CK(c, cudaMemcpyAsync(d_segs, segs.data(), sizeof(DeflateSeg) * n, cudaMemcpyHostToDevice, c->st));
        CK(c, launch_deflate_segments(c->L, (const DeflateSeg*)d_segs, (int)n, (uint32_t*)d_res, d_sizes, d_adler, d_err, c->st));
        CK(c, cudaMemcpyAsync(h_small.data(), d_small, (3 * (size_t)W + 1) * 4, cudaMemcpyDeviceToHost, c->st));
        CK(c, cudaStreamSynchronize(c->st));
        if (h_small[3 * (size_t)W]) return set_err(c, RBF_ERR_STATE, "zlib: a coded segment overran its region (flags %u)", h_small[3 * (size_t)W]);
        const uint64_t wave_start = pos;
        for (uint32_t i = 0; i < n; i++) {
            const Ref& r = refs[i];
            const uint32_t size = h_small[i];
            if (r.first) { offsets[r.buf] = pos; pos += 2; s1 = 1; s2 = 0; }
            adler_combine(s1, s2, r.len, h_small[W + 2 * i], h_small[W + 2 * i + 1]);
            DeflateCopy cp;
            cp.src = (const uint8_t*)d_out + (size_t)i * region;
            cp.dst = pos - wave_start;
            cp.len = size;
            cp.flags = (r.first ? 1u : 0u) | (r.last ? 2u : 0u);
            cp.adler = (s2 << 16) | s1;
            cp.pad = 0;
            copies.push_back(cp);
            pos += size;
            if (r.last) { pos += 6; offsets[r.buf + 1] = pos; }
        }
        if (pos > capacity)
            return set_err(c, RBF_ERR_INVALID, "zlib: output buffer too small (%llu < %llu so far)", (unsigned long long)capacity,
                           (unsigned long long)pos);
        CK(c, cudaMemcpyAsync(d_copies, copies.data(), sizeof(DeflateCopy) * n, cudaMemcpyHostToDevice, c->st));
        CK(c, launch_deflate_concat(c->L, (const DeflateCopy*)d_copies, (int)n, (uint8_t*)d_stage, stage_cap, d_err, c->st));
        CK(c, cudaMemcpyAsync(out_host + wave_start, d_stage, (size_t)(pos - wave_start), cudaMemcpyDeviceToHost, c->st));
        CK(c, cudaMemcpyAsync(h_small.data() + 3 * (size_t)W, d_err, 4, cudaMemcpyDeviceToHost, c->st));
        c->d2h += (int64_t)(pos - wave_start);
        CK(c, cudaStreamSynchronize(c->st));
        if (h_small[3 * (size_t)W]) return set_err(c, RBF_ERR_STATE, "zlib: joined streams overran the staging buffer");
    }
    return RBF_OK;
}

extern "C" int rbf_zlib_compress_batch(rbf_ctx* c, uint32_t count, const void* const* srcs, const uint64_t* lens, int srcs_on_device,
                                       uint8_t* out_host, uint64_t out_capacity, uint64_t* out_offsets) {
    if (!c || !out_offsets || (count && (!srcs || !lens || !out_host))) return set_err(c, RBF_ERR_INVALID, "rbf_zlib_compress_batch: NULL");
    return zlib_batch(c, count, srcs, lens, srcs_on_device != 0, out_host, out_capacity, out_offsets);
}

extern "C" int rbf_stream_zlib_changed(rbf_stream* s, uint32_t pairs, uint8_t* out_host, uint64_t out_capacity, uint64_t* out_offsets) {
    if (!s || !out_host || !out_offsets) return set_err(s ? s->c : nullptr, RBF_ERR_INVALID, "rbf_stream_zlib_changed: NULL");
    rbf_ctx* c = s->c;
    if (pairs == 0 || pairs > s->last_pairs) return set_err(c, RBF_ERR_INVALID, "only %u pairs were encoded", s->last_pairs);
    CK(c, cudaSetDevice(c->device));
    std::vector<uint64_t> voff(pairs + 1);
    changed_offsets(s, pairs, voff.data());
    uint8_t* d_vals;
    if (int r = gather_values(s, pairs, voff.data(), &d_vals)) return r;
    std::vector<const void*> srcs(pairs);
    std::vector<uint64_t> lens(pairs);
    for (uint32_t i = 0; i < pairs; i++) { srcs[i] = d_vals + voff[i]; lens[i] = voff[i + 1] - voff[i]; }
    return zlib_batch(c, pairs, srcs.data(), lens.data(), true, out_host, out_capacity, out_offsets);   // same stream: after the gather
}

// ------------------------------------------------------------------------------------------
// inflate of the streams the device coder writes (rbf_inflate.cuh)
// ------------------------------------------------------------------------------------------
extern "C" int rbf_inflate_segment(const uint8_t* in, uint64_t avail, uint8_t* out, uint32_t* status, uint64_t* consumed,
                                   uint32_t* produced, uint32_t* s1, uint32_t* s2) {
    if ((!in && avail) || !out || !status || !consumed || !produced || !s1 || !s2)
        return set_err(nullptr, RBF_ERR_INVALID, "rbf_inflate_segment: NULL");
    InflateSegResult r;
    inflate_segment_host(in, avail, out, &r);
    *status = r.status; *consumed = r.consumed; *produced = r.produced; *s1 = r.adler & 0xffffu; *s2 = r.adler >> 16;
    return RBF_OK;
}

// What inflate_streams leaves for inflate_place: per stream, its segments' slots in order and its inflated length; ok[i] == 0
// for a stream the device declined (not in the layout, a segment refused on the chain, a bad trailer, more candidates than its
// bound allows, or more output than its bound)
struct InflateRun {
    std::vector<std::vector<uint32_t>> chain;
    std::vector<uint32_t> produced;     // per slot
    std::vector<uint64_t> full;
    std::vector<uint8_t> ok;
    uint8_t* d_slots = nullptr;
};

// Host streams in: one H2D copy of each stream's bytes, k_inflate_scan, one sync for the candidate counts, k_inflate_segments
// over every candidate, one sync for the results, and the chains resolved here.
static int inflate_streams(rbf_ctx* c, uint32_t count, const void* const* srcs, const uint64_t* lens, const uint64_t* bounds,
                           InflateRun& R) {
    R.chain.assign(count, {}); R.full.assign(count, 0); R.ok.assign(count, 0); R.produced.clear();
    std::vector<uint64_t> base(count, 0), cand0(count, 0), cap(count, 0);
    std::vector<InflateScanJob> jobs;
    uint64_t in_bytes = 0, ncand = 0;
    for (uint32_t i = 0; i < count; i++) {
        const uint8_t* p = (const uint8_t*)srcs[i];
        if (!p || lens[i] < 8 || lens[i] > 0xfffffff0ull || p[0] != 0x78 || p[1] != 0x9c) continue;
        const uint64_t by_bound = 2 * ((bounds[i] + kDeflateSeg - 1) / kDeflateSeg) + 8, by_len = lens[i] / 4 + 2;
        cap[i] = by_bound < by_len ? by_bound : by_len;                // no more starts than 00 00 FF FF fits in the stream
        base[i] = in_bytes; cand0[i] = ncand;
        in_bytes += align_up(lens[i], 16); ncand += cap[i];
        for (uint64_t q = 2; q < lens[i] - 6; q += kInflateScanChunk) {   // starts below the 6-byte trailer
            const uint64_t e = q + kInflateScanChunk < lens[i] - 6 ? q + kInflateScanChunk : lens[i] - 6;
            InflateScanJob J;
            J.base = base[i]; J.begin = (uint32_t)q; J.end = (uint32_t)e; J.stream = i; J.cand0 = (uint32_t)cand0[i]; J.cap = (uint32_t)cap[i]; J.pad = 0;
            jobs.push_back(J);
        }
        R.ok[i] = 1;
    }
    if (ncand > 0xffffffffull) return set_err(c, RBF_ERR_INVALID, "zlib inflate: %llu candidate starts in one call", (unsigned long long)ncand);
    if (in_bytes == 0) return RBF_OK;
    // small: counts[count] | cand[ncand] | start[ncand] | slot_stream[ncand] | streams[count] | jobs | err
    const size_t o_cand = align_up(4 * (size_t)count, 16), o_start = align_up(o_cand + 4 * ncand, 16);
    const size_t o_ss = align_up(o_start + 4 * ncand, 16), o_st = align_up(o_ss + 4 * ncand, 16);
    const size_t o_jobs = align_up(o_st + sizeof(InflateStream) * count, 16), o_err = align_up(o_jobs + sizeof(InflateScanJob) * jobs.size(), 16);
    void *d_in, *d_small;
    int rc;
    if ((rc = scratch_get(c, kScrInflateIn, in_bytes, &d_in)) || (rc = scratch_get(c, kScrInflateSmall, o_err + 16, &d_small))) return rc;
    uint8_t* sm = (uint8_t*)d_small;
    uint32_t* d_counts = (uint32_t*)sm;
    for (uint32_t i = 0; i < count; i++)
        if (R.ok[i]) { CK(c, cudaMemcpyAsync((uint8_t*)d_in + base[i], srcs[i], lens[i], cudaMemcpyHostToDevice, c->st)); c->h2d += (int64_t)lens[i]; }
    CK(c, cudaMemsetAsync(d_counts, 0, 4 * (size_t)count, c->st));
    CK(c, cudaMemcpyAsync(sm + o_jobs, jobs.data(), sizeof(InflateScanJob) * jobs.size(), cudaMemcpyHostToDevice, c->st));
    CK(c, launch_inflate_scan(c->L, (const InflateScanJob*)(sm + o_jobs), (int)jobs.size(), (const uint8_t*)d_in, d_counts,
                              (uint32_t*)(sm + o_cand), c->st));
    std::vector<uint32_t> counts(count);
    CK(c, cudaMemcpyAsync(counts.data(), d_counts, 4 * (size_t)count, cudaMemcpyDeviceToHost, c->st));
    c->d2h += 4 * (int64_t)count;
    CK(c, cudaStreamSynchronize(c->st));
    std::vector<InflateStream> streams(count);
    std::vector<uint32_t> slot_stream;
    for (uint32_t i = 0; i < count; i++) {
        if (!R.ok[i]) continue;
        if (counts[i] > cap[i]) { R.ok[i] = 0; continue; }
        streams[i].base = base[i]; streams[i].len = lens[i]; streams[i].cand0 = (uint32_t)cand0[i]; streams[i].slot0 = (uint32_t)slot_stream.size();
        slot_stream.insert(slot_stream.end(), counts[i], i);
    }
    const uint32_t nslots = (uint32_t)slot_stream.size();
    std::vector<InflateSegResult> res(nslots);
    std::vector<uint32_t> start(nslots);
    if (nslots) {
        void *d_slots, *d_res;
        if ((rc = scratch_get(c, kScrInflateSlots, (size_t)nslots * kDeflateSeg, &d_slots)) ||
            (rc = scratch_get(c, kScrInflateRes, sizeof(InflateSegResult) * (size_t)nslots, &d_res)))
            return rc;
        R.d_slots = (uint8_t*)d_slots;
        CK(c, cudaMemcpyAsync(sm + o_ss, slot_stream.data(), 4 * (size_t)nslots, cudaMemcpyHostToDevice, c->st));
        CK(c, cudaMemcpyAsync(sm + o_st, streams.data(), sizeof(InflateStream) * count, cudaMemcpyHostToDevice, c->st));
        CK(c, launch_inflate_segments(c->L, (const uint32_t*)(sm + o_ss), (const InflateStream*)(sm + o_st), (int)nslots,
                                      (const uint8_t*)d_in, (const uint32_t*)(sm + o_cand), R.d_slots, (InflateSegResult*)d_res,
                                      (uint32_t*)(sm + o_start), c->st));
        CK(c, cudaMemcpyAsync(res.data(), d_res, sizeof(InflateSegResult) * (size_t)nslots, cudaMemcpyDeviceToHost, c->st));
        CK(c, cudaMemcpyAsync(start.data(), sm + o_start, 4 * (size_t)nslots, cudaMemcpyDeviceToHost, c->st));
        c->d2h += (int64_t)(sizeof(InflateSegResult) + 4) * nslots;
        CK(c, cudaStreamSynchronize(c->st));
    }
    R.produced.resize(nslots);
    for (uint32_t k = 0; k < nslots; k++) R.produced[k] = res[k].produced;
    // the chains: from offset 2 through each accepted segment's end, every segment but the last 64 KiB of output, to the trailer
    std::vector<std::pair<uint32_t, uint32_t>> at;                     // (start, slot) of one stream, sorted
    for (uint32_t i = 0; i < count; i++) {
        if (!R.ok[i]) continue;
        const uint8_t* p = (const uint8_t*)srcs[i];
        const uint64_t end = lens[i] - 6;
        at.clear();
        for (uint32_t k = streams[i].slot0; k < streams[i].slot0 + counts[i]; k++) at.push_back({start[k], k});
        std::sort(at.begin(), at.end());
        uint64_t pos = 2, total = 0;
        uint32_t s1 = 1, s2 = 0;
        bool good = true;
        std::vector<uint32_t>& chain = R.chain[i];
        while (good && pos < end) {
            auto it = std::lower_bound(at.begin(), at.end(), std::make_pair((uint32_t)pos, 0u));
            good = it != at.end() && it->first == pos && res[it->second].status == kInflateOk &&
                   (chain.empty() || res[chain.back()].produced == kDeflateSeg);
            if (!good) break;
            const InflateSegResult& r = res[it->second];
            adler_combine(s1, s2, r.produced, r.adler & 0xffffu, r.adler >> 16);
            total += r.produced;
            pos += r.consumed;
            chain.push_back(it->second);
        }
        const uint32_t trailer = (uint32_t)p[end + 2] << 24 | (uint32_t)p[end + 3] << 16 | (uint32_t)p[end + 4] << 8 | p[end + 5];
        good = good && pos == end && p[end] == 0x03 && p[end + 1] == 0x00 && trailer == (s2 << 16 | s1) && total <= bounds[i];
        if (!good) { R.ok[i] = 0; chain.clear(); continue; }
        R.full[i] = total;
    }
    return RBF_OK;
}

// Copies each accepted stream's segments from their slots to d_dst + dst_off[i] (k_deflate_concat without header or trailer)
static int inflate_place(rbf_ctx* c, const InflateRun& R, const uint64_t* dst_off, uint8_t* d_dst, uint64_t cap) {
    std::vector<DeflateCopy> copies;
    for (size_t i = 0; i < R.chain.size(); i++) {
        uint64_t o = dst_off[i];
        for (uint32_t k : R.chain[i]) {
            DeflateCopy cp;
            cp.src = R.d_slots + (size_t)k * kDeflateSeg; cp.dst = o; cp.len = R.produced[k]; cp.flags = cp.adler = cp.pad = 0;
            copies.push_back(cp);
            o += R.produced[k];
        }
    }
    if (copies.empty()) return RBF_OK;
    void* d_jobs;
    if (int rc = scratch_get(c, kScrInflateRes, sizeof(DeflateCopy) * copies.size() + 16, &d_jobs)) return rc;   // the results are read
    uint32_t* d_err = (uint32_t*)((uint8_t*)d_jobs + sizeof(DeflateCopy) * copies.size());
    CK(c, cudaMemsetAsync(d_err, 0, 4, c->st));
    CK(c, cudaMemcpyAsync(d_jobs, copies.data(), sizeof(DeflateCopy) * copies.size(), cudaMemcpyHostToDevice, c->st));
    CK(c, launch_deflate_concat(c->L, (const DeflateCopy*)d_jobs, (int)copies.size(), d_dst, cap, d_err, c->st));
    uint32_t err = 0;
    CK(c, cudaMemcpyAsync(&err, d_err, 4, cudaMemcpyDeviceToHost, c->st));
    c->d2h += 4;
    CK(c, cudaStreamSynchronize(c->st));
    if (err) return set_err(c, RBF_ERR_STATE, "zlib inflate: a placed segment overran the output");
    return RBF_OK;
}

extern "C" int rbf_zlib_decompress_batch(rbf_ctx* c, uint32_t count, const void* const* srcs, const uint64_t* lens, const uint64_t* bounds,
                                         uint8_t* out_host, uint64_t out_capacity, uint64_t* out_offsets, uint8_t* on_device) {
    if (!c || !out_offsets || (count && (!srcs || !lens || !bounds || !on_device)))
        return set_err(c, RBF_ERR_INVALID, "rbf_zlib_decompress_batch: NULL");
    CK(c, cudaSetDevice(c->device));
    InflateRun R;
    if (int rc = inflate_streams(c, count, srcs, lens, bounds, R)) return rc;
    out_offsets[0] = 0;
    for (uint32_t i = 0; i < count; i++) {
        if (R.ok[i] && R.full[i] > out_capacity - out_offsets[i]) { R.ok[i] = 0; R.full[i] = 0; R.chain[i].clear(); }   // does not fit
        on_device[i] = R.ok[i];
        out_offsets[i + 1] = out_offsets[i] + R.full[i];
    }
    const uint64_t total = out_offsets[count];
    if (total == 0) return RBF_OK;
    if (!out_host) return set_err(c, RBF_ERR_INVALID, "rbf_zlib_decompress_batch: out_host is NULL");
    void* d_out;
    if (int rc = scratch_get(c, kScrInflateOut, total, &d_out)) return rc;
    if (int rc = inflate_place(c, R, out_offsets, (uint8_t*)d_out, total)) return rc;
    CK(c, cudaMemcpyAsync(out_host, d_out, total, cudaMemcpyDeviceToHost, c->st));
    c->d2h += (int64_t)total;
    CK(c, cudaStreamSynchronize(c->st));
    return RBF_OK;
}

extern "C" int rbf_stream_inflate_values(rbf_stream* s, uint32_t count, const void* const* srcs, const uint64_t* lens,
                                         const uint64_t* bounds, uint64_t* out_lens, uint8_t* on_device) {
    if (!s || (count && (!srcs || !lens || !bounds || !out_lens || !on_device)))
        return set_err(s ? s->c : nullptr, RBF_ERR_INVALID, "rbf_stream_inflate_values: NULL");
    rbf_ctx* c = s->c;
    CK(c, cudaSetDevice(c->device));
    s->inflated_bytes = 0;
    InflateRun R;
    if (int rc = inflate_streams(c, count, srcs, lens, bounds, R)) return rc;
    std::vector<uint64_t> off(count + 1, 0);
    for (uint32_t i = 0; i < count; i++) { on_device[i] = R.ok[i]; out_lens[i] = R.full[i]; off[i + 1] = off[i] + R.full[i]; }
    const uint64_t total = off[count];
    if (total + 256 > s->inflated_cap) {
        if (s->d_inflated) CK(c, cudaFree(s->d_inflated));
        s->d_inflated = nullptr; s->inflated_cap = 0;
        const size_t nb = align_up((size_t)total + (total >> 2) + 256, 256);
        CK(c, cudaMalloc((void**)&s->d_inflated, nb));
        s->inflated_cap = nb;
    }
    if (int rc = inflate_place(c, R, off.data(), s->d_inflated, total)) return rc;
    s->inflated_bytes = total;
    return RBF_OK;
}

// ------------------------------------------------------------------------------------------
// NCCL (dlopen'ed so that single-GPU use needs no NCCL at all)
// ------------------------------------------------------------------------------------------
typedef struct { char internal[128]; } nccl_uid;
typedef int (*fn_GetUniqueId)(nccl_uid*);
typedef int (*fn_CommInitRank)(void**, int, nccl_uid, int);
typedef int (*fn_AllGather)(const void*, void*, size_t, int, void*, cudaStream_t);
typedef int (*fn_CommDestroy)(void*);
typedef const char* (*fn_GetErrorString)(int);

static void* g_nccl = nullptr;
static void* nccl_handle() {
    if (!g_nccl) {
        g_nccl = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!g_nccl) g_nccl = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    }
    return g_nccl;
}
extern "C" int rbf_nccl_unique_id(uint8_t id_out[128]) {
    void* h = nccl_handle();
    if (!h) return set_err(nullptr, RBF_ERR_NCCL, "cannot dlopen libnccl.so.2: %s", dlerror());
    fn_GetUniqueId f = (fn_GetUniqueId)dlsym(h, "ncclGetUniqueId");
    if (!f) return set_err(nullptr, RBF_ERR_NCCL, "ncclGetUniqueId not found");
    nccl_uid u;
    int r = f(&u);
    if (r) return set_err(nullptr, RBF_ERR_NCCL, "ncclGetUniqueId failed: %d", r);
    memcpy(id_out, u.internal, 128);
    return RBF_OK;
}
extern "C" int rbf_nccl_init(rbf_ctx* c, const uint8_t id[128], int rank, int nranks) {
    if (!c || !id) return set_err(c, RBF_ERR_INVALID, "rbf_nccl_init: NULL");
    void* h = nccl_handle();
    if (!h) return set_err(c, RBF_ERR_NCCL, "cannot dlopen libnccl.so.2: %s", dlerror());
    fn_CommInitRank f = (fn_CommInitRank)dlsym(h, "ncclCommInitRank");
    if (!f) return set_err(c, RBF_ERR_NCCL, "ncclCommInitRank not found");
    CK(c, cudaSetDevice(c->device));
    nccl_uid u;
    memcpy(u.internal, id, 128);
    void* comm = nullptr;
    int r = f(&comm, nranks, u, rank);
    if (r) {
        fn_GetErrorString es = (fn_GetErrorString)dlsym(h, "ncclGetErrorString");
        return set_err(c, RBF_ERR_NCCL, "ncclCommInitRank failed: %s", es ? es(r) : "?");
    }
    c->nccl_lib = h; c->nccl_comm = comm; c->rank = rank; c->nranks = nranks;
    return RBF_OK;
}
// The caller has checked that c->nccl_comm is initialised.
static int nccl_allgather_on(rbf_ctx* c, const void* d_send, void* d_recv, uint64_t bytes_per_rank, cudaStream_t st) {
    fn_AllGather f = (fn_AllGather)dlsym(c->nccl_lib, "ncclAllGather");
    if (!f) return set_err(c, RBF_ERR_NCCL, "ncclAllGather not found");
    int r = f(d_send, d_recv, (size_t)bytes_per_rank, /*ncclUint8*/ 1, c->nccl_comm, st);
    if (r) {
        fn_GetErrorString es = (fn_GetErrorString)dlsym(c->nccl_lib, "ncclGetErrorString");
        return set_err(c, RBF_ERR_NCCL, "ncclAllGather failed: %s", es ? es(r) : "?");
    }
    c->L.launches++;
    return RBF_OK;
}
// Packs the bit arrays of the last encode into fixed-size slots and all-gathers them on the context's communication
// stream: the call returns once the work is enqueued, the next rbf_stream_encode overlaps it (it only waits for the
// packing before it clears the bit arrays).  d_recv is complete after rbf_sync, rbf_timer_stop_ms or rbf_memcpy_d2h.
static int ensure_comm_stream(rbf_ctx* c) {
    if (!c->st_comm) {
        CK(c, cudaStreamCreateWithFlags(&c->st_comm, cudaStreamNonBlocking));
        CK(c, cudaEventCreateWithFlags(&c->ev_enc, cudaEventDisableTiming));
        CK(c, cudaEventCreateWithFlags(&c->ev_pack, cudaEventDisableTiming));
        CK(c, cudaEventCreateWithFlags(&c->ev_comm, cudaEventDisableTiming));
    }
    return RBF_OK;
}
extern "C" int rbf_stream_allgather_bitmaps(rbf_stream* s, uint32_t pairs, uint64_t slot_bytes, void* d_send, void* d_recv) {
    if (!s || !d_recv) return set_err(s ? s->c : nullptr, RBF_ERR_INVALID, "rbf_stream_allgather_bitmaps: NULL");
    rbf_ctx* c = s->c;
    const size_t stride = s->mask_stride_w * 4;
    if (slot_bytes == 0 || slot_bytes > stride || (slot_bytes & 15) || pairs == 0 || pairs > s->max_pairs)
        return set_err(c, RBF_ERR_INVALID, "bad slot/pairs");
    if (c->peer_nranks > 0) {
        // peer-memory exchange: one kernel stores this rank's slots into every rank's receive buffer over NVLink
        if (d_recv != (void*)c->peer_recv[c->peer_rank]) return set_err(c, RBF_ERR_INVALID, "d_recv is not the buffer given to rbf_peer_gather_init");
        if (int r = ensure_comm_stream(c)) return r;
        CK(c, cudaEventRecord(c->ev_enc, c->st));                   // the encode that produced the bit arrays
        CK(c, cudaStreamWaitEvent(c->st_comm, c->ev_enc, 0));
        // every rank has signalled the previous exchange => it has consumed the one before it: that half is free everywhere
        if (c->peer_seq > 0)
            CK(c, launch_peer_wait(c->L, c->peer_flags[c->peer_rank], c->peer_nranks, c->peer_seq, kPeerTimeoutCycles, c->peer_err, c->st_comm));
        c->peer_seq++;
        const uint32_t slot_w = (uint32_t)(slot_bytes / 4);
        const size_t half_w = (size_t)c->peer_nranks * pairs * slot_w;
        const size_t dst_off_w = (size_t)(c->peer_seq & 1u) * half_w + (size_t)c->peer_rank * pairs * slot_w;
        CK(c, launch_push_slots(c->L, s->d_bits, s->mask_stride_w, slot_w, pairs, c->peer_recv, c->peer_flags, c->peer_nranks, c->peer_rank,
                                    dst_off_w, c->peer_seq, c->st_comm));
        CK(c, cudaEventRecord(c->ev_pack, c->st_comm));
        CK(c, cudaEventRecord(c->ev_comm, c->st_comm));
        c->pack_pending = c->comm_pending = c->peer_wait_pending = true;
        return RBF_OK;
    }
    if (!d_send) return set_err(c, RBF_ERR_INVALID, "rbf_stream_allgather_bitmaps: d_send is NULL");
    if (!c->nccl_comm) return set_err(c, RBF_ERR_STATE, "rbf_stream_allgather_bitmaps: communicator not initialised");
    if (int r = ensure_comm_stream(c)) return r;
    CK(c, cudaEventRecord(c->ev_enc, c->st));                       // the encode that produced the bit arrays
    CK(c, cudaStreamWaitEvent(c->st_comm, c->ev_enc, 0));
    CK(c, cudaMemcpy2DAsync(d_send, slot_bytes, s->d_bits, stride, slot_bytes, pairs, cudaMemcpyDeviceToDevice, c->st_comm));
    CK(c, cudaEventRecord(c->ev_pack, c->st_comm));
    c->pack_pending = true;
    if (int r = nccl_allgather_on(c, d_send, d_recv, slot_bytes * pairs, c->st_comm)) return r;
    CK(c, cudaEventRecord(c->ev_comm, c->st_comm));
    c->comm_pending = true;
    return RBF_OK;
}

// ------------------------------------------------------------------------------------------
// exchange over NVLink peer memory: CUDA IPC handles travel over the caller's channel (like the NCCL id)
// ------------------------------------------------------------------------------------------
extern "C" int rbf_peer_export(rbf_ctx* c, const void* d_ptr, uint8_t handle_out[64]) {
    if (!c || !d_ptr || !handle_out) return set_err(c, RBF_ERR_INVALID, "rbf_peer_export: NULL");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    CK(c, cudaSetDevice(c->device));
    cudaIpcMemHandle_t h;
    CK(c, cudaIpcGetMemHandle(&h, const_cast<void*>(d_ptr)));
    memcpy(handle_out, &h, 64);
    return RBF_OK;
}
extern "C" int rbf_peer_open(rbf_ctx* c, const uint8_t handle[64], void** d_out) {
    if (!c || !handle || !d_out) return set_err(c, RBF_ERR_INVALID, "rbf_peer_open: NULL");
    CK(c, cudaSetDevice(c->device));
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    CK(c, cudaIpcOpenMemHandle(d_out, h, cudaIpcMemLazyEnablePeerAccess));
    return RBF_OK;
}
extern "C" int rbf_peer_close(rbf_ctx* c, void* d_ptr) {
    if (!c) return RBF_ERR_INVALID;
    if (d_ptr) CK(c, cudaIpcCloseMemHandle(d_ptr));
    return RBF_OK;
}
extern "C" int rbf_peer_gather_init(rbf_ctx* c, int rank, int nranks, void* const* recv_ptrs, void* const* flag_ptrs) {
    if (!c || !recv_ptrs || !flag_ptrs) return set_err(c, RBF_ERR_INVALID, "rbf_peer_gather_init: NULL");
    if (nranks < 1 || nranks > 16 || rank < 0 || rank >= nranks) return set_err(c, RBF_ERR_INVALID, "rank %d of %d", rank, nranks);
    for (int r = 0; r < nranks; r++)
        if (!recv_ptrs[r] || !flag_ptrs[r]) return set_err(c, RBF_ERR_INVALID, "rbf_peer_gather_init: pointer of rank %d is NULL", r);
    CK(c, cudaSetDevice(c->device));
    if (!c->peer_err) {
        CK(c, cudaHostAlloc((void**)&c->peer_err, 64, cudaHostAllocMapped));
        *c->peer_err = 0;
    }
    for (int r = 0; r < 16; r++) {
        c->peer_recv[r] = r < nranks ? (uint32_t*)recv_ptrs[r] : nullptr;
        c->peer_flags[r] = r < nranks ? (uint32_t*)flag_ptrs[r] : nullptr;
    }
    c->peer_rank = rank; c->peer_nranks = nranks; c->peer_seq = 0; c->peer_wait_pending = false;
    return RBF_OK;
}
extern "C" int rbf_peer_gather_half(rbf_ctx* c, uint32_t* half_out) {
    if (!c || !half_out) return RBF_ERR_INVALID;
    if (c->peer_nranks == 0 || c->peer_seq == 0) return set_err(c, RBF_ERR_STATE, "no peer exchange has run");
    *half_out = c->peer_seq & 1u;
    return RBF_OK;
}
extern "C" int rbf_peer_gather_shutdown(rbf_ctx* c) {
    if (!c) return RBF_ERR_INVALID;
    if (c->st_comm) CK(c, cudaStreamSynchronize(c->st_comm));
    if (c->st) CK(c, cudaStreamSynchronize(c->st));
    c->peer_nranks = 0; c->peer_seq = 0; c->peer_wait_pending = false; c->comm_pending = c->pack_pending = false;
    return RBF_OK;
}
extern "C" int rbf_nccl_destroy(rbf_ctx* c) {
    if (!c) return RBF_ERR_INVALID;
    if (c->st_comm) cudaStreamSynchronize(c->st_comm);
    c->comm_pending = c->pack_pending = false;
    if (c->nccl_comm && c->nccl_lib) {
        fn_CommDestroy f = (fn_CommDestroy)dlsym(c->nccl_lib, "ncclCommDestroy");
        if (f) f(c->nccl_comm);
    }
    c->nccl_comm = nullptr;
    return RBF_OK;
}
