// sse_host.cu -- C ABI of libssegpu.so (include/sse_gpu.h): context, pinned staging, batch pipeline.
//
// One context per GPU. A batch slot owns pinned host staging + device buffers + a CUDA stream:
//   sse_submit:  H2D(segs, input)  ->  [wait: previous batch's kernel]  ->  kernel  ->  D2H(counters)  ->  record kernel_done
//   sse_poll:    query kernel_done (never blocks)
//   sse_collect: sync, then exact-size D2H of the result arrays, sync.
// Kernels of consecutive batches are ordered by an event because they share per-connection state
// (carry, finished flag) -- the per-connection FIFO of provider.go:307-340; H2D of batch k+1 and D2H of
// batch k overlap kernel k on their own streams.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <new>
#include <vector>
#include "sse_device.cuh"

static_assert(sizeof(sse_counters) == 8 + CN_COUNT * sizeof(uint64_t) && offsetof(sse_counters, p_segments) == 8 &&
              offsetof(sse_counters, d_items) == 8 + 8 * CN_D_ITEMS && offsetof(sse_counters, c_unquote) == 8 + 8 * CN_C_UNQUOTE,
              "sse_counters holds the counter block in CN_* order");

namespace {

thread_local char g_cuda_err[256] = "";

bool cu_ok(cudaError_t e, const char *what) {
    if (e == cudaSuccess) return true;
    snprintf(g_cuda_err, sizeof g_cuda_err, "%s: %s", what, cudaGetErrorString(e));
    return false;
}
#define CU(call) do { if (!cu_ok((call), #call)) return SSE_ERR_CUDA; } while (0)

enum SlotState { SLOT_FREE = 0, SLOT_ACQUIRED, SLOT_SUBMITTED, SLOT_COLLECTED };

struct Slot {
    int state = SLOT_FREE;
    cudaStream_t stream = nullptr;
    cudaEvent_t kernel_done = nullptr;
    // host (pinned)
    uint8_t *h_in = nullptr; sse_seg *h_segs = nullptr;
    uint8_t *h_out = nullptr; sse_frame *h_frames = nullptr; sse_rec *h_recs = nullptr; sse_tc *h_tcs = nullptr;
    sse_usage *h_usages = nullptr; uint8_t *h_text = nullptr; sse_run *h_runs = nullptr; sse_seg_result *h_segres = nullptr;
    Counters *h_ctr = nullptr;
    // device
    uint8_t *d_in = nullptr; sse_seg *d_segs = nullptr;
    uint8_t *d_out = nullptr; sse_frame *d_frames = nullptr; sse_rec *d_recs = nullptr; sse_tc *d_tcs = nullptr;
    sse_usage *d_usages = nullptr; uint8_t *d_text = nullptr; sse_run *d_runs = nullptr; sse_seg_result *d_segres = nullptr;
    Counters *d_ctr = nullptr;
    uint4 *d_items = nullptr; uint32_t *d_segterm = nullptr;   // split pipeline scratch (device only)
    uint4 *d_items2 = nullptr;                                 // items ordered for the decode kernel
    uint2 *d_tiles = nullptr;                                  // fused pipeline: tile list of the plan kernel
    uint32_t n_segs = 0, in_bytes = 0;
    uint32_t cap_tcs = 0, cap_usages = 0, cap_text = 0;        // decode-stage capacities (SSE_FLAG_DEFER grows them per slot)
    // SSE_FLAG_COUNTERS: the batch's counter block (CN_*), device and pinned; kept apart from Counters, which the default path
    // clears and downloads every batch
    unsigned long long *d_cnt = nullptr, *h_cnt = nullptr;
    uint32_t decode_passes = 0;
    bool cnt_ready = false;                                    // h_cnt holds the counters of the batch last downloaded
    bool ctr_queued = false;                                   // sse_submit queued the D2H of h_ctr (do_download does not)
    uint32_t pool_short = 0;                                   // SSE_OVF_POOL: pages the collected batch's lines lacked
    uint32_t pool_gen = 0;                                     // sse_ctx.pool_gen when the batch was launched
    bool trim = false;                                         // sse_trim: shrink the decode arenas at sse_release
};

// Line-pool arrays replaced by a growth, freed once the event recorded after their last reader has completed.
struct RetiredPool {
    uint8_t *pool; uint32_t *stack, *next;
    cudaEvent_t done;
    uint32_t pages;
};

} // namespace

// Device layout of a slot's byte arenas: [out arena | pad | in arena] in ONE allocation, so that a single base pointer and
// a 32-bit offset address both. Offsets >= in_base are input bytes (zero-copy frames and their spans).
static inline uint32_t in_base_of(const sse_config &cfg) { return (cfg.out_arena_bytes + 255u) & ~255u; }

struct sse_ctx {
    int device = 0;
    int sm_count = 0;
    sse_config cfg{};
    ConnState *d_conns = nullptr;
    uint8_t *d_carry = nullptr;
    uint32_t *d_tcache = nullptr;        // fused kernel: skeleton templates kept between launches
    sse_line_pool pool{};                // pool_pages == 0: no line pool
    uint8_t *d_pool = nullptr; PoolHdr *d_pool_hdr = nullptr; uint32_t *d_pool_stack = nullptr, *d_pool_next = nullptr;
    PoolChain *d_pool_chain = nullptr;
    PoolHdr *h_pool_hdr = nullptr;       // pinned: sse_line_pool_stats
    uint32_t pool_max = 0;               // sse_line_pool_set_growth: most pages the pool may grow to (0: no growth)
    std::vector<RetiredPool> retired;    // pool arrays a growth replaced, until no queued work can read them
    uint32_t pool_gen = 0;               // growths and trims so far
    uint64_t device_bytes = 0, pinned_bytes = 0;   // sse_memory_held: what the allocations below hold now
    cudaStream_t ctl_stream = nullptr;
    cudaEvent_t last_kernel = nullptr;   // completion of the most recently launched kernel
    bool have_last = false;
    std::vector<Slot> slots;
    uint64_t launches = 0;
};

namespace {

// Every allocation of a context goes through these (or adds its bytes to device_bytes / pinned_bytes where it is made), and every
// free before sse_destroy takes its bytes off, so that sse_memory_held is what the context holds.
template <class T> size_t alloc_bytes(size_t n) { return n ? n * sizeof(T) : sizeof(T); }
template <class T> bool dalloc(sse_ctx *c, T *&p, size_t n) {
    if (!cu_ok(cudaMalloc((void **)&p, alloc_bytes<T>(n)), "cudaMalloc")) return false;
    c->device_bytes += alloc_bytes<T>(n);
    return true;
}
template <class T> bool halloc(sse_ctx *c, T *&p, size_t n) {
    if (!cu_ok(cudaHostAlloc((void **)&p, alloc_bytes<T>(n), cudaHostAllocDefault), "cudaHostAlloc")) return false;
    c->pinned_bytes += alloc_bytes<T>(n);
    return true;
}
uint64_t pool_bytes(const sse_ctx *c, uint32_t pages) { return (uint64_t)pages * (c->pool.page_bytes + 8u); }   // pages, stack, next

void free_slot(Slot &s) {
    if (s.stream) cudaStreamDestroy(s.stream);
    if (s.kernel_done) cudaEventDestroy(s.kernel_done);
    cudaFreeHost(s.h_in); cudaFreeHost(s.h_segs); cudaFreeHost(s.h_out); cudaFreeHost(s.h_frames); cudaFreeHost(s.h_recs);
    cudaFreeHost(s.h_tcs); cudaFreeHost(s.h_usages); cudaFreeHost(s.h_text); cudaFreeHost(s.h_runs); cudaFreeHost(s.h_segres);
    cudaFreeHost(s.h_ctr); cudaFreeHost(s.h_cnt); cudaFree(s.d_cnt);
    cudaFree(s.d_segs); cudaFree(s.d_out);   // d_in lives inside d_out's allocation
    cudaFree(s.d_frames); cudaFree(s.d_recs); cudaFree(s.d_tcs);
    cudaFree(s.d_usages); cudaFree(s.d_text); cudaFree(s.d_runs); cudaFree(s.d_segres); cudaFree(s.d_ctr); cudaFree(s.d_items); cudaFree(s.d_segterm); cudaFree(s.d_items2); cudaFree(s.d_tiles);
}

KParams make_params(sse_ctx *c, Slot &s, uint32_t n_segs) {
    KParams p{};
    p.in = s.d_in; p.segs = s.d_segs; p.n_segs = n_segs; p.max_conns = c->cfg.max_conns;
    p.conns = c->d_conns; p.carry = c->d_carry; p.carry_slot = c->cfg.carry_slot_bytes;
    p.out = s.d_out; p.cap_out = c->cfg.out_arena_bytes; p.in_base = in_base_of(c->cfg);
    p.frames = s.d_frames; p.cap_frames = c->cfg.max_frames;
    p.recs = s.d_recs; p.cap_recs = c->cfg.max_recs;
    p.tcs = s.d_tcs; p.cap_tcs = s.cap_tcs;
    p.usages = s.d_usages; p.cap_usages = s.cap_usages;
    p.text = s.d_text; p.cap_text = s.cap_text;
    p.runs = s.d_runs; p.cap_runs = c->cfg.max_runs;
    p.seg_results = s.d_segres; p.ctr = s.d_ctr;
    p.items = s.d_items; p.cap_items = c->cfg.max_recs; p.seg_term = s.d_segterm;
    p.items_sorted = s.d_items2; p.flags = c->cfg.flags;
    p.tiles = s.d_tiles; p.cap_tiles = c->cfg.max_segs + 64;
    p.tcache = (c->cfg.flags & SSE_FLAG_TEMPLATES) ? c->d_tcache : nullptr;
    p.pool = c->d_pool; p.pool_hdr = c->d_pool_hdr; p.pool_stack = c->d_pool_stack; p.pool_next = c->d_pool_next;
    p.pool_chain = c->d_pool_chain;
    p.page_bytes = c->pool.page_bytes; p.pool_pages = c->pool.pool_pages;
    p.max_line = c->pool.pool_pages ? c->pool.max_line_bytes : c->cfg.carry_slot_bytes;
    p.long_line = (SSE_LONG_LINE && !(c->cfg.flags & SSE_FLAG_KERNEL_FUSED) && p.max_line >= SSE_LONG_LINE) ? SSE_LONG_LINE : 0u;
    p.cnt = s.d_cnt;
    return p;
}

// KParams for the line-pool maintenance kernel (no batch slot involved)
KParams pool_params(sse_ctx *c) {
    KParams p{};
    p.max_conns = c->cfg.max_conns; p.conns = c->d_conns;
    p.pool = c->d_pool; p.pool_hdr = c->d_pool_hdr; p.pool_stack = c->d_pool_stack; p.pool_next = c->d_pool_next;
    p.pool_chain = c->d_pool_chain; p.page_bytes = c->pool.page_bytes; p.pool_pages = c->pool.pool_pages;
    return p;
}

int validate_segs(sse_ctx *c, Slot &s, uint32_t n_segs, uint32_t in_bytes) {
    if (n_segs > c->cfg.max_segs || in_bytes > c->cfg.in_arena_bytes) return SSE_ERR_ARG;
    for (uint32_t i = 0; i < n_segs; i++) {
        const sse_seg &g = s.h_segs[i];
        if (g.conn >= c->cfg.max_conns || (g.in_off & 15u) || (uint64_t)g.in_off + g.in_len > in_bytes) return SSE_ERR_ARG;
    }
    return SSE_OK;
}

int do_upload(sse_ctx *c, Slot &s, uint32_t n_segs, uint32_t in_bytes, cudaStream_t st) {
    if (n_segs) CU(cudaMemcpyAsync(s.d_segs, s.h_segs, (size_t)n_segs * sizeof(sse_seg), cudaMemcpyHostToDevice, st));
    if (in_bytes) CU(cudaMemcpyAsync(s.d_in, s.h_in, ((size_t)in_bytes + 15) & ~(size_t)15, cudaMemcpyHostToDevice, st));
    s.n_segs = n_segs; s.in_bytes = in_bytes;
    (void)c;
    return SSE_OK;
}

int do_launch(sse_ctx *c, Slot &s, uint32_t n_segs, cudaStream_t st) {
    CU(cudaMemsetAsync(s.d_ctr, 0, sizeof(Counters), st));
    s.cnt_ready = false;
    s.pool_gen = c->pool_gen;
    if (s.d_cnt) CU(cudaMemsetAsync(s.d_cnt, 0, CN_COUNT * sizeof(unsigned long long), st));
    if (n_segs) {
        KParams p = make_params(c, s, n_segs);
        int e;
        if (c->cfg.flags & SSE_FLAG_KERNEL_FUSED) {   // plan + single-pass tile kernel
            e = sse_launch_fused(p, (void *)st, c->sm_count, c->device);
            c->launches += 2;
        }
        else {   // default: produce -> sort -> decode (templates / automaton) -> finalize
            e = sse_launch_produce_kernel(p, (void *)st, c->sm_count);
            if (e == 0) e = sse_launch_decode_finalize(p, (void *)st, c->sm_count, c->device);
            c->launches += p.long_line ? 7 : 6;   // produce, bucket hist/scan/scatter, [long-line decode,] decode, finalize
        }
        if (e != 0) { cu_ok((cudaError_t)e, "stream kernel launch"); return SSE_ERR_CUDA; }
    }
    s.n_segs = n_segs;
    return SSE_OK;
}

// The decode stage's arenas for a batch whose decoded payloads take at most `payload` bytes: a tool-call element is allocated only
// while its line can still be JSON_OK, so it takes at least 3 payload bytes ("{},"); a decoded string takes at most 4 text bytes per
// payload byte (U+FFFD for every invalid byte, 4-byte aligned allocations); there is at most one usage per record.
void decode_caps(sse_config &w, uint64_t payload) {
    const uint64_t cap = 0xF0000000ull;
    auto clamp = [&](uint64_t v) { return (uint32_t)(v > cap ? cap : v); };
    w.max_usages = w.max_recs;
    w.max_tcs = clamp(payload / 3 + 64);
    w.text_arena_bytes = clamp(4 * payload + 65536);
}

// Upper bounds of what one batch can ask of the decode stage's arenas. Every payload the decode stage reads stands in the batch's
// input arena or in its out arena (lines completed from the carry slot or the line pool), so the bounds are decode_caps over both
// arenas together (the out arena already includes the line pool's growth).
sse_config worst_decode_caps(const sse_ctx *c) {
    sse_config w = c->cfg;
    decode_caps(w, (uint64_t)w.in_arena_bytes + w.out_arena_bytes);
    return w;
}

// One decode-stage arena of a slot goes from cap to want elements of T, device and pinned (the slot's stream is idle): grows it
// (redecode) or gives back what a growth took (sse_trim).
template <class T> int resize_arena(sse_ctx *c, T *&d, T *&h, uint32_t &cap, uint32_t want) {
    T *nd = nullptr, *nh = nullptr;
    if (cudaMalloc((void **)&nd, alloc_bytes<T>(want)) != cudaSuccess) { cudaGetLastError(); return SSE_ERR_NOMEM; }
    if (cudaHostAlloc((void **)&nh, alloc_bytes<T>(want), cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); cudaFree(nd); return SSE_ERR_NOMEM; }
    cudaFree(d); cudaFreeHost(h);
    c->device_bytes += alloc_bytes<T>(want) - alloc_bytes<T>(cap);
    c->pinned_bytes += alloc_bytes<T>(want) - alloc_bytes<T>(cap);
    d = nd; h = nh; cap = want;
    return SSE_OK;
}

// sse_trim: the slot's decode arenas back to the configured capacities (the slot holds no batch, or its stream is idle and its
// results are no longer lent).
int trim_arenas(sse_ctx *c, Slot &s) {
    int rc = SSE_OK;
    if (s.cap_tcs != c->cfg.max_tcs) rc = resize_arena(c, s.d_tcs, s.h_tcs, s.cap_tcs, c->cfg.max_tcs);
    if (rc == SSE_OK && s.cap_usages != c->cfg.max_usages) rc = resize_arena(c, s.d_usages, s.h_usages, s.cap_usages, c->cfg.max_usages);
    if (rc == SSE_OK && s.cap_text != c->cfg.text_arena_bytes) rc = resize_arena(c, s.d_text, s.h_text, s.cap_text, c->cfg.text_arena_bytes);
    s.trim = rc != SSE_OK;   // an allocation failed: the next sse_release tries again
    return rc;
}

// SSE_FLAG_DEFER: the decode stage ran out of tool-call, usage or text arena (k: its counters, which count on past a capacity, so
// they say what the batch needs, less what the records that failed earlier could not ask for). Grows each arena that ran out to at
// least what was counted, and to twice its size where that stays within worst_decode_caps, then runs the decode stage again over the
// same sorted work items; repeats until the batch fits. Every pass grows an arena past its count, so the loop ends, at the latest
// when an allocation fails (SSE_ERR_NOMEM). The finalize stage is not run again: where a segment terminates does not depend on these
// arenas, and it already ran, so connection state and line-pool pages are never touched twice. Later batches may have been
// submitted meanwhile: the pass is ordered after them (the template cache is shared) and they after it.
int redecode(sse_ctx *c, Slot &s, Counters &k, cudaStream_t st, uint32_t &grown) {
    const sse_config w = worst_decode_caps(c);
    auto want = [](uint32_t cap, uint32_t need, uint32_t worst) {
        uint64_t v = (uint64_t)cap * 2u;
        if (v > worst) v = worst;
        if (v < need) v = need;
        return (uint32_t)(v > 0xF0000000ull ? 0xF0000000ull : v);
    };
    auto grow = [&](auto *&d, auto *&h, uint32_t &cap, uint32_t need, uint32_t worst) {
        const uint32_t n = want(cap, need, worst);
        return n > cap ? resize_arena(c, d, h, cap, n) : (int)SSE_ERR_NOMEM;
    };
    while (k.status == SSE_ERR_OVERFLOW) {
        const uint32_t ovf = k.overflow & (SSE_OVF_TCS | SSE_OVF_USAGES | SSE_OVF_TEXT);
        if (!ovf) return SSE_ERR_OVERFLOW;   // not reachable: with SSE_FLAG_DEFER only the decode stage fails a batch
        int rc = SSE_OK;
        if (ovf & SSE_OVF_TCS) rc = grow(s.d_tcs, s.h_tcs, s.cap_tcs, k.n_tcs, w.max_tcs);
        if (rc == SSE_OK && (ovf & SSE_OVF_USAGES)) rc = grow(s.d_usages, s.h_usages, s.cap_usages, k.n_usages, w.max_usages);
        if (rc == SSE_OK && (ovf & SSE_OVF_TEXT)) rc = grow(s.d_text, s.h_text, s.cap_text, k.text_bytes, w.text_arena_bytes);
        if (rc != SSE_OK) return rc;
        grown |= ovf;
        // the lane decoder's items start after the long ones (items_sorted[0, n_long)), which the long-line kernel takes again
        k.n_tcs = k.n_usages = k.text_bytes = 0; k.item_ticket = k.n_long; k.long_ticket = 0; k.status = SSE_OK; k.overflow = 0;
        *s.h_ctr = k;
        CU(cudaMemcpyAsync(s.d_ctr, s.h_ctr, offsetof(Counters, class_count), cudaMemcpyHostToDevice, st));
        if (s.d_cnt) {   // the decode counters describe the pass whose records the batch returns
            CU(cudaMemsetAsync(s.d_cnt + CN_DECODE_FIRST, 0, (CN_COUNT - CN_DECODE_FIRST) * sizeof(unsigned long long), st));
            s.decode_passes++;
        }
        if (c->have_last) CU(cudaStreamWaitEvent(st, c->last_kernel, 0));
        const KParams p = make_params(c, s, s.n_segs);
        const int e = sse_launch_decode(p, (void *)st, c->sm_count, c->device);
        if (e != 0) { cu_ok((cudaError_t)e, "decode kernel launch"); return SSE_ERR_CUDA; }
        c->launches += p.long_line ? 2 : 1;
        CU(cudaEventRecord(c->last_kernel, st));
        c->have_last = true;
        CU(cudaMemcpyAsync(s.h_ctr, s.d_ctr, offsetof(Counters, class_count), cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        k = *s.h_ctr;
    }
    return SSE_OK;
}

int do_download(sse_ctx *c, Slot &s, sse_result *res, cudaStream_t st) {
    if (!s.ctr_queued) CU(cudaMemcpyAsync(s.h_ctr, s.d_ctr, offsetof(Counters, class_count), cudaMemcpyDeviceToHost, st));
    s.ctr_queued = false;
    CU(cudaStreamSynchronize(st));
    Counters k = *s.h_ctr;
    s.pool_short = k.pool_short;
    memset(res, 0, sizeof *res);
    res->n_segs = s.n_segs;
    s.decode_passes = s.n_segs ? 1u : 0u;
    uint32_t bits = 0;
    if (c->cfg.flags & SSE_FLAG_DEFER) {
        // the produce stage reports what it deferred in k.overflow without failing the batch; only the decode stage sets status
        bits = k.overflow;
        const int rc = redecode(c, s, k, st, bits);
        if (rc != SSE_OK) { res->status = rc; res->overflow = bits | k.overflow; return rc; }
    }
    res->status = k.status;
    if (k.status != SSE_OK) {   // overflow: the batch result is unusable, report loudly
        res->overflow = k.overflow;
        return k.status;
    }
    res->overflow = bits;
    // a deferred allocation may leave a produce-stage counter past its capacity (the holes below it are never referenced)
    auto lim = [](uint32_t n, uint32_t cap) { return n < cap ? n : cap; };
    k.n_frames = lim(k.n_frames, c->cfg.max_frames); k.n_recs = lim(k.n_recs, c->cfg.max_recs); k.n_runs = lim(k.n_runs, c->cfg.max_runs);
    k.out_bytes = lim(k.out_bytes, c->cfg.out_arena_bytes); k.n_items = lim(k.n_items, c->cfg.max_recs);
    k.n_tcs = lim(k.n_tcs, s.cap_tcs); k.n_usages = lim(k.n_usages, s.cap_usages); k.text_bytes = lim(k.text_bytes, s.cap_text);
    res->n_frames = k.n_frames; res->n_recs = k.n_recs; res->n_tcs = k.n_tcs; res->n_usages = k.n_usages;
    res->n_runs = k.n_runs; res->out_bytes = k.out_bytes; res->text_bytes = k.text_bytes;
    res->n_decoded = k.n_items; res->n_derived = 0;
    if (k.out_bytes) CU(cudaMemcpyAsync(s.h_out, s.d_out, k.out_bytes, cudaMemcpyDeviceToHost, st));
    if (k.n_frames) CU(cudaMemcpyAsync(s.h_frames, s.d_frames, (size_t)k.n_frames * sizeof(sse_frame), cudaMemcpyDeviceToHost, st));
    if (k.n_recs) CU(cudaMemcpyAsync(s.h_recs, s.d_recs, (size_t)k.n_recs * sizeof(sse_rec), cudaMemcpyDeviceToHost, st));
    if (k.n_tcs) CU(cudaMemcpyAsync(s.h_tcs, s.d_tcs, (size_t)k.n_tcs * sizeof(sse_tc), cudaMemcpyDeviceToHost, st));
    if (k.n_usages) CU(cudaMemcpyAsync(s.h_usages, s.d_usages, (size_t)k.n_usages * sizeof(sse_usage), cudaMemcpyDeviceToHost, st));
    if (k.text_bytes) CU(cudaMemcpyAsync(s.h_text, s.d_text, k.text_bytes, cudaMemcpyDeviceToHost, st));
    if (k.n_runs) CU(cudaMemcpyAsync(s.h_runs, s.d_runs, (size_t)k.n_runs * sizeof(sse_run), cudaMemcpyDeviceToHost, st));
    if (s.n_segs) CU(cudaMemcpyAsync(s.h_segres, s.d_segres, (size_t)s.n_segs * sizeof(sse_seg_result), cudaMemcpyDeviceToHost, st));
    if (s.d_cnt) CU(cudaMemcpyAsync(s.h_cnt, s.d_cnt, CN_COUNT * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    s.cnt_ready = s.d_cnt != nullptr;
    res->out = s.h_out; res->frames = s.h_frames; res->recs = s.h_recs; res->tcs = s.h_tcs; res->usages = s.h_usages;
    res->text = s.h_text; res->runs = s.h_runs; res->segs = s.h_segres;
    res->in = s.h_in; res->in_base = in_base_of(c->cfg);
    return SSE_OK;
}

// Frees the retired pool arrays whose last reader has completed (all: every one, the device being idle).
void free_retired(sse_ctx *c, bool all) {
    size_t k = 0;
    for (RetiredPool &r : c->retired) {
        if (!all) {
            const cudaError_t e = cudaEventQuery(r.done);
            if (e == cudaErrorNotReady && cudaPeekAtLastError() == cudaErrorNotReady) cudaGetLastError();   // still queued: not an error
            if (e != cudaSuccess) { c->retired[k++] = r; continue; }
        }
        cudaFree(r.pool); cudaFree(r.stack); cudaFree(r.next); cudaEventDestroy(r.done);
        c->device_bytes -= pool_bytes(c, r.pages);
    }
    c->retired.resize(k);
}

// SSE_FLAG_DEFER with pool growth: a batch's lines lacked `lacked` pages. The pool grows to twice its pages, or by what was
// lacked when that is more, at most to pool_max. The new arrays start with copies of the old ones, so page ids, chains and held
// lines stay as they are; the copies and the kernel that frees the new pages are ordered after every submitted batch (which
// were launched with the old arrays) and every later launch is ordered after them and gets the new arrays. When the device
// cannot allocate them the pool stays as it is and stops growing: its lines fail at the limit as without growth.
int grow_pool(sse_ctx *c, uint32_t lacked) {
    const uint32_t cap = c->pool.pool_pages, PB = c->pool.page_bytes;
    uint64_t want = (uint64_t)cap * 2u;
    if (want < (uint64_t)cap + lacked) want = (uint64_t)cap + lacked;
    if (want > c->pool_max) want = c->pool_max;
    if (want <= cap) return SSE_OK;
    free_retired(c, false);
    RetiredPool old{ c->d_pool, c->d_pool_stack, c->d_pool_next, nullptr, cap };
    uint8_t *pool = nullptr; uint32_t *stack = nullptr, *next = nullptr;
    bool ok = cudaMalloc((void **)&pool, (size_t)want * PB) == cudaSuccess && cudaMalloc((void **)&stack, (size_t)want * 4) == cudaSuccess &&
              cudaMalloc((void **)&next, (size_t)want * 4) == cudaSuccess &&
              cudaEventCreateWithFlags(&old.done, cudaEventDisableTiming) == cudaSuccess;
    if (!ok) {
        if (cudaPeekAtLastError() == cudaErrorMemoryAllocation) cudaGetLastError();   // the failed allocation only
        cudaFree(pool); cudaFree(stack); cudaFree(next);
        if (old.done) cudaEventDestroy(old.done);
        c->pool_max = cap;
        if (c->have_last) CU(cudaStreamWaitEvent(c->ctl_stream, c->last_kernel, 0));
        CU(cudaMemsetAsync(&c->d_pool_hdr->grow, 0, sizeof(uint32_t), c->ctl_stream));
        CU(cudaEventRecord(c->last_kernel, c->ctl_stream));
        c->have_last = true;
        return SSE_OK;
    }
    cudaStream_t st = c->ctl_stream;
    if (c->have_last) CU(cudaStreamWaitEvent(st, c->last_kernel, 0));
    CU(cudaMemcpyAsync(pool, c->d_pool, (size_t)cap * PB, cudaMemcpyDeviceToDevice, st));
    CU(cudaMemcpyAsync(stack, c->d_pool_stack, (size_t)cap * 4, cudaMemcpyDeviceToDevice, st));
    CU(cudaMemcpyAsync(next, c->d_pool_next, (size_t)cap * 4, cudaMemcpyDeviceToDevice, st));
    CU(cudaEventRecord(old.done, st));
    c->retired.push_back(old);
    c->device_bytes += pool_bytes(c, (uint32_t)want);
    c->d_pool = pool; c->d_pool_stack = stack; c->d_pool_next = next; c->pool.pool_pages = (uint32_t)want;
    c->pool_gen++;
    if (!cu_ok((cudaError_t)sse_launch_pool_extend(pool_params(c), cap, want < c->pool_max, st), "pool extend kernel")) return SSE_ERR_CUDA;
    CU(cudaEventRecord(c->last_kernel, st));
    c->have_last = true;
    return SSE_OK;
}

// sse_trim of a pool with a growth limit; the context's stream has just waited for every submitted batch, so the pool is idle
// and n_free is final. The pool shrinks to max(min_pages, pages held, 1) pages when that is below its capacity: the held pages
// are repacked into the first pages of new, smaller arrays (sse_launch_pool_repack), the rest go on the free stack. Every
// later launch is ordered after the repack and gets the new arrays; the old ones are freed before this returns (cudaFree waits
// for the queued repack, their last reader).
int trim_pool(sse_ctx *c, uint32_t min_pages) {
    cudaStream_t st = c->ctl_stream;
    CU(cudaMemcpyAsync(c->h_pool_hdr, c->d_pool_hdr, sizeof(PoolHdr), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    free_retired(c, false);   // every growth's copy is done
    const uint32_t cap = c->pool.pool_pages, held = cap - c->h_pool_hdr->n_free, PB = c->pool.page_bytes;
    uint32_t want = min_pages > held ? min_pages : held;
    if (want < 1) want = 1;
    if (want >= cap) return SSE_OK;
    uint8_t *pool = nullptr; uint32_t *stack = nullptr, *next = nullptr;
    if (cudaMalloc((void **)&pool, (size_t)want * PB) != cudaSuccess || cudaMalloc((void **)&stack, (size_t)want * 4) != cudaSuccess ||
        cudaMalloc((void **)&next, (size_t)want * 4) != cudaSuccess) {
        if (cudaPeekAtLastError() == cudaErrorMemoryAllocation) cudaGetLastError();   // the failed allocation only
        cudaFree(pool); cudaFree(stack); cudaFree(next);
        return SSE_ERR_NOMEM;
    }
    KParams p = pool_params(c);   // the old arrays
    const int e = sse_launch_pool_repack(p, pool, stack, next, held, want, want < c->pool_max, c->sm_count, st);
    if (!cu_ok((cudaError_t)e, "pool repack kernels")) { cudaFree(pool); cudaFree(stack); cudaFree(next); return SSE_ERR_CUDA; }
    CU(cudaEventRecord(c->last_kernel, st));
    c->have_last = true;
    cudaFree(c->d_pool); cudaFree(c->d_pool_stack); cudaFree(c->d_pool_next);
    c->device_bytes += pool_bytes(c, want);
    c->device_bytes -= pool_bytes(c, cap);
    c->d_pool = pool; c->d_pool_stack = stack; c->d_pool_next = next; c->pool.pool_pages = want;
    c->pool_gen++;            // a batch launched before the trim reports its lack against the old pool: it does not grow this one
    return SSE_OK;
}

} // namespace

extern "C" {

int sse_abi_version(void) { return SSE_ABI_VERSION; }

const uint8_t *sse_at(const sse_result *r, uint32_t off) { return off >= r->in_base ? r->in + (off - r->in_base) : r->out + off; }

const char *sse_last_cuda_error(void) { return g_cuda_err; }

const char *sse_strerror(int status) {
    switch (status) {
    case SSE_OK: return "ok";
    case SSE_ERR_NO_DEVICE: return "no CUDA device available (libssegpu has no CPU fallback)";
    case SSE_ERR_CUDA: return "CUDA error (see sse_last_cuda_error)";
    case SSE_ERR_ARG: return "invalid argument";
    case SSE_ERR_BUSY: return "batch slot busy or in the wrong state";
    case SSE_ERR_OVERFLOW: return "result arena overflow: batch discarded (increase sse_config capacities)";
    case SSE_ERR_NOMEM: return "out of memory";
    case SSE_ERR_UNDECODED: return "a line was not decoded (SSE_F_TOO_LONG / SSE_F_DEPTH_LIMIT): fold results are incomplete";
    default: return "unknown status";
    }
}

void sse_default_config(sse_config *cfg, uint32_t max_conns, uint32_t bytes_per_batch) {
    memset(cfg, 0, sizeof *cfg);
    cfg->struct_size = sizeof *cfg;
    cfg->max_conns = max_conns;
    cfg->max_segs = max_conns;
    uint64_t in = ((uint64_t)bytes_per_batch + 16ull * max_conns + 4095) & ~4095ull;
    cfg->in_arena_bytes = (uint32_t)(in > 0xF0000000ull ? 0xF0000000ull : in);
    uint64_t out = in + in / 8 + 65536;
    cfg->out_arena_bytes = (uint32_t)(out > 0xF0000000ull ? 0xF0000000ull : out);
    cfg->max_frames = (uint32_t)(in / 32 + 4ull * max_conns + 1024);
    cfg->max_recs = (uint32_t)(in / 64 + 2ull * max_conns + 1024);
    cfg->max_tcs = (uint32_t)(in / 256 + 1024);
    cfg->max_usages = cfg->max_recs;
    cfg->text_arena_bytes = (uint32_t)(in / 4 + 65536);
    cfg->max_runs = (uint32_t)(in / 2048 + max_conns + 1024);   // one extra run per round of 64 lines: lines of 32 bytes or more
    cfg->carry_slot_bytes = 16384;
    cfg->n_slots = 2;
}

void sse_worst_case_config(sse_config *cfg, uint32_t max_conns, uint32_t bytes_per_batch) {
    sse_default_config(cfg, max_conns, bytes_per_batch);
    const uint64_t in = cfg->in_arena_bytes, cap = 0xF0000000ull;
    auto clamp = [&](uint64_t v) { return (uint32_t)(v > cap ? cap : v); };
    cfg->carry_slot_bytes = 65536;                                   // longest supported line
    cfg->max_frames = clamp(in + 64);                                // a frame needs its own '\n' in this batch
    cfg->max_recs = clamp(in / 4 + 2ull * max_conns + 64);           // "data: x\n" is 8 bytes; one carried line per segment
    cfg->out_arena_bytes = clamp(in + in / 4 + (uint64_t)max_conns * (cfg->carry_slot_bytes + 32ull) + (1u << 20));
    // the decode stage reads the batch's input and, for every connection, at most one line completed from its carry slot
    decode_caps(*cfg, in + (uint64_t)max_conns * cfg->carry_slot_bytes);
    // one runs[] entry per round of up to 64 lines after a segment's first: a round per 64 one-byte lines, and at most one more
    // per window (a window after a segment's first takes half a window of new bytes or more, a line longer than a window
    // completes once)
    cfg->max_runs = clamp(in / 64 + in / 2048 + 2ull * max_conns + 1024);
}

void sse_line_pool_config(sse_config *cfg, const sse_line_pool *pool) {
    if (!cfg || !pool || pool->struct_size != sizeof(sse_line_pool) || pool->pool_pages == 0 || cfg->in_arena_bytes == 0) return;
    // every capacity grows by the pool's bytes at the ratio (capacity / input byte) the config already has
    const unsigned __int128 extra = (unsigned __int128)pool->pool_pages * (pool->page_bytes ? pool->page_bytes : 65536u);
    const uint64_t in = cfg->in_arena_bytes, cap = 0xF0000000ull;
    auto grow = [&](uint32_t &x) {
        const unsigned __int128 v = (unsigned __int128)x + ((unsigned __int128)x * extra + in - 1) / in;
        x = (uint32_t)(v > cap ? cap : (uint64_t)v);
    };
    grow(cfg->out_arena_bytes); grow(cfg->max_frames); grow(cfg->max_recs); grow(cfg->max_tcs);
    grow(cfg->max_usages); grow(cfg->text_arena_bytes); grow(cfg->max_runs);
}

int sse_init(int device, const sse_config *cfg, sse_ctx **out) { return sse_init_ex(device, cfg, nullptr, out); }

int sse_init_ex(int device, const sse_config *cfg_in, const sse_line_pool *pool_in, sse_ctx **out) {
    if (!cfg_in || !out || cfg_in->struct_size != sizeof(sse_config)) return SSE_ERR_ARG;
    sse_line_pool pool{};
    pool.struct_size = sizeof pool;
    sse_config grown = *cfg_in;
    if (pool_in) {
        if (pool_in->struct_size != sizeof(sse_line_pool) || (pool_in->page_bytes & 15u) || pool_in->pool_pages == SSE_NONE ||
            pool_in->max_line_bytes > SSE_MAX_LINE_BYTES || pool_in->max_line_bytes < cfg_in->carry_slot_bytes ||
            (cfg_in->flags & SSE_FLAG_KERNEL_FUSED)) return SSE_ERR_ARG;   // the tile kernel has no line pool
        pool = *pool_in;
        if (!pool.page_bytes) pool.page_bytes = 65536;
        sse_line_pool_config(&grown, &pool);
    }
    const sse_config *cfg = &grown;
    if (cfg->n_slots < 1 || cfg->n_slots > 8 || cfg->max_conns == 0 || cfg->max_segs == 0 ||
        (cfg->in_arena_bytes & 15u) || cfg->carry_slot_bytes < 8192 + 16 || (cfg->carry_slot_bytes & 15u)) return SSE_ERR_ARG;
    if ((uint64_t)in_base_of(*cfg) + cfg->in_arena_bytes + 16 >= (1ull << 31)) return SSE_ERR_ARG;   // arena offsets are 31-bit
    if (cfg->flags & ~(SSE_FLAG_KERNEL_FUSED | SSE_FLAG_COPY_OUT | SSE_FLAG_TEMPLATES | SSE_FLAG_DEFER | SSE_FLAG_COUNTERS)) return SSE_ERR_ARG;   // unknown engine flag
    if ((cfg->flags & SSE_FLAG_DEFER) && (cfg->flags & SSE_FLAG_KERNEL_FUSED)) return SSE_ERR_ARG;   // the tile kernel does not defer
    if ((cfg->flags & SSE_FLAG_COUNTERS) && (cfg->flags & SSE_FLAG_KERNEL_FUSED)) return SSE_ERR_ARG;   // ... and has no counting instantiation
    // with SSE_FLAG_DEFER a segment alone in a batch must always get somewhere: one round of up to 64 lines (at most a window of
    // bytes plus a '\n' per line), and the longest line a connection may hold, must fit an empty batch
    if ((cfg->flags & SSE_FLAG_DEFER) &&
        (cfg->max_frames < 64 || cfg->max_recs < 64 || cfg->out_arena_bytes < 8192 + 1024 ||
         (uint64_t)cfg->out_arena_bytes < (uint64_t)(pool.pool_pages ? pool.max_line_bytes : cfg->carry_slot_bytes) + 64)) return SSE_ERR_ARG;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0 || device < 0 || device >= n) {
        cu_ok(cudaGetLastError(), "cudaGetDeviceCount");
        return SSE_ERR_NO_DEVICE;
    }
    CU(cudaSetDevice(device));
    sse_ctx *c = new (std::nothrow) sse_ctx();
    if (!c) return SSE_ERR_NOMEM;
    c->device = device; c->cfg = *cfg; c->pool = pool;
    cudaDeviceProp prop;
    if (!cu_ok(cudaGetDeviceProperties(&prop, device), "cudaGetDeviceProperties")) { delete c; return SSE_ERR_CUDA; }
    c->sm_count = prop.multiProcessorCount;
    if (cfg->flags & SSE_FLAG_KERNEL_FUSED) {
        if (cfg->carry_slot_bytes > sse_fused_max_line()) { delete c; return SSE_ERR_ARG; }
        int e2 = sse_fused_prepare(device);
        if (e2 != 0) { cu_ok((cudaError_t)e2, "sse_fused_prepare"); delete c; return SSE_ERR_CUDA; }
    } else {
        int e2 = sse_v2_prepare(device);
        if (e2 != 0) { cu_ok((cudaError_t)e2, "sse_v2_prepare"); delete c; return SSE_ERR_CUDA; }
    }
    bool ok = true;
    ok = ok && cu_ok(cudaStreamCreateWithFlags(&c->ctl_stream, cudaStreamNonBlocking), "cudaStreamCreate");
    ok = ok && cu_ok(cudaEventCreateWithFlags(&c->last_kernel, cudaEventDisableTiming), "cudaEventCreate");
    ok = ok && dalloc(c, c->d_conns, cfg->max_conns);
    ok = ok && dalloc(c, c->d_carry, (size_t)cfg->max_conns * cfg->carry_slot_bytes);
    ok = ok && cu_ok(cudaMemset(c->d_conns, 0, (size_t)cfg->max_conns * sizeof(ConnState)), "cudaMemset");
    ok = ok && dalloc(c, c->d_tcache, sse_fused_tcache_words());
    ok = ok && cu_ok(cudaMemset(c->d_tcache, 0, (size_t)sse_fused_tcache_words() * sizeof(uint32_t)), "cudaMemset");
    if (ok && pool.pool_pages) {
        ok = ok && dalloc(c, c->d_pool, (size_t)pool.pool_pages * pool.page_bytes) && dalloc(c, c->d_pool_hdr, 1);
        ok = ok && dalloc(c, c->d_pool_stack, pool.pool_pages) && dalloc(c, c->d_pool_next, pool.pool_pages);
        ok = ok && dalloc(c, c->d_pool_chain, cfg->max_conns) && halloc(c, c->h_pool_hdr, 1);
        ok = ok && cu_ok(cudaMemset(c->d_pool_hdr, 0, sizeof(PoolHdr)), "cudaMemset");
        ok = ok && cu_ok((cudaError_t)sse_launch_pool_reset(pool_params(c), SSE_NONE, c->ctl_stream), "pool reset kernel");
        ok = ok && cu_ok(cudaStreamSynchronize(c->ctl_stream), "cudaStreamSynchronize");
    }
    c->slots.resize(cfg->n_slots);
    for (auto &s : c->slots) {
        if (!ok) break;
        ok = ok && cu_ok(cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking), "cudaStreamCreate");
        ok = ok && cu_ok(cudaEventCreateWithFlags(&s.kernel_done, cudaEventDisableTiming), "cudaEventCreate");
        ok = ok && halloc(c, s.h_in, (size_t)cfg->in_arena_bytes + 16) && halloc(c, s.h_segs, cfg->max_segs);
        ok = ok && halloc(c, s.h_out, cfg->out_arena_bytes) && halloc(c, s.h_frames, cfg->max_frames) && halloc(c, s.h_recs, cfg->max_recs);
        ok = ok && halloc(c, s.h_tcs, cfg->max_tcs) && halloc(c, s.h_usages, cfg->max_usages) && halloc(c, s.h_text, cfg->text_arena_bytes);
        ok = ok && halloc(c, s.h_runs, cfg->max_runs) && halloc(c, s.h_segres, cfg->max_segs) && halloc(c, s.h_ctr, 1);
        ok = ok && dalloc(c, s.d_segs, cfg->max_segs);
        ok = ok && dalloc(c, s.d_out, (size_t)in_base_of(*cfg) + cfg->in_arena_bytes + 16);
        if (ok) s.d_in = s.d_out + in_base_of(*cfg);
        // recs[max_recs]: the sink record of the empty work items a deferred allocation leaves (SSE_FLAG_DEFER), never returned
        ok = ok && dalloc(c, s.d_frames, cfg->max_frames) && dalloc(c, s.d_recs, (size_t)cfg->max_recs + 1);
        s.cap_tcs = cfg->max_tcs; s.cap_usages = cfg->max_usages; s.cap_text = cfg->text_arena_bytes;
        ok = ok && dalloc(c, s.d_tcs, cfg->max_tcs) && dalloc(c, s.d_usages, cfg->max_usages) && dalloc(c, s.d_text, cfg->text_arena_bytes);
        ok = ok && dalloc(c, s.d_runs, cfg->max_runs) && dalloc(c, s.d_segres, cfg->max_segs) && dalloc(c, s.d_ctr, 1);
        ok = ok && dalloc(c, s.d_items, cfg->max_recs) && dalloc(c, s.d_segterm, cfg->max_segs);
        ok = ok && dalloc(c, s.d_items2, cfg->max_recs);
        ok = ok && dalloc(c, s.d_tiles, (size_t)cfg->max_segs + 64);
        if (ok && (cfg->flags & SSE_FLAG_COUNTERS))
            ok = dalloc(c, s.d_cnt, CN_COUNT) && halloc(c, s.h_cnt, CN_COUNT) && cu_ok(cudaMemset(s.d_cnt, 0, CN_COUNT * sizeof(unsigned long long)), "cudaMemset");
    }
    if (!ok) { sse_destroy(c); return SSE_ERR_CUDA; }
    *out = c;
    return SSE_OK;
}

void sse_destroy(sse_ctx *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    free_retired(c, true);
    for (auto &s : c->slots) free_slot(s);
    cudaFree(c->d_conns); cudaFree(c->d_carry); cudaFree(c->d_tcache);
    cudaFree(c->d_pool); cudaFree(c->d_pool_hdr); cudaFree(c->d_pool_stack); cudaFree(c->d_pool_next); cudaFree(c->d_pool_chain);
    cudaFreeHost(c->h_pool_hdr);
    if (c->ctl_stream) cudaStreamDestroy(c->ctl_stream);
    if (c->last_kernel) cudaEventDestroy(c->last_kernel);
    delete c;
}

int sse_acquire(sse_ctx *c, int *slot, sse_batch *batch) {
    if (!c || !slot || !batch) return SSE_ERR_ARG;
    for (size_t i = 0; i < c->slots.size(); i++) {
        if (c->slots[i].state == SLOT_FREE) {
            Slot &s = c->slots[i];
            s.state = SLOT_ACQUIRED;
            *slot = (int)i;
            batch->in_arena = s.h_in; batch->segs = s.h_segs;
            batch->in_arena_bytes = c->cfg.in_arena_bytes; batch->max_segs = c->cfg.max_segs;
            return SSE_OK;
        }
    }
    return SSE_ERR_BUSY;
}

int sse_submit(sse_ctx *c, int slot, uint32_t n_segs, uint32_t in_bytes) {
    if (!c || slot < 0 || slot >= (int)c->slots.size()) return SSE_ERR_ARG;
    Slot &s = c->slots[slot];
    if (s.state != SLOT_ACQUIRED) return SSE_ERR_BUSY;
    int rc = validate_segs(c, s, n_segs, in_bytes);
    if (rc != SSE_OK) return rc;
    CU(cudaSetDevice(c->device));
    rc = do_upload(c, s, n_segs, in_bytes, s.stream);
    if (rc != SSE_OK) return rc;
    if (c->have_last) CU(cudaStreamWaitEvent(s.stream, c->last_kernel, 0));   // per-connection FIFO across batches
    rc = do_launch(c, s, n_segs, s.stream);
    if (rc != SSE_OK) return rc;
    CU(cudaEventRecord(c->last_kernel, s.stream));
    c->have_last = true;
    // the counters sse_collect reads first travel now, so that a slot sse_poll reports done is one copy away from its result
    CU(cudaMemcpyAsync(s.h_ctr, s.d_ctr, offsetof(Counters, class_count), cudaMemcpyDeviceToHost, s.stream));
    CU(cudaEventRecord(s.kernel_done, s.stream));
    s.ctr_queued = true;
    s.state = SLOT_SUBMITTED;
    return SSE_OK;
}

int sse_poll(sse_ctx *c, int slot) {
    if (!c || slot < 0 || slot >= (int)c->slots.size()) return SSE_ERR_ARG;
    Slot &s = c->slots[slot];
    if (s.state != SLOT_SUBMITTED) return SSE_ERR_BUSY;
    CU(cudaSetDevice(c->device));
    const cudaError_t e = cudaEventQuery(s.kernel_done);
    if (e == cudaErrorNotReady) return 0;
    CU(e);
    return 1;
}

int sse_collect(sse_ctx *c, int slot, sse_result *res) {
    if (!c || !res || slot < 0 || slot >= (int)c->slots.size()) return SSE_ERR_ARG;
    Slot &s = c->slots[slot];
    if (s.state != SLOT_SUBMITTED) return SSE_ERR_BUSY;
    CU(cudaSetDevice(c->device));
    int rc = do_download(c, s, res, s.stream);
    s.state = SLOT_COLLECTED;
    // a batch launched before the last growth measured its lack against the smaller pool: its lines try the grown one first
    if (rc == SSE_OK && (res->overflow & SSE_OVF_POOL) && s.pool_gen == c->pool_gen) rc = grow_pool(c, s.pool_short);
    else if (!c->retired.empty()) free_retired(c, false);
    return rc;
}

int sse_release(sse_ctx *c, int slot) {
    if (!c || slot < 0 || slot >= (int)c->slots.size()) return SSE_ERR_ARG;
    Slot &s = c->slots[slot];
    if (s.state == SLOT_SUBMITTED) { CU(cudaSetDevice(c->device)); CU(cudaStreamSynchronize(s.stream)); }
    s.state = SLOT_FREE;
    s.cnt_ready = false;
    s.ctr_queued = false;
    if (s.trim) { CU(cudaSetDevice(c->device)); return trim_arenas(c, s); }
    return SSE_OK;
}

int sse_trim(sse_ctx *c, uint32_t min_pool_pages) {
    if (!c || !(c->cfg.flags & SSE_FLAG_DEFER) || min_pool_pages == SSE_NONE) return SSE_ERR_ARG;
    CU(cudaSetDevice(c->device));
    if (c->have_last) CU(cudaStreamWaitEvent(c->ctl_stream, c->last_kernel, 0));
    CU(cudaStreamSynchronize(c->ctl_stream));
    int rc = SSE_OK;
    if (c->pool.pool_pages && c->pool_max) rc = trim_pool(c, min_pool_pages);
    // a slot that holds a batch may still lend its results (or a device-resident download) to the caller: sse_release trims it
    for (Slot &s : c->slots) {
        s.trim = true;
        if (s.state == SLOT_FREE) {
            const int r = trim_arenas(c, s);
            if (rc == SSE_OK) rc = r;
        }
    }
    return rc;
}

int sse_memory_held(sse_ctx *c, uint64_t *device_bytes, uint64_t *pinned_bytes) {
    if (!c || !device_bytes || !pinned_bytes) return SSE_ERR_ARG;
    *device_bytes = c->device_bytes;
    *pinned_bytes = c->pinned_bytes;
    return SSE_OK;
}

int sse_reset_conn(sse_ctx *c, uint32_t conn) {
    if (!c || conn >= c->cfg.max_conns) return SSE_ERR_ARG;
    CU(cudaSetDevice(c->device));
    if (c->have_last) CU(cudaStreamWaitEvent(c->ctl_stream, c->last_kernel, 0));
    if (c->pool.pool_pages) {   // the connection's pages go back to the pool with its state
        if (!cu_ok((cudaError_t)sse_launch_pool_reset(pool_params(c), conn, c->ctl_stream), "pool reset kernel")) return SSE_ERR_CUDA;
    } else CU(cudaMemsetAsync(c->d_conns + conn, 0, sizeof(ConnState), c->ctl_stream));
    CU(cudaEventRecord(c->last_kernel, c->ctl_stream));   // later kernels are ordered after the reset
    c->have_last = true;
    return SSE_OK;
}

int sse_reset_all(sse_ctx *c, void *cuda_stream) {
    if (!c) return SSE_ERR_ARG;
    CU(cudaSetDevice(c->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : c->ctl_stream;
    if (!cuda_stream && c->have_last) CU(cudaStreamWaitEvent(st, c->last_kernel, 0));
    CU(cudaMemsetAsync(c->d_conns, 0, (size_t)c->cfg.max_conns * sizeof(ConnState), st));
    if (c->pool.pool_pages && !cu_ok((cudaError_t)sse_launch_pool_reset(pool_params(c), SSE_NONE, st), "pool reset kernel")) return SSE_ERR_CUDA;
    if (!cuda_stream) { CU(cudaEventRecord(c->last_kernel, st)); c->have_last = true; }
    return SSE_OK;
}

int sse_line_pool_stats(sse_ctx *c, uint32_t *pages_in_use, uint32_t *pages_high_water) {
    if (!c || !pages_in_use || !pages_high_water) return SSE_ERR_ARG;
    *pages_in_use = *pages_high_water = 0;
    if (!c->pool.pool_pages) return SSE_OK;
    CU(cudaSetDevice(c->device));
    if (c->have_last) CU(cudaStreamWaitEvent(c->ctl_stream, c->last_kernel, 0));
    CU(cudaMemcpyAsync(c->h_pool_hdr, c->d_pool_hdr, sizeof(PoolHdr), cudaMemcpyDeviceToHost, c->ctl_stream));
    CU(cudaStreamSynchronize(c->ctl_stream));
    *pages_in_use = c->pool.pool_pages - c->h_pool_hdr->n_free;
    *pages_high_water = c->h_pool_hdr->high_water;
    return SSE_OK;
}

int sse_line_pool_set_growth(sse_ctx *c, uint32_t max_pages) {
    if (!c || !c->pool.pool_pages || !(c->cfg.flags & SSE_FLAG_DEFER) || max_pages == SSE_NONE ||
        (max_pages && max_pages < c->pool.pool_pages)) return SSE_ERR_ARG;
    CU(cudaSetDevice(c->device));
    c->pool_max = max_pages;
    if (c->have_last) CU(cudaStreamWaitEvent(c->ctl_stream, c->last_kernel, 0));
    CU(cudaMemsetAsync(&c->d_pool_hdr->grow, max_pages > c->pool.pool_pages ? 1 : 0, sizeof(uint32_t), c->ctl_stream));
    CU(cudaEventRecord(c->last_kernel, c->ctl_stream));   // later kernels see the new setting
    c->have_last = true;
    return SSE_OK;
}

int sse_line_pool_capacity(sse_ctx *c, uint32_t *pages, uint32_t *max_pages) {
    if (!c || !pages || !max_pages) return SSE_ERR_ARG;
    *pages = c->pool.pool_pages;
    *max_pages = c->pool_max;
    return SSE_OK;
}

int sse_upload(sse_ctx *c, int slot, uint32_t n_segs, uint32_t in_bytes, void *cuda_stream) {
    if (!c || slot < 0 || slot >= (int)c->slots.size()) return SSE_ERR_ARG;
    Slot &s = c->slots[slot];
    if (s.state != SLOT_ACQUIRED) return SSE_ERR_BUSY;
    int rc = validate_segs(c, s, n_segs, in_bytes);
    if (rc != SSE_OK) return rc;
    CU(cudaSetDevice(c->device));
    return do_upload(c, s, n_segs, in_bytes, cuda_stream ? (cudaStream_t)cuda_stream : s.stream);
}

int sse_launch(sse_ctx *c, int slot, uint32_t n_segs, void *cuda_stream) {
    if (!c || slot < 0 || slot >= (int)c->slots.size()) return SSE_ERR_ARG;
    Slot &s = c->slots[slot];
    if (s.state != SLOT_ACQUIRED || n_segs > c->cfg.max_segs) return SSE_ERR_BUSY;
    CU(cudaSetDevice(c->device));
    return do_launch(c, s, n_segs, cuda_stream ? (cudaStream_t)cuda_stream : s.stream);
}

int sse_download(sse_ctx *c, int slot, sse_result *res, void *cuda_stream) {
    if (!c || !res || slot < 0 || slot >= (int)c->slots.size()) return SSE_ERR_ARG;
    Slot &s = c->slots[slot];
    if (s.state != SLOT_ACQUIRED) return SSE_ERR_BUSY;
    CU(cudaSetDevice(c->device));
    return do_download(c, s, res, cuda_stream ? (cudaStream_t)cuda_stream : s.stream);
}

/* debugging aid (tools/dump_templates.py): the fused kernel's template cache, as sse_fused.cu lays it out */
int sse_debug_tcache(sse_ctx *c, uint32_t *out, uint32_t words) {
    if (!c || !out || !c->d_tcache) return SSE_ERR_ARG;
    CU(cudaSetDevice(c->device));
    CU(cudaDeviceSynchronize());
    const uint32_t n = words < sse_fused_tcache_words() ? words : sse_fused_tcache_words();
    CU(cudaMemcpy(out, c->d_tcache, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    return (int)n;
}

int sse_counters_read(sse_ctx *c, int slot, sse_counters *out) {
    if (!c || !out || out->struct_size != sizeof(sse_counters) || !(c->cfg.flags & SSE_FLAG_COUNTERS) || slot < 0 ||
        slot >= (int)c->slots.size()) return SSE_ERR_ARG;
    const Slot &s = c->slots[slot];
    if ((s.state != SLOT_COLLECTED && s.state != SLOT_ACQUIRED) || !s.cnt_ready) return SSE_ERR_BUSY;
    out->decode_passes = s.decode_passes;
    memcpy(&out->p_segments, s.h_cnt, CN_COUNT * sizeof(uint64_t));
    return SSE_OK;
}

int sse_launch_count(sse_ctx *c, uint64_t *kernel_launches) {
    if (!c || !kernel_launches) return SSE_ERR_ARG;
    *kernel_launches = c->launches;
    return SSE_OK;
}

} // extern "C"
