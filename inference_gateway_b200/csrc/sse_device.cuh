// sse_device.cuh -- device-side data layout shared by the kernels and the host library.
//
// HBM layout (one context per GPU):
//   in      u8[in_arena_bytes]         micro-batch input: per-connection segments, 16-byte aligned
//   segs    sse_seg[max_segs]          segment descriptors (conn, in_off, in_len, mode)
//   conns   ConnState[max_conns]       persistent per-connection state (carry length, flags)
//   carry   u8[max_conns*carry_slot]   persistent held-back tail of each connection (provider.go:322
//                                      ReadBytes would keep these bytes inside bufio.Reader)
//   out, frames, recs, tcs, usages, text, runs, seg_results   per-batch results (see include/sse_gpu.h)
//   ctr     Counters                   bump allocators + work ticket, zeroed per launch
// line pool (sse_init_ex, optional; one per context):
//   pool        u8[pool_pages*page_bytes]  pages holding lines longer than the carry slot, page k = bytes [k*page_bytes, ...)
//                                          of the line in chain order
//   pool_hdr    PoolHdr                    lock + free-stack height + high-water mark + whether the pool may still grow
//   pool_stack  u32[pool_pages]            free pages: pool_stack[0 .. n_free)
//   pool_next   u32[pool_pages]            next page of the same chain
//   pool_chain  PoolChain[max_conns]       per connection: first / last page, pages held (0: none)
#pragma once
#include <cstddef>
#include <stdint.h>
#include "../../include/sse_gpu.h"

struct ConnState {
    uint32_t carry_len;    // bytes of the held-back line: in the carry slot while <= carry_slot, else all of them in pool pages
    uint32_t flags;
};
struct PoolHdr {
    uint32_t lock;         // taken by one lane around every allocation / release (pages move rarely: one per page_bytes of a long line)
    uint32_t n_free;
    uint32_t high_water;   // most pages ever held at once
    uint32_t grow;         // nonzero: the pool may still grow (sse_line_pool_set_growth, below the limit): a line of the SSE_FLAG_DEFER
                           // produce kernel that finds too few free pages defers instead of failing its connection
};
struct PoolChain {
    uint32_t first, last, n_pages, pad;
};
#define CONN_FINISHED 1u   // mode R: terminating chunk seen (agent.go:235-242); later bytes are never read
#define CONN_DEAD     2u   // line exceeded carry_slot_bytes and could not continue in the line pool
#define CONN_LONG     4u   // a line longer than the smem window is being assembled in the carry slot

#ifndef SSE_LEN_SHIFT
#define SSE_LEN_SHIFT 5
#endif
#define SSE_LEN_BUCKETS (4096 >> SSE_LEN_SHIFT)
#define SSE_N_BUCKETS (32 * SSE_LEN_BUCKETS)
struct alignas(8) Counters {
    uint32_t ticket;       // next segment to process
    uint32_t n_tcs;
    // two 8-byte pairs: the produce kernel allocates a round's output with ONE 64-bit atomicAdd per pair (low word | high word
    // << 32) instead of four 32-bit ones; every counter stays below 2^31 (capacities are 31-bit), so the low word never carries
    uint32_t out_bytes;
    uint32_t n_items;      // split pipeline: work items written by the produce kernel
    uint32_t n_frames;
    uint32_t n_recs;
    uint32_t n_usages;
    uint32_t text_bytes;
    uint32_t n_runs;
    int32_t  status;
    uint32_t item_ticket;  // split pipeline: next item batch for the decode kernel
    uint32_t n_tiles;      // fused pipeline: tiles written by the plan kernel
    uint32_t pool_short;   // SSE_FLAG_DEFER with pool growth: pages lines of this batch asked for and did not find (SSE_OVF_POOL)
    uint32_t overflow;     // SSE_OVF_* bits: which arena was too small (SSE_FLAG_DEFER: also what the produce stage deferred)
    uint32_t n_long;       // split pipeline: work items of at least KParams.long_line payload bytes (items_sorted[0, n_long))
    uint32_t long_ticket;  // split pipeline: next long item for the long-line decode kernel
    // device-only tail (the host reads the struct up to here)
    uint32_t class_count[SSE_N_BUCKETS];  // split pipeline: items per bucket (see item_bucket)
    uint32_t class_cursor[SSE_N_BUCKETS];
    uint32_t long_cursor;                 // split pipeline: next free place of a long item in items_sorted
};

// Work items whose payload is at least SSE_LONG_LINE bytes are decoded by a whole warp each (sse_long_decode_kernel) instead of
// one decode lane, in contexts that can hold a line that long (KParams.long_line). 0: no long-line stage (A/B builds only).
#ifndef SSE_LONG_LINE
#define SSE_LONG_LINE 32768
#endif
static_assert(SSE_LONG_LINE == 0 || SSE_LONG_LINE > 8192, "the long-line threshold lies above every line a produce window holds");

static_assert(offsetof(Counters, out_bytes) % 8 == 0 && offsetof(Counters, n_items) == offsetof(Counters, out_bytes) + 4 &&
              offsetof(Counters, n_frames) % 8 == 0 && offsetof(Counters, n_recs) == offsetof(Counters, n_frames) + 4,
              "the produce kernel adds to (out_bytes, n_items) and (n_frames, n_recs) with one 64-bit atomic each");

struct KParams {
    const uint8_t *in;
    const sse_seg *segs;
    uint32_t n_segs;
    uint32_t max_conns;
    ConnState *conns;
    uint8_t *carry;
    uint32_t carry_slot;
    // results
    uint8_t *out;            uint32_t cap_out;
    uint32_t in_base;        // in == out + in_base: arena offsets >= in_base are input bytes (zero-copy frames)
    sse_frame *frames;       uint32_t cap_frames;
    sse_rec *recs;           uint32_t cap_recs;
    sse_tc *tcs;             uint32_t cap_tcs;
    sse_usage *usages;       uint32_t cap_usages;
    uint8_t *text;           uint32_t cap_text;
    sse_run *runs;           uint32_t cap_runs;
    sse_seg_result *seg_results;
    Counters *ctr;
    // split pipeline (produce -> decode -> finalize)
    uint4 *items;            uint32_t cap_items;   // src, len | rmode << 31, rec, seg
    uint32_t *seg_term;                            // per segment: smallest terminating record index, SSE_NONE if none
    uint32_t flags;                                // sse_config.flags
    uint4 *items_sorted;                           // items ordered by (length bucket, shape class): the 32 lanes of a decode batch walk alike lines
    // fused pipeline (plan -> fused tile kernel)
    uint2 *tiles;            uint32_t cap_tiles;   // {first segment, segment count} per tile
    uint32_t *tcache;                              // skeleton templates kept between launches: [0] words used, [1..256] buckets, store
    // line pool (pool_pages == 0: none; max_line == carry_slot then, and every line longer than the slot fails its connection)
    uint8_t *pool;           PoolHdr *pool_hdr;
    uint32_t *pool_stack;    uint32_t *pool_next;
    PoolChain *pool_chain;
    uint32_t page_bytes, pool_pages, max_line;
    // split pipeline: payload length from which a work item goes to the long-line decode kernel (0: the context cannot hold such
    // a line, and neither the sort nor the launch has a long-line stage)
    uint32_t long_line;
    // SSE_FLAG_COUNTERS: the slot's counter block (CN_*), which selects the counting kernels; nullptr: the default kernels
    unsigned long long *cnt;
};

// SSE_FLAG_COUNTERS: the counter block of a slot, one 64-bit counter per index, in the order of the uint64_t fields of
// sse_counters (include/sse_gpu.h). The produce part is written by the produce and finalize kernels, the rest by the decode kernel.
enum : uint32_t {
    CN_P_SEGMENTS, CN_P_SEGMENTS_SKIPPED, CN_P_WINDOWS, CN_P_WINDOW_BYTES, CN_P_ROUNDS, CN_P_LINES, CN_P_FRAMES_ZERO_COPY,
    CN_P_FRAMES_MATERIALISED, CN_P_BYTES_MATERIALISED, CN_P_ITEMS, CN_P_LONG_LINES, CN_P_POOL_PAGES_TAKEN, CN_P_POOL_PAGES_RETURNED,
    CN_P_DEFERRED_ROUNDS,
    CN_D_ITEMS, CN_D_PULLS, CN_D_ITEMS_PER_PULL, CN_D_WARP_ROUNDS, CN_D_BUSY_LANE_ROUNDS, CN_D_SKIP_WINDOWS, CN_D_SKIP_BYTES,
    CN_D_COOP_STRINGS, CN_D_COOP_STEPS, CN_D_COOP_BYTES, CN_D_PLAIN_STEPS, CN_D_ACTIONS, CN_D_ACTION_REDOS, CN_D_ABANDONED_BYTES,
    CN_D_TEMPLATE_LINES, CN_D_TEMPLATE_BYTES, CN_D_TEMPLATE_MISSES, CN_D_UNQUOTE_JOBS, CN_D_UNQUOTE_BYTES, CN_D_LINES_FINISHED,
    CN_C_TOTAL, CN_C_PULL, CN_C_SKIP, CN_C_COOP, CN_C_STEPS, CN_C_FINISH, CN_C_UNQUOTE,
    CN_COUNT
};
constexpr uint32_t CN_DECODE_FIRST = CN_D_ITEMS;   // the decode part: [CN_DECODE_FIRST, CN_COUNT)
static_assert(CN_DECODE_FIRST <= 32 && CN_COUNT - CN_DECODE_FIRST <= 32, "a warp keeps one counter per lane");

#ifdef __CUDACC__
__device__ __forceinline__ void sse_overflow(Counters *c, uint32_t which) {
    atomicOr(&c->overflow, which);
    atomicExch(&c->status, (int)SSE_ERR_OVERFLOW);
}

// SSE_FLAG_COUNTERS: a warp's counters, one per lane (lane k holds counter first + k, 64-bit). add() takes a warp-uniform value
// and is called by all lanes of the warp; flush() adds them to the counter block with one atomicAdd per counter.
struct WarpTally {
    unsigned long long v;
    __device__ __forceinline__ void add(uint32_t k, unsigned long long x) { if ((threadIdx.x & 31u) == k) v += x; }
    __device__ __forceinline__ void flush(unsigned long long *first, uint32_t n) {
        const uint32_t k = threadIdx.x & 31u;
        if (k < n && v) atomicAdd(first + k, v);
    }
};
#endif

// What a context's kernels are launched with. sse_init_ex fills it once, on the context's own device: kernel attributes and
// occupancy belong to the device they were read on, so no two contexts share them.
struct LaunchState {
    int sm_count = 0;
    int produce_ctas = 0;            // split pipeline: CTAs per SM of the produce kernel the context's flags select
    int long_ctas = 0;               // split pipeline: CTAs per SM of the long-line decode kernel
    const void *tables = nullptr;    // the context's decode tables on the device: ssetab::DfaTables, or FTables for the tile kernel
    uint64_t launches = 0;           // kernels launched so far (sse_launch_count); the batch wrappers add the kernels they launch
};

// Launch setup on the current device, for a context whose sse_config.flags are `flags`: the shared-memory attribute and the
// occupancy of each kernel those flags select.
int sse_produce_prepare(LaunchState &ls, uint32_t flags);                              // sse_kernel.cu
int sse_decode_prepare(LaunchState &ls, uint32_t flags);                               // sse_kernel2.cu (with sse_long_prepare)
int sse_long_prepare(LaunchState &ls);                                                 // sse_long.cu
namespace ssetab { struct DfaTables; }
int sse_fused_prepare(const ssetab::DfaTables &D, void *image);  // the tile kernel's FTables, derived from D, into `image`; its attribute

// launch wrappers
int sse_launch_produce_kernel(const KParams &p, void *stream, LaunchState &ls);       // split pipeline, stage 1
int sse_launch_decode_finalize(const KParams &p, void *stream, LaunchState &ls);      // split pipeline, stages 2+3
int sse_launch_decode(const KParams &p, void *stream, LaunchState &ls);               // SSE_FLAG_DEFER: stage 2 again (grown arenas)
void sse_launch_long_decode(const KParams &p, void *stream, LaunchState &ls);         // split pipeline, stage 2a
int sse_launch_fused(const KParams &p, void *stream, LaunchState &ls);                // plan kernel + fused tile kernel
int sse_launch_pool_reset(const KParams &p, uint32_t conn, void *stream);              // line pool: reset one connection (SSE_NONE: all)
int sse_launch_pool_extend(const KParams &p, uint32_t old_pages, bool grow, void *stream); // line pool: pages [old_pages, pool_pages) free
// line pool trim: the held pages of p's idle pool repacked into the first `held` pages of new arrays of `pages` pages
int sse_launch_pool_repack(const KParams &p, uint8_t *pool, uint32_t *stack, uint32_t *next, uint32_t held, uint32_t pages, bool grow,
                           const LaunchState &ls, void *stream);
int sse_build_tables(ssetab::DfaTables &T);                                            // the decode tables of the schema (host)
uint32_t sse_fused_max_line(void);                                                     // longest carry_slot_bytes the fused kernel supports
uint32_t sse_fused_tables_bytes(void);                                                 // size of the tile kernel's FTables
uint32_t sse_fused_tcache_words(void);                                                 // size of KParams.tcache
