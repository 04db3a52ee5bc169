/*
 * sse_gpu.h -- C ABI of libssegpu.so: the H100 (sm_90a) implementation of inference-gateway's
 * streaming-response hot path.  This is the drop-in boundary: the Go side (integration/go, see
 * INTEGRATION.md) binds exactly these symbols through cgo and keeps core.IProvider /
 * registry.ProviderRegistry unchanged above them.
 *
 * What each entry point replaces in the reference (paths relative to the reference root):
 *   sse_submit/sse_collect   the per-line work of ProviderImpl.StreamChatCompletions' reader goroutine
 *                            (providers/core/provider.go:308-341: ReadBytes('\n'), tail held back),
 *                            the verbatim writers (api/routes.go:600-625, :178-231) [mode P], and the
 *                            MCP agent's per-line trim / [DONE] / "data: " / reframe / json.Unmarshal /
 *                            early-termination loop (mcp/agent.go:169-248) [mode R]
 *   sse_rec / sse_tc / sse_usage   the decoded fields of types.CreateChatCompletionStreamResponse that
 *                            the reference consumes (providers/types/common_types.go:271-297,:300-346,
 *                            :384-393,:451-478), i.e. what agent.go:199-242, agent.go:377-481 and
 *                            api/middlewares/telemetry.go:190-277 read after json.Unmarshal
 *   sse_reset_conn           a new upstream stream on the slot (new ProviderImpl per request,
 *                            providers/registry/registry.go:58-69; next agent iteration, agent.go:145-148)
 *   sse_agent_* / sse_telemetry_*  host-side folds of the records that reproduce the accumulators of
 *                            agent.go:156-260 (+ :377-481) and telemetry.go:190-277
 *
 * Conventions: every function returns 0 (SSE_OK) or a negative sse_status; nothing throws across the
 * ABI; every buffer handed to the caller is allocated by the library (cudaHostAlloc) and stays valid
 * until sse_release()/sse_destroy(); the library never retains caller pointers.  There is NO CPU
 * fallback: without a CUDA device sse_init fails with SSE_ERR_NO_DEVICE.  Contexts share no state: different contexts, on
 * the same device or on different ones, may be created, driven and destroyed on different threads at the same time; one
 * context is driven by one thread at a time.
 */
#ifndef SSE_GPU_H
#define SSE_GPU_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SSE_ABI_VERSION 2

typedef enum {
    SSE_OK = 0,
    SSE_ERR_NO_DEVICE = -1,   /* no CUDA device / driver: the product path has no CPU fallback */
    SSE_ERR_CUDA = -2,        /* a CUDA call failed; sse_last_cuda_error() has the text */
    SSE_ERR_ARG = -3,
    SSE_ERR_BUSY = -4,        /* no free batch slot / slot in wrong state */
    SSE_ERR_OVERFLOW = -5,    /* a result arena was too small for this batch (config too small); never with SSE_FLAG_DEFER */
    SSE_ERR_NOMEM = -6,
    SSE_ERR_UNDECODED = -7    /* sse_agent_feed / sse_telemetry_feed: the segment holds a record flagged SSE_F_TOO_LONG or SSE_F_DEPTH_LIMIT, i.e. a
                                 line the reference would have decoded and this library did not: the fold took the rest, the caller must
                                 fail the stream (or decode that frame itself) instead of trusting the accumulators */
} sse_status;

/* segment modes (per connection, chosen by which reference consumer sits above the provider) */
#define SSE_MODE_P     0u  /* passthrough: every complete line verbatim (routes.go:613, :220) */
#define SSE_MODE_R     1u  /* MCP reframe "data: "+payload+"\n\n" with agent.go:178-242 rules; implies PARSE */
#define SSE_MODE_PARSE 2u  /* decode payloads of lines that start with "data: " into sse_rec (telemetry tap) */

typedef struct {
    uint32_t struct_size;      /* sizeof(sse_config), for ABI evolution */
    uint32_t max_conns;        /* connection slots [0, max_conns) with persistent carry state */
    uint32_t max_segs;         /* segments per batch (at most one per connection per batch) */
    uint32_t in_arena_bytes;   /* input bytes per batch */
    uint32_t out_arena_bytes;  /* emitted bytes per batch */
    uint32_t max_frames;       /* emitted frames per batch */
    uint32_t max_recs;         /* parsed lines per batch */
    uint32_t max_tcs;          /* tool-call elements per batch */
    uint32_t max_usages;       /* usage objects per batch */
    uint32_t text_arena_bytes; /* decoded (unescaped) strings per batch */
    uint32_t max_runs;         /* extra result runs per batch (segments with > 64 lines) */
    uint32_t carry_slot_bytes; /* per-connection held-back tail capacity == longest line without a line pool (sse_init_ex) */
    uint32_t n_slots;          /* batches in flight (pipeline depth), 1..8 */
    uint32_t flags;            /* SSE_FLAG_* */
} sse_config;

#define SSE_FLAG_KERNEL_FUSED 4u /* single-pass tile kernel (1-D TMA staging, stop bitmap, warp-per-line template replay): reads the payload from HBM
                                    once; slower than the default pipeline on H100 (DESIGN.md 4.3) */
#define SSE_FLAG_TEMPLATES 16u /* skeleton-template replay: lines whose JSON skeleton was seen before skip the automaton (results identical;
                                  on H100 slower than the automaton alone in most measured shapes, faster in two, DESIGN.md 4.3,
                                  so off by default) */
#define SSE_FLAG_COPY_OUT 8u   /* materialise every frame in the out arena. Default: a frame whose bytes already stand in the
                                  caller's input arena exactly as the reference would send them (every mode P line, and a mode R
                                  "data: ...\n" line followed by a blank line) is returned as a span of the input arena and is
                                  neither copied on the device nor sent back over PCIe (see sse_at) */
#define SSE_FLAG_DEFER 64u     /* a batch whose results do not fit the config's capacities is not failed (SSE_ERR_OVERFLOW never happens):
                                  - out bytes / frames / records / runs: a segment stops at the start of the round of lines that does not
                                    fit; its connection state describes exactly the bytes before that point, the segment is flagged
                                    SSE_SEG_DEFERRED and sse_seg_result.consumed tells how many of its bytes the batch took. The caller
                                    submits the rest (in[consumed:]) for that connection in a later batch, before any newer bytes.
                                  - tool calls / usages / decoded text: sse_collect grows the slot's arenas and decodes the batch again
                                    (they stay grown until sse_trim).
                                  sse_result.overflow reports the SSE_OVF_* bits of what was deferred or grown. Not with SSE_FLAG_KERNEL_FUSED.
                                  - line-pool pages, on a context with a pool growth limit (sse_line_pool_set_growth) above its capacity:
                                    a line that needs a page when none is free stops its segment at the byte that needed it (deferred
                                    as above, the connection keeps the pages it holds) and sse_collect grows the pool (SSE_OVF_POOL).
                                  With batches in flight (n_slots > 1): a deferred rest must reach the connection before its newer bytes,
                                  so produce-side deferral is only safe while each connection is in at most one uncollected batch. Growing
                                  the decode arenas has no such limit: the batch is decoded again behind whatever was submitted since. */
#define SSE_FLAG_COUNTERS 256u /* run counting instantiations of the produce, decode and finalize kernels and keep a block of counters per
                                  slot (sse_counters_read): what the kernels did for the batch. Results are identical; the counting
                                  kernels are slower (DESIGN.md 4.3). Not with SSE_FLAG_KERNEL_FUSED. */

/* One segment = the bytes read from ONE connection since the previous batch. in_off is 16-byte aligned. */
typedef struct {
    uint32_t conn;
    uint32_t in_off;
    uint32_t in_len;
    uint8_t  mode;             /* SSE_MODE_* bits */
    uint8_t  provider;         /* remap-table selector; all 11 reference providers are identity (SURVEY 0) */
    uint16_t reserved;
} sse_seg;

/* An emitted frame: one element of the reference's chan []byte. `off` is an arena offset: below sse_result.in_base it
 * indexes sse_result.out, at or above it indexes the batch's own input arena (off - in_base); use sse_at(). The same
 * holds for every span in sse_rec / sse_tc that is not flagged *_TEXT. */
typedef struct { uint32_t off, len; } sse_frame;

/* sse_rec.flags */
#define SSE_F_JSON_OK        0x0001u /* json.Unmarshal returned nil (syntax valid, no type mismatch) */
#define SSE_F_HAS_USAGE      0x0002u /* resp.Usage != nil */
#define SSE_F_TC_NONNIL      0x0004u /* choices[0].delta.tool_calls != nil */
#define SSE_F_TC_VALID       0x0008u /* agent.go:224-233 predicate true for some element */
#define SSE_F_CONTENT_TEXT   0x0010u /* content span is in the text arena (needed unescaping), else an arena offset (sse_at) */
#define SSE_F_DONE_LINE      0x0020u /* mode R: line contained "[DONE]" and was swallowed (agent.go:181-184) */
#define SSE_F_DONE_EXACT     0x0040u /* ... and its payload is exactly "[DONE]" (agent.go:394-396 break) */
#define SSE_F_TERMINATES     0x0080u /* mode R: finish_reason stop/tool_calls on an emitted chunk (agent.go:235-242) */
#define SSE_F_DEPTH_LIMIT    0x0100u /* nesting deeper than 128: reported as not JSON_OK (documented limit) */
#define SSE_F_TOO_LONG       0x0200u /* line longer than the parse window: frame exact, side-band not decoded */
#define SSE_F_FINISH_SHIFT   12      /* bits 12..14: SSE_FIN_* of choices[0].finish_reason */
#define SSE_F_FINISH_MASK    0x7000u
enum { SSE_FIN_NONE = 0, SSE_FIN_STOP = 1, SSE_FIN_TOOL_CALLS = 2, SSE_FIN_LENGTH = 3,
       SSE_FIN_CONTENT_FILTER = 4, SSE_FIN_FUNCTION_CALL = 5, SSE_FIN_OTHER = 7 };

#define SSE_NONE 0xFFFFFFFFu

/* One record per line whose payload was decoded. 32 bytes. */
typedef struct {
    uint32_t frame;        /* index into frames[] of the emitted frame, SSE_NONE if not emitted */
    uint32_t flags;        /* SSE_F_* */
    uint32_t content_off;  /* decoded choices[0].delta.content */
    uint32_t content_len;
    uint32_t tc_first;     /* first tool-call element (linked through sse_tc.next), SSE_NONE if none */
    uint16_t tc_count;     /* len(*choices[0].delta.tool_calls), saturating */
    uint16_t n_choices;    /* len(resp.Choices), saturating */
    uint32_t usage;        /* index into usages[], SSE_NONE if resp.Usage == nil */
    uint32_t payload_len;  /* bytes handed to json.Unmarshal */
} sse_rec;

/* sse_tc.flags */
#define SSE_TC_HAS_ID    0x01u
#define SSE_TC_HAS_TYPE  0x02u
#define SSE_TC_HAS_FUNC  0x04u
#define SSE_TC_ID_TEXT   0x10u   /* span is in the text arena (else an arena offset, sse_at) */
#define SSE_TC_TYPE_TEXT 0x20u
#define SSE_TC_NAME_TEXT 0x40u
#define SSE_TC_ARGS_TEXT 0x80u

/* One element of choices[0].delta.tool_calls (ChatCompletionMessageToolCallChunk). 48 bytes. */
typedef struct {
    int64_t  index;
    uint32_t flags;
    uint32_t next;         /* next element of the same chunk, SSE_NONE at the end */
    uint32_t id_off, id_len, type_off, type_len, name_off, name_len, args_off, args_len;
} sse_tc;

typedef struct { int64_t prompt_tokens, completion_tokens, total_tokens; } sse_usage;

/* sse_seg_result.flags */
#define SSE_SEG_TERMINATED   0x01u  /* a chunk with SSE_F_TERMINATES was emitted in this batch */
#define SSE_SEG_FINISHED     0x02u  /* connection had terminated earlier: bytes ignored (never read by the reference) */
#define SSE_SEG_LINE_TOO_LONG 0x04u /* a line exceeded carry_slot_bytes and could not continue in the line pool (longer than
                                       max_line_bytes, or no free page): stream failed, connection dead until reset */
#define SSE_SEG_DEAD         0x08u  /* connection is in the failed state */
#define SSE_SEG_DEFERRED     0x10u  /* SSE_FLAG_DEFER: the result arenas (or a growable line pool) were full: only the first `consumed` bytes were taken */

/* A run: contiguous frames/recs produced by up to 64 consecutive lines of one segment. */
typedef struct {
    uint32_t frame_first, frame_count;
    uint32_t rec_first, rec_count;
    uint32_t next;         /* next run of the same segment in runs[], SSE_NONE at the end */
} sse_run;

/* Per-segment result, same index as the submitted sse_seg. 32 bytes. */
typedef struct {
    sse_run  run;          /* first run inline */
    uint32_t carry_len;    /* bytes held back (unterminated tail), carried to the next batch: carry slot plus line pool */
    uint32_t flags;        /* SSE_SEG_* */
    uint32_t consumed;     /* this segment's input bytes the batch took: in_len unless SSE_SEG_DEFERRED (then resubmit in[consumed:]).
                              A line that continues in the carry slot or line pool counts as taken; a deferred line does not */
} sse_seg_result;

typedef struct {
    int32_t  status;       /* SSE_OK or SSE_ERR_OVERFLOW */
    uint32_t n_segs, n_frames, n_recs, n_tcs, n_usages, n_runs;
    uint32_t out_bytes, text_bytes;
    const uint8_t        *out;      /* emitted bytes that had to be materialised (reframed, carried over or assembled lines) */
    const sse_frame      *frames;
    const sse_rec        *recs;
    const sse_tc         *tcs;
    const sse_usage      *usages;
    const uint8_t        *text;     /* decoded strings */
    const sse_run        *runs;
    const sse_seg_result *segs;
    uint32_t n_decoded, n_derived;  /* statistics: lines decoded by the automaton; n_derived is reserved (0) */
    uint32_t overflow;              /* SSE_OVF_* bits: status == SSE_ERR_OVERFLOW: which sse_config capacity to raise; with
                                       SSE_FLAG_DEFER (status SSE_OK): what this batch deferred (OUT, RUNS, POOL) or grew and decoded
                                       again (TCS, USAGES, TEXT); 0 when everything fit */
    uint32_t in_base;               /* arena offsets >= in_base refer to in[off - in_base] */
    const uint8_t *in;              /* the batch's input arena (sse_batch.in_arena), lent until sse_release like out */
} sse_result;

/* Resolve an arena offset (frame.off, content_off, tool-call spans without the *_TEXT flag):
 * off >= r->in_base ? r->in + (off - r->in_base) : r->out + off. */
const uint8_t *sse_at(const sse_result *r, uint32_t off);

#define SSE_OVF_OUT    0x01u  /* out_arena_bytes / max_frames / max_recs / work items (bump-allocated together per round) */
#define SSE_OVF_TCS    0x02u  /* max_tcs */
#define SSE_OVF_USAGES 0x04u  /* max_usages */
#define SSE_OVF_TEXT   0x08u  /* text_arena_bytes */
#define SSE_OVF_RUNS   0x10u  /* max_runs */
#define SSE_OVF_POOL   0x20u  /* line-pool pages (SSE_FLAG_DEFER with pool growth): lines deferred for want of a free page; sse_collect
                                 grew the pool after the batch, up to the limit of sse_line_pool_set_growth */

typedef struct {
    uint8_t *in_arena;     /* pinned; caller writes each segment's bytes at a 16-byte aligned in_off */
    sse_seg *segs;         /* pinned; caller writes descriptors */
    uint32_t in_arena_bytes, max_segs;
} sse_batch;

typedef struct sse_ctx sse_ctx;

/* lifecycle */
int  sse_init(int device, const sse_config *cfg, sse_ctx **out);
void sse_destroy(sse_ctx *ctx);
const char *sse_strerror(int status);
const char *sse_last_cuda_error(void);
int  sse_abi_version(void);
void sse_default_config(sse_config *cfg, uint32_t max_conns, uint32_t bytes_per_batch);
/* Capacities under which NO input can overflow a result arena (a batch of bytes_per_batch bytes on max_conns connections):
 * memory grows to ~48x the batch size plus ~1.4 MB per connection (every connection may complete a line of its whole carry
 * slot, whose payload the decode stage reads beyond the batch's input), meant for small batcher arenas (sse_gateway.h uses it). With sse_default_config the
 * capacities fit realistic SSE traffic and a pathological batch fails as a whole with SSE_ERR_OVERFLOW, unless the context
 * runs with SSE_FLAG_DEFER (then what does not fit waits for the next batch, or the decode arenas grow). */
void sse_worst_case_config(sse_config *cfg, uint32_t max_conns, uint32_t bytes_per_batch);

/* Line pool: pages in HBM shared by all connections of a context. A line that outgrows its connection's carry slot
 * continues in pool pages instead of failing the stream; its pages return to the pool when the line completes, when the
 * connection dies or finishes, and on sse_reset_conn / sse_reset_all. A connection fails (SSE_SEG_LINE_TOO_LONG |
 * SSE_SEG_DEAD) only when its line would exceed max_line_bytes or no page is free (with SSE_FLAG_DEFER and a growth limit
 * above the pool's capacity, a line that finds no free page waits for the pool to grow instead: sse_line_pool_set_growth).
 * A completed pooled line is always
 * materialised in the out arena (never a zero-copy span). A payload of 32 KiB or more is decoded by a whole warp (a context
 * whose longest line, max_line_bytes here or carry_slot_bytes without a pool, is at least that long runs one more kernel per
 * batch, which sse_launch_count counts). Not available with SSE_FLAG_KERNEL_FUSED. */
#define SSE_MAX_LINE_BYTES 16777215u   /* decode work items carry a 24-bit payload length */
typedef struct {
    uint32_t struct_size;      /* sizeof(sse_line_pool) */
    uint32_t page_bytes;       /* pool page size, multiple of 16; 0 = library default (64 KiB) */
    uint32_t pool_pages;       /* pages shared by all connections for lines longer than carry_slot_bytes; 0 = no pool */
    uint32_t max_line_bytes;   /* longest line ONE connection may assemble (carry_slot_bytes .. SSE_MAX_LINE_BYTES): no upstream can take the whole pool */
} sse_line_pool;
/* sse_init with a line pool (pool NULL == sse_init). The per-batch result capacities grow as sse_line_pool_config says. */
int  sse_init_ex(int device, const sse_config *cfg, const sse_line_pool *pool, sse_ctx **out);
/* The capacities sse_init_ex will actually allocate: up to pool_pages * page_bytes bytes of pooled lines can complete in one
 * batch, so out, frames, recs, tcs, usages, text and runs each grow by that many bytes at the ratio to in_arena_bytes the
 * config already has (a worst-case config stays overflow-free, a default one stays sized for realistic traffic). A NULL or
 * zero-page pool leaves cfg unchanged. */
void sse_line_pool_config(sse_config *cfg, const sse_line_pool *pool);
/* Pages held by connections now and the most ever held at once; ordered after already submitted batches and resets. The
 * high-water mark is never lowered, so after sse_trim it may exceed the pool's capacity. */
int  sse_line_pool_stats(sse_ctx *ctx, uint32_t *pages_in_use, uint32_t *pages_high_water);
/* Pool growth (SSE_FLAG_DEFER contexts with a line pool): max_pages is the most pages the pool may grow to, 0 = never grow (the
 * default). While the capacity is below the limit, a line that needs a page when none is free does not fail its connection: its
 * segment is deferred at the byte that needed the page (SSE_SEG_DEFERRED, consumed counts the bytes before it; the connection
 * keeps the pages it holds) and the batch reports SSE_OVF_POOL. sse_collect of such a batch then grows the pool to twice its
 * capacity or by the pages the batch's lines lacked, whichever is more, and never above the limit. The growth is ordered after
 * every batch already submitted; later batches use the grown pool; page ids, and so held lines, are unchanged by it; the old
 * pages are freed once no queued work can read them. At the limit a line that finds no page fails as without growth. If the
 * device cannot allocate a larger pool, the limit becomes the current capacity. The per-batch result capacities stay those of
 * the initial pool (sse_line_pool_config): a batch that completes more pooled bytes than they hold defers the rest.
 * Only sse_collect grows the pool. On the device-resident path (sse_upload / sse_launch / sse_download) a line that lacks a page
 * is deferred and its batch reports SSE_OVF_POOL as well, but the pool does not grow, so the line makes no progress there until
 * a batch through sse_submit / sse_collect grows it; a growth is queued on the context's own stream, so a caller that launches
 * on its own stream after an sse_collect synchronises first, as for any mix of the two paths.
 * SSE_ERR_ARG: no context, no pool, no SSE_FLAG_DEFER, or max_pages nonzero and below the current capacity or SSE_NONE. Ordered
 * like sse_reset_conn: after already submitted batches. */
int  sse_line_pool_set_growth(sse_ctx *ctx, uint32_t max_pages);
/* The pool's pages now (after every growth of the batches collected so far, and every sse_trim) and its growth limit (0: no growth). */
int  sse_line_pool_capacity(sse_ctx *ctx, uint32_t *pages, uint32_t *max_pages);
/* Give back what on-demand growth (SSE_FLAG_DEFER) took. Returns once the old memory is freed.
 *   Line pool (only with a growth limit: a pool without one never grew): the pool shrinks to max(min_pool_pages, pages held
 *     now, 1) pages when that is below its capacity, else it stays as it is. The held pages move to the first pages of the new
 *     pool on the device, in chain order; lines held across the trim go on byte for byte as if nothing happened, and
 *     sse_line_pool_stats' pages in use is unchanged. The pool grows again on demand, up to its limit.
 *   Decode arenas: each slot's tool-call, usage and text arenas, device and pinned, go back to the config's capacities: at once
 *     for a free slot, at its sse_release for a slot that holds a batch (its results may still be lent to the caller).
 * Ordered like sse_reset_conn: after every batch already submitted, whose completion on the device it waits for; it does not
 * collect them, and their results, which do not refer to pool pages, are collected afterwards as usual. A batch submitted
 * before the trim that reports SSE_OVF_POOL does not grow the trimmed pool (its lines try it first, as after a growth). On the
 * device-resident path (sse_upload / sse_launch / sse_download) the caller synchronises its own streams before the trim, as for
 * any mix of the two paths.
 * SSE_ERR_ARG: no context, no SSE_FLAG_DEFER, or min_pool_pages == SSE_NONE. SSE_ERR_NOMEM: the device could not allocate the
 * smaller pool (it stays as it was). */
int  sse_trim(sse_ctx *ctx, uint32_t min_pool_pages);
/* Device and pinned bytes the context holds now: every allocation, its decode tables, slots, pool and grown arenas included
 * (and a growth's old pool arrays until they are freed, at the next sse_collect or sse_trim). SSE_ERR_ARG, writing nothing,
 * for a NULL argument. */
int  sse_memory_held(sse_ctx *ctx, uint64_t *device_bytes, uint64_t *pinned_bytes);

/* pipeline: acquire -> fill -> submit -> collect -> release (one slot = one batch in flight) */
int sse_acquire(sse_ctx *ctx, int *slot, sse_batch *batch);
int sse_submit(sse_ctx *ctx, int slot, uint32_t n_segs, uint32_t in_bytes);
int sse_collect(sse_ctx *ctx, int slot, sse_result *res);
int sse_release(sse_ctx *ctx, int slot);
/* Whether a submitted batch is done, without blocking: 1 when the work sse_submit queued for the slot (its kernels and the copy
 * of its counters to the host) has completed, so that sse_collect waits only for its own result copies; 0 while it is still
 * running; SSE_ERR_BUSY when the slot is not in the submitted state; SSE_ERR_ARG for a bad context or slot; SSE_ERR_CUDA (text
 * in sse_last_cuda_error) when the device reports an error. Under SSE_FLAG_DEFER, sse_collect on a slot polled ready may still
 * run the decode stage again, when its decode arenas grow. */
int sse_poll(sse_ctx *ctx, int slot);

/* connection state */
int sse_reset_conn(sse_ctx *ctx, uint32_t conn);                 /* ordered after already submitted batches */
int sse_reset_all(sse_ctx *ctx, void *cuda_stream);              /* all connections; async on the stream (NULL: ordered
                                                                    after already submitted batches, like sse_reset_conn) */

/* device-resident replay (bench / roofline measurement): the three stages of sse_submit/sse_collect.
 * sse_upload, sse_launch, sse_download and sse_reset_all with a non-NULL stream are ordered only by the stream passed to them,
 * not with sse_submit, sse_reset_conn or sse_reset_all(NULL). A caller that mixes the two paths synchronises in between. */
int sse_upload(sse_ctx *ctx, int slot, uint32_t n_segs, uint32_t in_bytes, void *cuda_stream);
int sse_launch(sse_ctx *ctx, int slot, uint32_t n_segs, void *cuda_stream);   /* kernels only */
int sse_download(sse_ctx *ctx, int slot, sse_result *res, void *cuda_stream); /* D2H + sync */
int sse_launch_count(sse_ctx *ctx, uint64_t *kernel_launches);                /* kernels launched so far */

/* ---- SSE_FLAG_COUNTERS: what the kernels did for one batch ----
 * Sums over the batch, in this order. Lines, frames and items count what the batch's results hold; bytes are payload or
 * frame bytes. The c_* fields are clock64() cycles of the counting decode kernel summed over its warps: they show how its time
 * divides, not the time of the default kernels, which run without the counting statements. */
typedef struct {
    uint32_t struct_size;          /* sizeof(sse_counters) */
    uint32_t decode_passes;        /* decode launches behind the records (SSE_FLAG_DEFER: 1 + passes after the arenas grew) */
    /* produce stage (and the finalize stage's page returns) */
    uint64_t p_segments;           /* segments the produce kernel took a ticket for */
    uint64_t p_segments_skipped;   /* segments of finished or dead connections (bytes not read) */
    uint64_t p_windows;            /* windows staged into shared memory */
    uint64_t p_window_bytes;       /* their bytes: carried tail plus segment bytes */
    uint64_t p_rounds;             /* line rounds (each round's allocation) */
    uint64_t p_lines;              /* complete lines ('\n' found) */
    uint64_t p_frames_zero_copy;   /* frames returned as spans of the input arena */
    uint64_t p_frames_materialised;/* frames written to the out arena */
    uint64_t p_bytes_materialised; /* their lengths (without alignment padding) */
    uint64_t p_items;              /* decode work items written */
    uint64_t p_long_lines;         /* lines completed outside the window (carry slot or line pool) */
    uint64_t p_pool_pages_taken;   /* line-pool pages taken */
    uint64_t p_pool_pages_returned;/* line-pool pages returned (completed, failed or finished lines) */
    uint64_t p_deferred_rounds;    /* SSE_FLAG_DEFER: rounds that did not fit and were left for a later batch */
    /* decode stage: the pass whose records the batch returns */
    uint64_t d_items;              /* work items decoded */
    uint64_t d_pulls;              /* pulls of work items by a warp */
    uint64_t d_items_per_pull;     /* items per pull the launch chose (8, 16 or 32; not a sum: ssegw_counters keeps the last) */
    uint64_t d_warp_rounds;        /* automaton rounds executed per warp */
    uint64_t d_busy_lane_rounds;   /* sum of the lanes busy with a line over those rounds (<= 32 * d_warp_rounds) */
    uint64_t d_skip_windows;       /* 16-byte windows a lane examined while skipping the plain bytes of strings and digit runs */
    uint64_t d_skip_bytes;         /* payload bytes those skips took */
    uint64_t d_coop_strings;       /* long strings the whole warp finished for a lane */
    uint64_t d_coop_steps;         /* 512-byte steps of the warp over them */
    uint64_t d_coop_bytes;         /* payload bytes they took */
    uint64_t d_plain_steps;        /* automaton steps without an action (one byte each) */
    uint64_t d_actions;            /* actions run (one byte each) */
    uint64_t d_action_redos;       /* extra action calls for a byte looked up again in a new state */
    uint64_t d_abandoned_bytes;    /* bytes jumped over after a syntax or depth error */
    uint64_t d_template_lines;     /* SSE_FLAG_TEMPLATES: lines retired by a template */
    uint64_t d_template_bytes;     /* their payload bytes */
    uint64_t d_template_misses;    /* lines that tried a template and went to the automaton */
    uint64_t d_unquote_jobs;       /* strings unquoted by the whole warp */
    uint64_t d_unquote_bytes;      /* their source bytes */
    uint64_t d_lines_finished;     /* records written by the decode kernel */
    uint64_t c_total;              /* cycles from a warp's first pull to its exit */
    uint64_t c_pull;               /* taking work items: ticket, item loads, template lookup */
    uint64_t c_skip;               /* skipping plain bytes lane by lane */
    uint64_t c_coop;               /* the warp finishing long strings */
    uint64_t c_steps;              /* automaton steps and actions */
    uint64_t c_finish;             /* writing records */
    uint64_t c_unquote;            /* unquoting strings with the whole warp */
} sse_counters;
/* Byte identity of a batch without SSE_F_DONE_EXACT lines (those get no work item):
 *   d_skip_bytes + d_coop_bytes + d_plain_steps + d_actions + d_abandoned_bytes + d_template_bytes == sum of sse_rec.payload_len.
 * A long line (a payload of 32 KiB or more, in a context that can hold one) is decoded by a whole warp and counted into the same
 * fields: one d_pulls and one d_items; its automaton rounds are d_warp_rounds with one busy lane; each jump of the warp over a
 * string body or digit run is one d_coop_strings, with its 512-byte d_coop_steps and d_coop_bytes (value bodies with their
 * escapes and UTF-8 sequences); every string it unquotes is one d_unquote_jobs; its cycles are in c_total and the c_* parts
 * (the jumps in c_coop).
 * Valid after a successful sse_collect or sse_download of the slot and before sse_release. SSE_ERR_ARG: the context has no
 * SSE_FLAG_COUNTERS, or out->struct_size != sizeof(sse_counters); SSE_ERR_BUSY: the slot holds no collected batch. */
int sse_counters_read(sse_ctx *ctx, int slot, sse_counters *out);

/* ---- host-side folds of the records (the reference's consumers, fed from the side-band) ---- */
typedef struct { const uint8_t *p; size_t n; } sse_bytes;
typedef struct { sse_bytes id, type, name, arguments; } sse_tool_call;

/* mcp/agent.go:156-260 for one agent iteration: content accumulator, hasToolCalls, finish, and
 * parseStreamingToolCalls (:377-481) evaluated from records instead of re-parsing the text. */
typedef struct sse_agent_fold sse_agent_fold;
sse_agent_fold *sse_agent_new(void);
void sse_agent_free(sse_agent_fold *f);
void sse_agent_reset(sse_agent_fold *f);
int  sse_agent_feed(sse_agent_fold *f, const sse_result *res, uint32_t seg_index);
sse_bytes sse_agent_content(const sse_agent_fold *f);
int  sse_agent_has_tool_calls(const sse_agent_fold *f);
int  sse_agent_terminated(const sse_agent_fold *f, int *finish);
size_t sse_agent_tool_calls(sse_agent_fold *f, sse_tool_call *calls, size_t cap);

/* api/middlewares/telemetry.go:190-277 evaluated from records of a mode P|PARSE or mode R stream. */
typedef struct sse_telemetry_fold sse_telemetry_fold;
sse_telemetry_fold *sse_telemetry_new(void);
void sse_telemetry_free(sse_telemetry_fold *f);
void sse_telemetry_reset(sse_telemetry_fold *f);
int  sse_telemetry_feed(sse_telemetry_fold *f, const sse_result *res, uint32_t seg_index);
/* Bytes the HOST writes to the client between upstream frames: ssegw_agent_recv's final "data: [DONE]\n\n" (agent.go:140-143).
 * They are part of the body telemetry.go:190-198 splits into pieces, so they move its last-4-pieces window; they are not decoded
 * (feed only frames that hold no chunk: "[DONE]", comments, error text). n must end on a '\n'. */
int  sse_telemetry_feed_bytes(sse_telemetry_fold *f, const uint8_t *bytes, size_t n);
/* The usage and the tool calls (at most cap written to calls; *n_calls is how many there are). Returns 1 when a piece was irregular
 * (DESIGN.md section 5, deviation 4), else SSE_OK. It closes the body's last piece once: called again, e.g. with a larger array,
 * it gives the same answer. Feed nothing after it. */
int  sse_telemetry_finish(sse_telemetry_fold *f, sse_usage *usage, sse_tool_call *calls, size_t cap, size_t *n_calls);

#ifdef __cplusplus
}
#endif
#endif
