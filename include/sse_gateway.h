/*
 * sse_gateway.h -- host-side mirror of the reference's streaming interfaces, above the C ABI of sse_gpu.h
 * (implemented in inference_gateway_b200/csrc/sse_gateway.cpp, exported by libssegpu.so).
 *
 *   ssegw_stream_chat_completions   core.IProvider.StreamChatCompletions (providers/core/interfaces.go:22; provider.go:277-344)
 *   ssegw_stream_with_telemetry     the same, with the response's telemetry fold fed from the stream's records
 *                                   (api/middlewares/telemetry.go:37-54, :190-277)
 *   ssegw_upstream_write / _close   response.Body bytes / EOF-or-error (provider.go:322-330)
 *   ssegw_pump                      one tick of the per-GPU batchers (INTEGRATION.md section 2), batches in flight per context
 *   ssegw_flush                     collects every batch still in flight
 *   ssegw_recv                      `line, ok := <-streamCh` (api/routes.go:602-606, mcp/agent.go:171)
 *   ssegw_agent_recv and friends    mcp.Agent.RunWithStream for one iteration (mcp/agent.go:126-290, final [DONE] :140-143)
 *   ssegw_proxy_stream / _step    handleStreamingRequest, the raw /proxy/:provider/... stream loop (api/routes.go:129-232)
 *   ssegw_counters                  what the device did for the collected batches (SSE_FLAG_COUNTERS), for export as metrics
 *   ssegw_line_pool_growth          lets the line pools grow on demand (SSE_FLAG_DEFER) instead of failing streams when full
 *   ssegw_trim                      gives back what that growth, and the growth of the decode arenas, took
 *   ssegw_mcp_writer_step           one turn of handleMCPStreamingRequest's writer (api/middlewares/mcp.go:253-299): the
 *                                   terminal-frame rule (:261-268) and the upstream-error sniff that may set 503 (:272-280)
 */
#ifndef SSE_GATEWAY_H
#define SSE_GATEWAY_H
#include "sse_gpu.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ssegw ssegw;

ssegw *ssegw_new(int device, uint32_t max_conns, uint32_t bytes_per_batch, int *status);
/* ssegw_new with a line pool (sse_init_ex): lines longer than the 64 KiB carry slot of the worst-case config continue in the
 * pool instead of failing their stream. Elements can then be longer than a receive buffer: ssegw_recv and friends return
 * SSE_ERR_ARG with *n set to the element's length and keep it queued, so the caller can grow the buffer and call again. */
ssegw *ssegw_new_ex(int device, uint32_t max_conns, uint32_t bytes_per_batch, const sse_line_pool *pool, int *status);
/* A gateway on any config (cfg->max_conns streams), e.g. sse_default_config with SSE_FLAG_DEFER: capacities sized for realistic
 * traffic instead of the worst case, and a batch whose results do not fit them leaves the rest of a stream's bytes queued for the
 * next tick (streams with deferred bytes are offered first) instead of failing every stream of the batch. ssegw_new and
 * ssegw_new_ex use sse_worst_case_config. pool may be NULL. A bad config is refused (SSE_ERR_ARG) before a device is touched. */
ssegw *ssegw_new_cfg(int device, const sse_config *cfg, const sse_line_pool *pool, int *status);
/* One gateway over several contexts, each with up to `depth` batches in flight: the per-GPU batchers of INTEGRATION.md
 * section 2 behind one set of streams. One context is opened per entry of devices (cfg and pool for each; a device may appear
 * more than once, which gives independent contexts on one GPU), and the gateway holds n_devices * cfg->max_conns streams:
 * stream id = context index * cfg->max_conns + connection. A new stream (ssegw_stream_chat_completions, ssegw_proxy_stream)
 * goes to a free connection of the context with the fewest open streams, the lowest index on a tie, and stays there for its
 * whole life (carry state and line-pool pages are per context).
 * depth (1 .. cfg->n_slots) is how many batches a context may have uncollected. ssegw_pump then runs, per context: fill and
 * submit a batch if any stream has bytes that may go in; collect every batch sse_poll reports done, oldest first; collect the
 * oldest, blocking, while depth batches are uncollected. Frames reach the channels, the agent folds, the telemetry taps and
 * the counters at collect time, in submission order per context. At depth 1 this is ssegw_new_cfg's tick: a pump delivers
 * what it submitted.
 * Bytes leave a stream's queue when they are submitted. Without SSE_FLAG_DEFER a stream may have bytes in several uncollected
 * batches (the device keeps their order); with it, a stream is not offered again while it is in an uncollected batch, and its
 * deferred rest goes back to the front of its queue when that batch is collected. A failed batch closes its streams, and
 * later batches deliver nothing more to them; what a batch returns for a stream released since goes to nobody. An upstream
 * EOF closes the channel once no byte of the stream is queued or in an uncollected batch.
 * Bad arguments are refused with SSE_ERR_ARG before a device is touched: n_devices 0 or above 64, depth outside 1 ..
 * cfg->n_slots, and what ssegw_new_cfg refuses. */
ssegw *ssegw_new_multi(const int *devices, uint32_t n_devices, const sse_config *cfg, const sse_line_pool *pool, uint32_t depth,
                       int *status);
/* Collects every uncollected batch of every context. Returns the frames delivered, or the first negative sse_status (the
 * batches after a failed one are still collected). ssegw_free flushes before it destroys the contexts. */
int    ssegw_flush(ssegw *g);
void   ssegw_free(ssegw *g);
/* Opens a stream on a free connection (placement as in ssegw_new_multi) and resets the connection. Returns the stream id,
 * or -1 when no connection is free. */
int    ssegw_stream_chat_completions(ssegw *g, uint8_t mode);
/* The telemetry tap (api/middlewares/telemetry.go:190-277 without buffering the body): opens a stream like
 * ssegw_stream_chat_completions(g, mode) whose records also feed the caller's fold `tel`.
 *   Modes: mode must carry SSE_MODE_PARSE or SSE_MODE_R (a mode P stream has no records); otherwise, or when tel is NULL,
 *     SSE_ERR_ARG. Placement, reset and the return value are those of ssegw_stream_chat_completions: the stream id, or -1
 *     when no connection is free.
 *   One feeder at a time: a fold feeds at most one open stream. Attaching it while another stream it feeds is open returns
 *     SSE_ERR_BUSY; once that stream is released, the fold may be attached to the next one (the next agent iteration).
 *   What is fed: at collect time, the segments whose frames the gateway delivers to this stream's channel, in submission
 *     order per context at any depth. Nothing is fed after ssegw_release_stream, including what batches still in flight
 *     return for the released stream. A segment the fold cannot decode (sse_telemetry_feed returns SSE_ERR_UNDECODED: a
 *     line past the nesting limit) closes the stream, as it does for the agent fold of a mode R stream.
 *   Host-written bytes: the gateway feeds only bytes it received from upstream. What the caller writes to the client itself
 *     goes in with sse_telemetry_feed_bytes: the agent's single final "data: [DONE]\n\n" (ssegw_agent_recv synthesises one
 *     per iteration; only the last iteration's belongs in the client's body) and any error frames.
 *   Ownership: the caller creates, finishes and frees the fold (sse_telemetry_new / _finish / _free). It must outlive every
 *     stream it is attached to until that stream is released or ssegw_free runs; ssegw_free does not free it.
 *   Proxy route: ssegw_proxy_step works on any stream id, so a tapped SSE_MODE_P | SSE_MODE_PARSE stream serves the raw
 *     proxy loop too (its frames are those of mode P). Whether proxy responses are recorded is the caller's decision: the
 *     reference's path filter (telemetry.go:60-63) matches some proxy paths, e.g. /compatibility/v1/chat/completions.
 * Streams opened without a tap behave as before: a mode P | PARSE stream ignores its records and is never closed by them. */
int    ssegw_stream_with_telemetry(ssegw *g, uint8_t mode, sse_telemetry_fold *tel);
size_t ssegw_upstream_write(ssegw *g, int stream, const uint8_t *data, size_t n);
void   ssegw_upstream_close(ssegw *g, int stream);
int    ssegw_pump(ssegw *g);
int    ssegw_recv(ssegw *g, int stream, uint8_t *buf, size_t cap, size_t *n);
void   ssegw_release_stream(ssegw *g, int stream);
int    ssegw_agent_recv(ssegw *g, int stream, uint8_t *buf, size_t cap, size_t *n);
sse_bytes ssegw_agent_content(ssegw *g, int stream);
int    ssegw_agent_has_tool_calls(ssegw *g, int stream);
int    ssegw_agent_terminated(ssegw *g, int stream, int *finish);
size_t ssegw_agent_tool_calls(ssegw *g, int stream, sse_tool_call *calls, size_t cap);
/* SSE_FLAG_COUNTERS: the sse_counters of every batch this gateway has collected, on every context, added up (d_items_per_pull:
 * the last batch's), e.g. for export as monotonic counters. SSE_ERR_ARG unless the gateway was made by ssegw_new_cfg or
 * ssegw_new_multi with a config that has the flag, or when out->struct_size != sizeof(sse_counters). */
int    ssegw_counters(ssegw *g, sse_counters *out);
/* sse_line_pool_set_growth(ctx, max_pages) on every context of the gateway: a gateway made by ssegw_new_cfg or ssegw_new_multi
 * with SSE_FLAG_DEFER and a line pool lets each context's pool grow up to max_pages (0: no growth) instead of failing a stream
 * whose line finds no free page; the stream's rest waits in its queue, like any deferred rest, until the pool has grown.
 * Returns the first error (SSE_ERR_ARG: no gateway, no pool, no SSE_FLAG_DEFER, or max_pages below a pool's capacity). */
int    ssegw_line_pool_growth(ssegw *g, uint32_t max_pages);
/* sse_trim(ctx, min_pool_pages) on every context of the gateway: gives back the line-pool pages and decode arenas that growth
 * took (SSE_FLAG_DEFER), e.g. on the operator's timer after a burst. Streams holding lines go on unchanged; batches in flight are
 * waited for on the device, collected by later pumps as usual, and their slots' arenas shrink when they are released. Returns
 * the first error (SSE_ERR_ARG: no gateway, a config without SSE_FLAG_DEFER, or min_pool_pages == SSE_NONE). */
int    ssegw_trim(ssegw *g, uint32_t min_pool_pages);

/* The raw proxy stream handler (api/routes.go:129-232, taken when Accept is exactly text/event-stream, :118): reader and
 * writer in one loop, no channel in between. ssegw_proxy_stream opens the upstream body as a mode P stream (fed through
 * ssegw_upstream_write / _close like any other); ssegw_proxy_step is one turn of the c.Stream callback (:178-231):
 *   1  a line (including its '\n') was copied to buf: the handler writes and flushes it (:220-228) and goes on;
 *   0  no complete line has arrived yet;
 *  -1  ReadBytes returned an error (EOF included): the callback returns false and the unterminated tail is never
 *      written (:187-195).
 * A zero-length element is skipped (:197-199; unreachable, ReadBytes never returns an empty slice with a nil error). */
int    ssegw_proxy_stream(ssegw *g);
int    ssegw_proxy_step(ssegw *g, int stream, uint8_t *buf, size_t cap, size_t *n);

/* The MCP writer (api/middlewares/mcp.go:253-299) for one element of the agent's channel. The frame is always written
 * unchanged. Returns 1 when the stream ends after this write (the frame is byte-equal to "data: [DONE]\n\n", :261-268),
 * else 0. *set_503 becomes 1 when the reference would call WriteHeader(503) for this frame (:272-280): it starts with
 * "data: {", contains "\"error\"", and json.Unmarshal(frame[6:], &struct{ Error string `json:"error"` }) returns nil --
 * i.e. the rest is valid JSON whose top-level keys matching "error" (exactly or case-insensitively) all hold a string or
 * null. Pure host code (no device involved): such frames are rare and the status is not part of the byte stream. */
int ssegw_mcp_writer_step(const uint8_t *frame, size_t n, int *set_503);

#ifdef __cplusplus
}
#endif
#endif
