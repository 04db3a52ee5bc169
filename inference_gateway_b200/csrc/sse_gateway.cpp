// sse_gateway.cpp -- host-side mirror of the reference's interfaces for the streaming path, above the C ABI.
//
// The reference is compiled Go; its toolchain is absent here, so the host side is C++ with the reference's names and
// error behaviour (the Go shim in integration/go/ is the same logic over cgo):
//
//   ssegw_stream_chat_completions  ~ core.IProvider.StreamChatCompletions (providers/core/interfaces.go:22,
//                                    provider.go:277-344): returns a stream whose channel carries one []byte per line
//   ssegw_upstream_write/close     ~ bytes arriving on response.Body / EOF-or-error (provider.go:322-330: the
//                                    unterminated tail is dropped, then the channel is closed)
//   ssegw_pump                     ~ one tick of the per-GPU batcher goroutine (INTEGRATION.md): micro-batch every
//                                    stream's pending bytes, sse_submit, sse_collect what is done (up to `depth` batches
//                                    stay in flight per context), deliver frames to the channels
//   ssegw_recv                     ~ `line, ok := <-streamCh` (api/routes.go:602-606, mcp/agent.go:171)
//   ssegw_agent_*                  ~ mcp.Agent.RunWithStream for one iteration (mcp/agent.go:126-290): forwards frames to
//                                    the middleware channel, exposes accumulated content / tool calls / finish, appends the
//                                    single final "data: [DONE]\n\n" (agent.go:140-143)
//
// Channel capacity is 100 as in provider.go:307: a stream with 100 undelivered elements stops accepting upstream bytes
// (ssegw_upstream_write returns 0 bytes accepted), which is the back-pressure the reader goroutine would feel.
#include <limits.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>
#include <deque>
#include <string>
#include <vector>
#include "../../include/sse_gateway.h"

namespace {

constexpr size_t CHAN_CAP = 100;
constexpr size_t PENDING_CAP = 4u << 20;   // per-stream bytes waiting for a batch
constexpr uint32_t MAX_DEVICES = 64;       // contexts of one gateway (ssegw_new_multi)

struct Stream {
    bool open = false;          // slot in use
    bool upstream_eof = false;  // response.Body returned EOF / error
    bool closed = false;        // channel closed (after the last line was delivered)
    uint8_t mode = 0;
    std::string pending;        // bytes read from upstream, not yet handed to the GPU
    std::deque<std::string> chan;
    bool terminated = false;    // mode R: agent loop left (finish_reason stop/tool_calls)
    sse_agent_fold *agent = nullptr;
    sse_telemetry_fold *tel = nullptr;   // the caller's tap (ssegw_stream_with_telemetry), not owned; null: no tap
    bool done_sent = false;
    bool deferred = false;      // SSE_FLAG_DEFER: the last batch left bytes of this stream in `pending`; offered first next tick
    uint64_t gen = 0;           // bumped at every open: a batch that holds bytes of an earlier stream on the slot delivers nothing here
    uint32_t in_flight = 0;     // uncollected batches that hold bytes of this stream (this generation)
};

// One stream's bytes in a submitted batch: where they stand in the batch's input arena, and which stream they were taken from.
struct Member { uint32_t stream; uint64_t gen; uint32_t off, len; };
struct InFlight { int slot; std::vector<Member> who; };

// One context (one device, or one of several contexts on a device): its connections are streams
// [index * max_conns, (index + 1) * max_conns) of the gateway, and its uncollected batches, oldest first.
struct Ctx {
    sse_ctx *ctx = nullptr;
    std::deque<InFlight> inflight;
    size_t rr = 0;              // the batcher starts its scan one connection further every tick (no slot is favoured)
    uint32_t n_open = 0;        // open streams, for placement
};

} // namespace

struct ssegw {
    std::vector<Ctx> ctxs;
    sse_config cfg{};
    uint32_t depth = 1;         // batches a context may have uncollected during a pump (a pump leaves at most depth - 1)
    std::vector<Stream> streams;
    std::string last_error;
    sse_counters sum{};         // SSE_FLAG_COUNTERS: every collected batch's counters added up (ssegw_counters)
};

namespace {

// SSE_FLAG_COUNTERS: adds the counters of the batch just collected in `slot` to the gateway's sums (d_items_per_pull is the
// launch's choice, not an amount: the last batch's is kept)
void add_counters(ssegw *g, sse_ctx *ctx, int slot) {
    sse_counters k{};
    k.struct_size = sizeof k;
    if (sse_counters_read(ctx, slot, &k) != SSE_OK) return;
    uint64_t *dst = &g->sum.p_segments;
    const uint64_t *src = &k.p_segments;
    const size_t n = (sizeof k - offsetof(sse_counters, p_segments)) / sizeof(uint64_t);
    for (size_t i = 0; i < n; i++) dst[i] += src[i];
    g->sum.d_items_per_pull = k.d_items_per_pull;
    g->sum.decode_passes += k.decode_passes;
}

// a failed batch fails its streams: the client sees EOF, exactly like an upstream read error (provider.go:323-330). With
// SSE_FLAG_DEFER a batch does not fail for want of arena space, only on a CUDA or allocation error.
void fail_batch(ssegw *g, Ctx &x, const InFlight &f) {
    for (const Member &m : f.who) {
        Stream &s = g->streams[m.stream];
        if (s.gen != m.gen) continue;
        s.in_flight--;
        s.closed = true;
    }
    sse_release(x.ctx, f.slot);
}

// Step 1 of a tick on context k: fills a batch with what the streams have pending and submits it (nothing when no stream
// has bytes that may go in). The bytes leave `pending` now.
int submit_batch(ssegw *g, size_t k) {
    Ctx &x = g->ctxs[k];
    int slot; sse_batch b;
    int rc = sse_acquire(x.ctx, &slot, &b);
    if (rc != SSE_OK) return rc;
    InFlight f{ slot, {} };
    uint32_t off = 0, n = 0;
    const size_t nc = g->cfg.max_conns, base = k * nc;
    const size_t start = x.rr++ % nc;
    const bool defer = (g->cfg.flags & SSE_FLAG_DEFER) != 0;
    // streams whose bytes a batch deferred (SSE_FLAG_DEFER) go first, so that a flood on other streams cannot keep them waiting
    for (int pass = 0; pass < 2; pass++)
    for (size_t q = 0; q < nc && n < b.max_segs; q++) {
        const size_t i = (start + q) % nc;
        Stream &s = g->streams[base + i];
        if (s.deferred != (pass == 0)) continue;
        if (!s.open || s.closed || s.pending.empty()) continue;
        if (s.chan.size() >= CHAN_CAP) continue;                      // receiver is slow: leave the bytes queued
        if (defer && s.in_flight) continue;                           // a deferred rest of that batch must come before these bytes
        // a stream takes what fits: the rest stays queued for the next tick (the carry state on the device makes any cut legal)
        const size_t room = b.in_arena_bytes > off + 16u ? (size_t)(b.in_arena_bytes - off - 16u) : 0;
        const size_t take = s.pending.size() < room ? s.pending.size() : room;
        if (take == 0) continue;
        memcpy(b.in_arena + off, s.pending.data(), take);
        b.segs[n] = sse_seg{ (uint32_t)i, off, (uint32_t)take, s.mode, 0, 0 };
        f.who.push_back(Member{ (uint32_t)(base + i), s.gen, off, (uint32_t)take });
        s.pending.erase(0, take);
        s.in_flight++;
        off = (off + (uint32_t)take + 15u) & ~15u;
        n++;
    }
    if (!n) return sse_release(x.ctx, slot);
    rc = sse_submit(x.ctx, slot, n, off);
    if (rc != SSE_OK) { fail_batch(g, x, f); return rc; }
    x.inflight.push_back(std::move(f));
    return SSE_OK;
}

// Collects the oldest uncollected batch of a context and fans it out: frames to the channels, records to the agent folds.
// Returns the frames delivered or a negative status (the batch failed).
int collect_oldest(ssegw *g, Ctx &x) {
    const InFlight f = std::move(x.inflight.front());
    x.inflight.pop_front();
    sse_result res;
    const int rc = sse_collect(x.ctx, f.slot, &res);
    if (rc != SSE_OK) { fail_batch(g, x, f); return rc; }
    if (g->cfg.flags & SSE_FLAG_COUNTERS) add_counters(g, x.ctx, f.slot);
    int delivered = 0;
    for (uint32_t k = 0; k < (uint32_t)f.who.size(); k++) {
        const Member &m = f.who[k];
        Stream &s = g->streams[m.stream];
        if (s.gen != m.gen) continue;       // released and reopened since: the connection was reset after this batch, its
                                            // results belong to nobody
        s.in_flight--;
        // released, or failed by an earlier batch or fold: the connection state no longer describes the stream
        if (!s.open || s.closed) continue;
        // only the bytes the batch took are gone: a deferred rest goes back to the front of the queue, before anything newer
        const uint32_t consumed = res.segs[k].consumed;
        if (consumed < m.len) s.pending.insert(0, (const char *)res.in + m.off + consumed, m.len - consumed);
        s.deferred = (res.segs[k].flags & SSE_SEG_DEFERRED) != 0;
        const sse_run *run = &res.segs[k].run;
        for (;;) {
            for (uint32_t fr = run->frame_first; fr < run->frame_first + run->frame_count; fr++) {
                s.chan.emplace_back((const char *)sse_at(&res, res.frames[fr].off), res.frames[fr].len);   // fresh copy per element
                delivered++;
            }
            if (run->next == SSE_NONE) break;
            run = &res.runs[run->next];
        }
        // a record the library could not decode (SSE_ERR_UNDECODED): the accumulators would be silently short, so the stream is failed
        bool undecoded = (s.mode & SSE_MODE_R) && sse_agent_feed(s.agent, &res, k) != SSE_OK;
        if (s.tel && sse_telemetry_feed(s.tel, &res, k) != SSE_OK) undecoded = true;
        if (undecoded) s.closed = true;
        if (res.segs[k].flags & SSE_SEG_TERMINATED) s.terminated = true;
        if (res.segs[k].flags & SSE_SEG_DEAD) s.closed = true;
    }
    sse_release(x.ctx, f.slot);
    return delivered;
}

// upstream EOF: the channel closes once no byte of the stream waits on the host or in a batch (the unterminated tail, if
// any, stays on the device and is dropped)
void close_drained(ssegw *g) {
    for (auto &s : g->streams)
        if (s.open && s.upstream_eof && s.pending.empty() && !s.in_flight) s.closed = true;
}

} // namespace

extern "C" {

ssegw *ssegw_new(int device, uint32_t max_conns, uint32_t bytes_per_batch, int *status) {
    return ssegw_new_ex(device, max_conns, bytes_per_batch, nullptr, status);
}

ssegw *ssegw_new_ex(int device, uint32_t max_conns, uint32_t bytes_per_batch, const sse_line_pool *pool, int *status) {
    // worst-case result capacities: whatever the upstreams send (a flood of one-byte lines, of empty tool-call elements ...), a
    // batch cannot overflow, so one connection can never fail the batch of the others; a line pool grows them by its size
    sse_config cfg;
    sse_worst_case_config(&cfg, max_conns, bytes_per_batch);
    return ssegw_new_cfg(device, &cfg, pool, status);
}

ssegw *ssegw_new_cfg(int device, const sse_config *cfg, const sse_line_pool *pool, int *status) {
    return ssegw_new_multi(&device, 1, cfg, pool, 1, status);
}

ssegw *ssegw_new_multi(const int *devices, uint32_t n_devices, const sse_config *cfg, const sse_line_pool *pool, uint32_t depth,
                       int *status) {
    if (!devices || n_devices == 0 || n_devices > MAX_DEVICES || !cfg || cfg->struct_size != sizeof(sse_config) || depth < 1 ||
        depth > cfg->n_slots || (uint64_t)n_devices * cfg->max_conns > (uint64_t)INT_MAX) {
        if (status) *status = SSE_ERR_ARG;
        return nullptr;
    }
    ssegw *g = new ssegw();
    g->cfg = *cfg;
    g->depth = depth;
    g->ctxs.resize(n_devices);
    for (uint32_t k = 0; k < n_devices; k++) {
        const int rc = sse_init_ex(devices[k], &g->cfg, pool, &g->ctxs[k].ctx);
        if (rc != SSE_OK) {   // no CUDA device: error, never a CPU path
            if (status) *status = rc;
            ssegw_free(g);
            return nullptr;
        }
    }
    g->streams.resize((size_t)n_devices * cfg->max_conns);
    if (status) *status = SSE_OK;
    return g;
}

void ssegw_free(ssegw *g) {
    if (!g) return;
    ssegw_flush(g);   // every slot is released, whatever the batches returned
    for (auto &s : g->streams) if (s.agent) sse_agent_free(s.agent);
    for (auto &x : g->ctxs) sse_destroy(x.ctx);
    delete g;
}

// StreamChatCompletions: binds a new stream to a free connection of the context with the fewest open streams (the lowest
// index on a tie), where it stays for its whole life; tel (may be null) is its telemetry tap. Returns the stream id or -1
// (no free slot).
static int open_stream(ssegw *g, uint8_t mode, sse_telemetry_fold *tel) {
    const size_t nc = g->cfg.max_conns;
    size_t k = g->ctxs.size();
    for (size_t j = 0; j < g->ctxs.size(); j++)
        if (g->ctxs[j].n_open < nc && (k == g->ctxs.size() || g->ctxs[j].n_open < g->ctxs[k].n_open)) k = j;
    if (k == g->ctxs.size()) return -1;
    for (size_t i = k * nc; i < (k + 1) * nc; i++) {
        Stream &s = g->streams[i];
        if (!s.open) {
            if (s.agent) sse_agent_reset(s.agent); else s.agent = sse_agent_new();
            sse_agent_fold *agent = s.agent;
            const uint64_t gen = s.gen + 1;
            s = Stream{};
            s.open = true; s.mode = mode; s.agent = agent; s.gen = gen;
            g->ctxs[k].n_open++;
            // ordered after every batch already submitted, which may still hold bytes of the slot's previous stream
            if (sse_reset_conn(g->ctxs[k].ctx, (uint32_t)(i - k * nc)) != SSE_OK) return -1;
            s.tel = tel;
            return (int)i;
        }
    }
    return -1;
}

int ssegw_stream_chat_completions(ssegw *g, uint8_t mode) { return open_stream(g, mode, nullptr); }

int ssegw_stream_with_telemetry(ssegw *g, uint8_t mode, sse_telemetry_fold *tel) {
    if (!g || !tel || !(mode & (SSE_MODE_PARSE | SSE_MODE_R))) return SSE_ERR_ARG;
    for (const Stream &s : g->streams)
        if (s.open && s.tel == tel) return SSE_ERR_BUSY;     // one feeder at a time: the pieces of two bodies would interleave
    return open_stream(g, mode, tel);
}

// Bytes from response.Body. Returns the number of bytes accepted (0 when the channel is full: back-pressure).
size_t ssegw_upstream_write(ssegw *g, int id, const uint8_t *data, size_t n) {
    Stream &s = g->streams[(size_t)id];
    if (!s.open || s.upstream_eof || s.closed) return 0;
    if (s.chan.size() >= CHAN_CAP) return 0;
    // bytes not yet handed to the GPU are bounded like a socket buffer: a reader that outruns the batcher is told to wait
    const size_t room = s.pending.size() < PENDING_CAP ? PENDING_CAP - s.pending.size() : 0;
    if (n > room) n = room;
    s.pending.append((const char *)data, n);
    return n;
}

void ssegw_upstream_close(ssegw *g, int id) { g->streams[(size_t)id].upstream_eof = true; }

// One batcher tick. For each context: fill and submit a batch, collect every batch that is done (oldest first), then collect
// the oldest, blocking, while `depth` are uncollected. At depth 1 the batch submitted is delivered in the same call. Fan-out
// happens at collect time, in submission order per context. Returns the number of frames delivered, or a negative sse_status.
int ssegw_pump(ssegw *g) {
    int delivered = 0;
    for (size_t k = 0; k < g->ctxs.size(); k++) {
        Ctx &x = g->ctxs[k];
        int rc = submit_batch(g, k);
        if (rc != SSE_OK) return rc;
        while (!x.inflight.empty() && sse_poll(x.ctx, x.inflight.front().slot) != 0) {   // done, or an error collect reports
            if ((rc = collect_oldest(g, x)) < 0) return rc;
            delivered += rc;
        }
        while (x.inflight.size() >= g->depth) {
            if ((rc = collect_oldest(g, x)) < 0) return rc;
            delivered += rc;
        }
    }
    close_drained(g);
    return delivered;
}

// Collects every uncollected batch of every context. Returns the frames delivered, or the first negative sse_status (the
// batches after a failed one are still collected).
int ssegw_flush(ssegw *g) {
    if (!g) return SSE_ERR_ARG;
    int delivered = 0, first = SSE_OK;
    for (auto &x : g->ctxs)
        while (!x.inflight.empty()) {
            const int rc = collect_oldest(g, x);
            if (rc < 0) { if (first == SSE_OK) first = rc; }
            else delivered += rc;
        }
    close_drained(g);
    return first != SSE_OK ? first : delivered;
}

// `line, ok := <-streamCh`: 1 = element copied to buf (*n bytes), 0 = nothing available yet, -1 = channel closed and drained.
int ssegw_recv(ssegw *g, int id, uint8_t *buf, size_t cap, size_t *n) {
    Stream &s = g->streams[(size_t)id];
    if (!s.chan.empty()) {
        const std::string &e = s.chan.front();
        *n = e.size();
        if (e.size() > cap) return SSE_ERR_ARG;
        memcpy(buf, e.data(), e.size());
        s.chan.pop_front();
        return 1;
    }
    return s.closed ? -1 : 0;
}

void ssegw_release_stream(ssegw *g, int id) {
    Stream &s = g->streams[(size_t)id];
    if (s.open) g->ctxs[(size_t)id / g->cfg.max_conns].n_open--;
    s.open = false;
    s.tel = nullptr;      // the caller may free or reattach its fold now: nothing collected later feeds it
}

int ssegw_counters(ssegw *g, sse_counters *out) {
    if (!g || !out || out->struct_size != sizeof(sse_counters) || !(g->cfg.flags & SSE_FLAG_COUNTERS)) return SSE_ERR_ARG;
    *out = g->sum;
    out->struct_size = sizeof(sse_counters);
    return SSE_OK;
}

int ssegw_line_pool_growth(ssegw *g, uint32_t max_pages) {
    if (!g) return SSE_ERR_ARG;
    for (auto &x : g->ctxs) {
        const int rc = sse_line_pool_set_growth(x.ctx, max_pages);
        if (rc != SSE_OK) return rc;
    }
    return SSE_OK;
}

int ssegw_trim(ssegw *g, uint32_t min_pool_pages) {
    if (!g) return SSE_ERR_ARG;
    int first = SSE_OK;
    for (auto &x : g->ctxs) {
        const int rc = sse_trim(x.ctx, min_pool_pages);
        if (rc != SSE_OK && first == SSE_OK) first = rc;
    }
    return first;
}

// ---- handleStreamingRequest (api/routes.go:129-232): the raw proxy loop reads and writes in one goroutine
int ssegw_proxy_stream(ssegw *g) { return ssegw_stream_chat_completions(g, SSE_MODE_P); }
int ssegw_proxy_step(ssegw *g, int id, uint8_t *buf, size_t cap, size_t *n) {
    for (;;) {
        const int rc = ssegw_recv(g, id, buf, cap, n);
        if (rc != 1) return rc;              // 0: nothing yet; -1: ReadBytes error / EOF, tail dropped (:187-195)
        if (*n == 0) continue;               // :197-199
        return 1;                            // :220-228 write + flush
    }
}

// ---- mcp.Agent.RunWithStream view of a mode-R stream (one iteration)
// Next element of the middleware channel: forwarded frames, then exactly one "data: [DONE]\n\n" once the iteration is
// over (finish_reason stop/tool_calls seen, or the provider channel closed). Same return codes as ssegw_recv.
int ssegw_agent_recv(ssegw *g, int id, uint8_t *buf, size_t cap, size_t *n) {
    Stream &s = g->streams[(size_t)id];
    int rc = ssegw_recv(g, id, buf, cap, n);
    if (rc == 1 || rc == SSE_ERR_ARG) return rc;      // SSE_ERR_ARG: the next element is longer than cap (*n), still queued
    const bool over = s.terminated || rc == -1;
    if (over && !s.done_sent) {
        static const char done[] = "data: [DONE]\n\n";
        *n = sizeof(done) - 1;
        if (*n > cap) return SSE_ERR_ARG;
        memcpy(buf, done, *n);
        s.done_sent = true;
        return 1;
    }
    return over ? -1 : 0;
}
sse_bytes ssegw_agent_content(ssegw *g, int id) { return sse_agent_content(g->streams[(size_t)id].agent); }
int ssegw_agent_has_tool_calls(ssegw *g, int id) { return sse_agent_has_tool_calls(g->streams[(size_t)id].agent); }
int ssegw_agent_terminated(ssegw *g, int id, int *finish) { return sse_agent_terminated(g->streams[(size_t)id].agent, finish); }
size_t ssegw_agent_tool_calls(ssegw *g, int id, sse_tool_call *calls, size_t cap) {
    return sse_agent_tool_calls(g->streams[(size_t)id].agent, calls, cap);
}

// ---- handleMCPStreamingRequest's writer, one channel element (api/middlewares/mcp.go:253-299)
namespace {

// encoding/json's checkValid + a walk of the top-level object, enough to tell whether
// json.Unmarshal(data, &struct{ Error string `json:"error"` }) returns nil. Iterative (Go's nesting limit is 10000).
struct ErrSniff {
    const uint8_t *p, *e;
    bool ws() { while (p < e && (*p == ' ' || *p == '\t' || *p == '\n' || *p == '\r')) p++; return p < e; }
    static int hexv(uint8_t c) { return c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : c >= 'A' && c <= 'F' ? c - 'A' + 10 : -1; }
    // scans a string starting at the opening quote; appends the unquoted bytes to *out when given
    bool str(std::string *out) {
        p++;
        while (p < e) {
            uint8_t c = *p;
            if (c == '"') { p++; return true; }
            if (c < 0x20) return false;
            if (c != '\\') { if (out) out->push_back((char)c); p++; continue; }
            if (++p >= e) return false;
            c = *p++;
            switch (c) {
            case '"': case '\\': case '/': if (out) out->push_back((char)c); break;
            case 'b': if (out) out->push_back('\b'); break;
            case 'f': if (out) out->push_back('\f'); break;
            case 'n': if (out) out->push_back('\n'); break;
            case 'r': if (out) out->push_back('\r'); break;
            case 't': if (out) out->push_back('\t'); break;
            case 'u': {
                if (e - p < 4) return false;
                int v = 0;
                for (int k = 0; k < 4; k++) { int h = hexv(p[k]); if (h < 0) return false; v = v * 16 + h; }
                p += 4;
                // only ASCII matters for the comparison with "error"; anything else makes the key differ
                if (out) out->push_back(v < 0x80 ? (char)v : (char)0xFF);
                break;
            }
            default: return false;
            }
        }
        return false;
    }
    bool number() {
        if (p < e && *p == '-') p++;
        if (p >= e) return false;
        if (*p == '0') p++;
        else if (*p >= '1' && *p <= '9') { while (p < e && *p >= '0' && *p <= '9') p++; }
        else return false;
        if (p < e && *p == '.') { p++; if (p >= e || *p < '0' || *p > '9') return false; while (p < e && *p >= '0' && *p <= '9') p++; }
        if (p < e && (*p == 'e' || *p == 'E')) {
            p++;
            if (p < e && (*p == '+' || *p == '-')) p++;
            if (p >= e || *p < '0' || *p > '9') return false;
            while (p < e && *p >= '0' && *p <= '9') p++;
        }
        return true;
    }
    bool lit(const char *w) { size_t n = strlen(w); if ((size_t)(e - p) < n || memcmp(p, w, n) != 0) return false; p += n; return true; }
    static bool is_error_key(const std::string &k) {
        if (k.size() != 5) return false;
        static const char want[] = "error";
        for (int i = 0; i < 5; i++) { char c = k[i]; if (c >= 'A' && c <= 'Z') c = (char)(c + 32); if (c != want[i]) return false; }
        return true;
    }
    // returns true when Unmarshal would return nil
    bool run() {
        std::vector<uint8_t> stk;     // 1 = object, 0 = array
        bool type_ok = true;
        if (!ws() || *p != '{') return false;       // (the caller checked the "data: {" prefix; kept for completeness)
        // state machine over values
        enum { VALUE, AFTER } st = VALUE;
        bool pending_error_key = false;             // the value about to be read belongs to a top-level "error" key
        for (;;) {
            if (st == VALUE) {
                if (!ws()) return false;
                const uint8_t c = *p;
                const bool top = stk.size() == 1 && stk.back() == 1;
                const bool chk = top && pending_error_key;
                if (c == '{' || c == '[') {
                    if (chk) type_ok = false;
                    pending_error_key = false;
                    if (stk.size() >= 10000) return false;
                    stk.push_back(c == '{');
                    p++;
                    if (!ws()) return false;
                    if (c == '{') {
                        if (*p == '}') { p++; stk.pop_back(); st = AFTER; continue; }
                        // key
                        if (*p != '"') return false;
                        std::string key; const bool want_key = stk.size() == 1;
                        if (!str(want_key ? &key : nullptr)) return false;
                        if (want_key) pending_error_key = is_error_key(key);
                        if (!ws() || *p != ':') return false;
                        p++;
                        continue;
                    }
                    if (*p == ']') { p++; stk.pop_back(); st = AFTER; continue; }
                    continue;
                }
                if (stk.empty()) return false;
                if (c == '"') { if (!str(nullptr)) return false; }
                else if (c == '-' || (c >= '0' && c <= '9')) { if (!number()) return false; if (chk) type_ok = false; }
                else if (c == 't') { if (!lit("true")) return false; if (chk) type_ok = false; }
                else if (c == 'f') { if (!lit("false")) return false; if (chk) type_ok = false; }
                else if (c == 'n') { if (!lit("null")) return false; }
                else return false;
                pending_error_key = false;
                st = AFTER;
                continue;
            }
            // AFTER a value
            if (stk.empty()) { ws(); return p == e && type_ok; }
            if (!ws()) return false;
            if (stk.back() == 1) {
                if (*p == '}') { p++; stk.pop_back(); continue; }
                if (*p != ',') return false;
                p++;
                if (!ws() || *p != '"') return false;
                std::string key; const bool want_key = stk.size() == 1;
                if (!str(want_key ? &key : nullptr)) return false;
                if (want_key) pending_error_key = is_error_key(key);
                if (!ws() || *p != ':') return false;
                p++;
                st = VALUE;
            } else {
                if (*p == ']') { p++; stk.pop_back(); continue; }
                if (*p != ',') return false;
                p++;
                st = VALUE;
            }
        }
    }
};

bool contains(const uint8_t *h, size_t n, const char *needle) {
    const size_t m = strlen(needle);
    if (n < m) return false;
    for (size_t i = 0; i + m <= n; i++) if (h[i] == (uint8_t)needle[0] && memcmp(h + i, needle, m) == 0) return true;
    return false;
}

} // namespace

int ssegw_mcp_writer_step(const uint8_t *frame, size_t n, int *set_503) {
    static const char done[] = "data: [DONE]\n\n";
    if (set_503) *set_503 = 0;
    if (n == sizeof(done) - 1 && memcmp(frame, done, n) == 0) return 1;                 // mcp.go:261-268
    if (n >= 7 && memcmp(frame, "data: {", 7) == 0 && contains(frame, n, "\"error\"")) {   // mcp.go:272-280
        ErrSniff s{ frame + 6, frame + n };
        if (s.run() && set_503) *set_503 = 1;
    }
    return 0;
}

} // extern "C"
