// sse_fold.cpp -- host-side folds of the device side-band (include/sse_gpu.h): the reference's per-stream
// accumulators fed from sse_rec / sse_tc / sse_usage instead of re-running json.Unmarshal on the host.
//
//   sse_agent_*      mcp/agent.go:156-260 (content builder :211-222, hasToolCalls :224-233, finish :235-242)
//                    and parseStreamingToolCalls mcp/agent.go:377-481 over the same records
//   sse_telemetry_*  api/middlewares/telemetry.go:190-277 (usage from the last <=4 "\n\n" pieces, tool calls
//                    over all pieces)
// No JSON is parsed here: every decision uses flags and spans the kernel already produced.
#include <stdint.h>
#include <string.h>
#include <string>
#include <vector>
#include "../../include/sse_gpu.h"

namespace {

struct Acc {
    int64_t index;
    std::string id, type, name, args;
};

struct AccMap {
    std::vector<Acc> v;   // insertion order; lookups by index (Go map[int]*ToolCall)
    Acc &get(int64_t index) {
        for (auto &a : v) if (a.index == index) return a;
        v.push_back(Acc{ index, "", "function", "", "" });   // Type: types.Function
        return v.back();
    }
    const Acc *find(int64_t index) const {
        for (auto &a : v) if (a.index == index) return &a;
        return nullptr;
    }
};

inline sse_bytes span(const sse_result *r, uint32_t off, uint32_t len, bool text) {
    sse_bytes b;
    b.p = text ? r->text + off : sse_at(r, off);
    b.n = len;
    return b;
}

// The tool-call elements of a record, in order. tc_count saturates at 0xFFFF: a saturated chain is walked to its end.
template <class F> void for_each_tc(const sse_result *res, const sse_rec &r, F f) {
    const uint32_t want = r.tc_count < 0xFFFFu ? r.tc_count : 0xFFFFFFFFu;
    uint32_t t = r.tc_first;
    for (uint32_t k = 0; k < want && t != SSE_NONE; k++) { f(res->tcs[t]); t = res->tcs[t].next; }
}

template <class F> void for_each_run(const sse_result *res, uint32_t seg, F f) {
    const sse_run *run = &res->segs[seg].run;
    for (;;) {
        f(*run);
        if (run->next == SSE_NONE) break;
        run = &res->runs[run->next];
    }
}

size_t emit_calls(const AccMap &m, std::vector<Acc> &store, sse_tool_call *calls, size_t cap, bool require_name) {
    // for i := 0; i < len(toolCallsMap); i++ { if toolCall, exists := toolCallsMap[i] ... }
    store.clear();
    for (size_t i = 0; i < m.v.size(); i++) {
        const Acc *a = m.find((int64_t)i);
        if (!a) continue;
        if (require_name && a->name.empty()) continue;
        store.push_back(*a);
    }
    for (size_t i = 0; i < store.size() && i < cap; i++) {
        calls[i].id = { (const uint8_t *)store[i].id.data(), store[i].id.size() };
        calls[i].type = { (const uint8_t *)store[i].type.data(), store[i].type.size() };
        calls[i].name = { (const uint8_t *)store[i].name.data(), store[i].name.size() };
        calls[i].arguments = { (const uint8_t *)store[i].args.data(), store[i].args.size() };
    }
    return store.size();
}

} // namespace

struct sse_agent_fold {
    std::string content;
    bool has_tool_calls = false, terminated = false, done_break = false;
    int finish = SSE_FIN_NONE;
    AccMap calls;
    std::vector<Acc> store;
};

struct sse_telemetry_fold {
    // "\n\n"-piece reconstruction over the emitted line sequence (mode P) or frames (mode R)
    struct Piece { bool has_usage; sse_usage usage; };
    Piece last4[4];
    uint64_t n_pieces = 0;       // closed pieces so far
    // current (open) piece
    uint32_t cur_lines = 0;      // non-empty lines in the open piece
    bool cur_leading_nl = false; // piece starts with '\n'
    bool cur_has_rec = false;    // its single line has a decoded record
    bool cur_ok = false, cur_has_usage = false, cur_tc = false;
    sse_usage cur_usage{};
    std::vector<Acc> cur_tcs;    // tool-call elements of the open piece's record, in order
    std::vector<uint32_t> cur_tc_flags;
    uint32_t nl_run = 0;
    uint64_t irregular = 0;      // multi-line pieces that start with "data: " (not decodable from per-line records)
    bool finished = false;       // sse_telemetry_finish closed the last piece
    AccMap calls;
    std::vector<Acc> store;
};

namespace {

void tele_close_piece(sse_telemetry_fold *f) {
    sse_telemetry_fold::Piece p{ false, {} };
    bool regular = f->cur_lines == 1 && !f->cur_leading_nl && f->cur_has_rec;
    if (f->cur_lines > 1 && !f->cur_leading_nl && f->cur_has_rec) f->irregular++;
    if (regular && f->cur_ok) {
        if (f->cur_has_usage) { p.has_usage = true; p.usage = f->cur_usage; }
        if (f->cur_tc) {                                  // telemetry.go:240-262
            for (size_t i = 0; i < f->cur_tcs.size(); i++) {
                const Acc &t = f->cur_tcs[i];
                uint32_t fl = f->cur_tc_flags[i];
                Acc &a = f->calls.get(t.index);
                if (fl & SSE_TC_HAS_ID) a.id = t.id;
                if (fl & SSE_TC_HAS_FUNC) {
                    if (!t.name.empty()) a.name = t.name;
                    if (!t.args.empty()) a.args += t.args;
                }
            }
        }
    }
    f->last4[f->n_pieces & 3] = p;
    f->n_pieces++;
    f->cur_lines = 0; f->cur_leading_nl = false; f->cur_has_rec = false; f->cur_ok = false;
    f->cur_has_usage = false; f->cur_tc = false; f->cur_tcs.clear(); f->cur_tc_flags.clear();
}

void tele_take_rec(sse_telemetry_fold *f, const sse_result *res, const sse_rec &r) {
    f->cur_has_rec = true;
    f->cur_ok = (r.flags & SSE_F_JSON_OK) != 0;
    if (!f->cur_ok) return;
    if (r.flags & SSE_F_HAS_USAGE) { f->cur_has_usage = true; f->cur_usage = res->usages[r.usage]; }
    if (r.n_choices > 0 && (r.flags & SSE_F_TC_NONNIL)) {
        f->cur_tc = true;
        for_each_tc(res, r, [&](const sse_tc &tc) {
            Acc a;
            a.index = tc.index;
            sse_bytes id = span(res, tc.id_off, tc.id_len, tc.flags & SSE_TC_ID_TEXT);
            sse_bytes nm = span(res, tc.name_off, tc.name_len, tc.flags & SSE_TC_NAME_TEXT);
            sse_bytes ar = span(res, tc.args_off, tc.args_len, tc.flags & SSE_TC_ARGS_TEXT);
            a.id.assign((const char *)id.p, id.n); a.name.assign((const char *)nm.p, nm.n); a.args.assign((const char *)ar.p, ar.n);
            f->cur_tcs.push_back(a); f->cur_tc_flags.push_back(tc.flags);
        });
    }
}

// one emitted line of a mode-P stream: `len` bytes including its '\n'
void tele_line(sse_telemetry_fold *f, const sse_result *res, uint32_t len, const sse_rec *rec) {
    if (len <= 1) {                       // blank line: another '\n'
        f->nl_run++;
        if (f->nl_run == 2) { tele_close_piece(f); f->nl_run = 0; }
        return;
    }
    if (f->nl_run == 1) {                 // a single '\n' before content: inside the piece
        if (f->cur_lines == 0) f->cur_leading_nl = true;
    }
    f->cur_lines++;
    if (f->cur_lines == 1 && rec) tele_take_rec(f, res, *rec);
    f->nl_run = 1;                        // this line's own '\n'
}

} // namespace

extern "C" {

sse_agent_fold *sse_agent_new(void) { return new sse_agent_fold(); }
void sse_agent_free(sse_agent_fold *f) { delete f; }
void sse_agent_reset(sse_agent_fold *f) { *f = sse_agent_fold(); }

int sse_agent_feed(sse_agent_fold *f, const sse_result *res, uint32_t seg) {
    if (!f || !res || seg >= res->n_segs) return SSE_ERR_ARG;
    bool undecoded = false;
    for_each_run(res, seg, [&](const sse_run &run) {
        for (uint32_t i = 0; i < run.rec_count; i++) {
            const sse_rec &r = res->recs[run.rec_first + i];
            if (r.flags & (SSE_F_TOO_LONG | SSE_F_DEPTH_LIMIT)) undecoded = true;     // the reference would have decoded this line
            const bool done_line = (r.flags & SSE_F_DONE_LINE) != 0;
            const bool ok = (r.flags & SSE_F_JSON_OK) != 0;
            if (!done_line && ok && r.n_choices > 0) {                         // agent.go:205-242
                if (r.content_len) {
                    sse_bytes c = span(res, r.content_off, r.content_len, r.flags & SSE_F_CONTENT_TEXT);
                    f->content.append((const char *)c.p, c.n);                 // :211-222
                }
                if (r.flags & SSE_F_TC_VALID) f->has_tool_calls = true;        // :224-233
                if (r.flags & SSE_F_TERMINATES) {                              // :235-242
                    f->terminated = true;
                    f->finish = (int)((r.flags & SSE_F_FINISH_MASK) >> SSE_F_FINISH_SHIFT);
                }
            }
            // parseStreamingToolCalls over the same builder line (agent.go:377-481)
            if (f->done_break) continue;
            if (r.flags & SSE_F_DONE_EXACT) { f->done_break = true; continue; }   // :394-396
            if (!ok || r.n_choices == 0 || !(r.flags & SSE_F_TC_NONNIL)) continue; // :398-406
            std::vector<const sse_tc *> els;
            for_each_tc(res, r, [&](const sse_tc &tc) { els.push_back(&tc); });
            for (const sse_tc *tc : els) {
                Acc &a = f->calls.get(tc->index);                                  // :409-421
                if (tc->flags & SSE_TC_HAS_ID) {                                   // :424-426
                    sse_bytes b = span(res, tc->id_off, tc->id_len, tc->flags & SSE_TC_ID_TEXT);
                    a.id.assign((const char *)b.p, b.n);
                }
                if (tc->flags & SSE_TC_HAS_TYPE) {                                 // :428-430
                    sse_bytes b = span(res, tc->type_off, tc->type_len, tc->flags & SSE_TC_TYPE_TEXT);
                    a.type.assign((const char *)b.p, b.n);
                }
                if (tc->flags & SSE_TC_HAS_FUNC) {                                 // :432-466: every element with this index
                    for (const sse_tc *t2 : els) {
                        if (t2->index != tc->index) continue;
                        if (t2->name_len) {
                            sse_bytes b = span(res, t2->name_off, t2->name_len, t2->flags & SSE_TC_NAME_TEXT);
                            a.name.assign((const char *)b.p, b.n);
                        }
                        if (t2->args_len) {
                            sse_bytes b = span(res, t2->args_off, t2->args_len, t2->flags & SSE_TC_ARGS_TEXT);
                            a.args.append((const char *)b.p, b.n);
                        }
                    }
                }
            }
        }
    });
    return undecoded ? SSE_ERR_UNDECODED : SSE_OK;
}

sse_bytes sse_agent_content(const sse_agent_fold *f) { return { (const uint8_t *)f->content.data(), f->content.size() }; }
int sse_agent_has_tool_calls(const sse_agent_fold *f) { return f->has_tool_calls ? 1 : 0; }
int sse_agent_terminated(const sse_agent_fold *f, int *finish) { if (finish) *finish = f->finish; return f->terminated ? 1 : 0; }
size_t sse_agent_tool_calls(sse_agent_fold *f, sse_tool_call *calls, size_t cap) {
    return emit_calls(f->calls, f->store, calls, cap, false);
}

sse_telemetry_fold *sse_telemetry_new(void) { return new sse_telemetry_fold(); }
void sse_telemetry_free(sse_telemetry_fold *f) { delete f; }
void sse_telemetry_reset(sse_telemetry_fold *f) { *f = sse_telemetry_fold(); }

int sse_telemetry_feed(sse_telemetry_fold *f, const sse_result *res, uint32_t seg) {
    if (!f || !res || seg >= res->n_segs) return SSE_ERR_ARG;
    bool undecoded = false;
    for_each_run(res, seg, [&](const sse_run &run) {
        for (uint32_t i = 0; i < run.rec_count; i++)
            if (res->recs[run.rec_first + i].flags & (SSE_F_TOO_LONG | SSE_F_DEPTH_LIMIT)) undecoded = true;
        // records of this run in frame order: rec.frame is increasing
        uint32_t ri = 0;
        for (uint32_t i = 0; i < run.frame_count; i++) {
            uint32_t fi = run.frame_first + i;
            const sse_frame &fr = res->frames[fi];
            const sse_rec *rec = nullptr;
            while (ri < run.rec_count && (res->recs[run.rec_first + ri].frame == SSE_NONE || res->recs[run.rec_first + ri].frame < fi)) ri++;
            if (ri < run.rec_count && res->recs[run.rec_first + ri].frame == fi) rec = &res->recs[run.rec_first + ri];
            const uint8_t *b = sse_at(res, fr.off);
            if (fr.len >= 2 && b[fr.len - 1] == '\n' && b[fr.len - 2] == '\n' && rec && !(fr.len >= 1 && b[0] == '\n')) {
                // a reframed "data: X\n\n" frame (mode R): the line and its separator in one element
                tele_line(f, res, fr.len - 1, rec);
                tele_line(f, res, 1, nullptr);
            } else tele_line(f, res, fr.len, rec);
        }
    });
    return undecoded ? SSE_ERR_UNDECODED : SSE_OK;
}

int sse_telemetry_feed_bytes(sse_telemetry_fold *f, const uint8_t *bytes, size_t n) {
    if (!f || (!bytes && n) || (n && bytes[n - 1] != '\n')) return SSE_ERR_ARG;
    size_t s0 = 0;
    for (size_t i = 0; i < n; i++)
        if (bytes[i] == '\n') { tele_line(f, nullptr, (uint32_t)(i + 1 - s0), nullptr); s0 = i + 1; }   // no record: a piece that is not a chunk
    return SSE_OK;
}

int sse_telemetry_finish(sse_telemetry_fold *f, sse_usage *usage, sse_tool_call *calls, size_t cap, size_t *n_calls) {
    if (!f || !usage) return SSE_ERR_ARG;
    // strings.Split always yields a final piece (possibly empty, possibly "X\n"); closed once, so that a second call (with a
    // larger array) gives the same answer
    if (!f->finished) { tele_close_piece(f); f->nl_run = 0; f->finished = true; }
    usage->prompt_tokens = usage->completion_tokens = usage->total_tokens = 0;
    uint64_t n = f->n_pieces, first = n > 4 ? n - 4 : 0;                  // telemetry.go:195-198
    for (uint64_t k = first; k < n; k++) {
        const auto &p = f->last4[k & 3];
        if (p.has_usage) *usage = p.usage;                                   // :219-223 last one wins
    }
    size_t nc = emit_calls(f->calls, f->store, calls, cap, true);            // :268-274
    if (n_calls) *n_calls = nc;
    return f->irregular ? 1 : SSE_OK;
}

} // extern "C"
