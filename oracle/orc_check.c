/* orc_check.c -- full-size parity checker: per-connection digests of everything the path produces, and a structural check of
 * one batch result.
 * TEST INFRASTRUCTURE ONLY (tests/ and __graft_entry__.smoke()); never on the product path.
 *
 * Comparing 65,536 streams x ~11 events field by field from Python takes minutes, so both sides are reduced in C to the
 * same canonical byte string per connection and hashed (FNV-1a, 64 bit):
 *   frames digest : for every emitted frame, in order:  u32 len, bytes
 *   records digest: for every decoded line, in order:   u8 json_ok, u8 done, u8 done_exact, u8 depth_limit,
 *                   u32 frame (ordinal of the linked frame among the connection's frames, or 0xFFFFFFFF), u32 payload_len,
 *                   u8 terminates, and when json_ok:
 *                   u32 min(n_choices, 65535), u32 finish, u8 has_usage [3 x i64], u32 content_len, content bytes,
 *                   u8 tool_calls_nonnil, u8 has_valid_tool_call, u32 min(tc_count, 65535), then per element
 *                   i64 index, u8 has_id [u32 len, bytes], u8 has_type [u32 len, bytes], u8 has_function,
 *                   u32 name_len, name, u32 args_len, args
 * On the oracle side depth_limit is the documented nesting limit restated (orc_json_scan at 128 levels, DESIGN.md §5
 * deviation 2): such a line is expected with json_ok 0, and on the GPU side it is the SSE_F_DEPTH_LIMIT flag.
 * orc_digest_streams runs the oracle (sse_oracle.c) over whole upstream bodies; orc_digest_result folds ONE batch result of
 * the GPU library (the plain C structs of include/sse_gpu.h) into the digests of the connections its segments belong to, so a
 * stream cut into any number of batches ends at the same digest as the oracle's single pass over it.
 * The record fields are the ones tests/util.py's check_stream compares (chunk_to_dict / rec_to_dict, plus the frame link,
 * payload_len, terminates and depth_limit).
 *
 * orc_check_result checks what the digests cannot see: that the indices of one batch result (runs, frame and record ranges,
 * record -> frame links, tool-call chains, usage indices, arena spans) stay in bounds, belong to one segment each and agree with
 * each other and with the submitted sse_seg descriptors. It validates every index before it dereferences it, so it runs
 * before orc_digest_result. */
#define _GNU_SOURCE
#include "sse_oracle.h"
#include "../include/sse_gpu.h"
#include <pthread.h>
#include <stdarg.h>
#include <stdatomic.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
    uint64_t frames_h, recs_h;      /* running FNV-1a states (start: ORC_FNV_INIT) */
    uint64_t n_frames, n_recs, frame_bytes;
    uint32_t inexact;               /* GPU side: records flagged TOO_LONG (side-band not decoded); + 1 << 16 per broken tool-call chain */
    uint32_t pad;
} orc_digest;

#define ORC_FNV_INIT 0xcbf29ce484222325ull
#define ORC_FNV_MUL 0x100000001b3ull

static inline uint64_t h_bytes(uint64_t h, const void *p, size_t n) {
    const uint8_t *b = (const uint8_t *)p;
    for (size_t i = 0; i < n; i++) { h ^= b[i]; h *= ORC_FNV_MUL; }
    return h;
}
static inline uint64_t h_u8(uint64_t h, uint32_t v) { uint8_t b = (uint8_t)v; return h_bytes(h, &b, 1); }
static inline uint64_t h_u32(uint64_t h, uint32_t v) { return h_bytes(h, &v, 4); }
static inline uint64_t h_i64(uint64_t h, int64_t v) { return h_bytes(h, &v, 8); }
static inline uint64_t h_str(uint64_t h, const uint8_t *p, uint32_t n) { h = h_u32(h, n); return h_bytes(h, p, n); }

void orc_digest_init(orc_digest *d, size_t n) {
    for (size_t i = 0; i < n; i++) { memset(&d[i], 0, sizeof d[i]); d[i].frames_h = d[i].recs_h = ORC_FNV_INIT; }
}

/* ---------------------------------------------------------------- oracle side */
/* depth: the line's payload hits the nesting limit (the record is then json_ok 0 whatever Go would say) */
static uint64_t h_chunk(uint64_t h, const orc_result *r, const orc_chunk *c, int done, int done_exact, int depth,
                        uint32_t frame, uint32_t payload_len, int terminates) {
    const int ok = c && c->json_ok && !depth;
    h = h_u8(h, (uint32_t)ok); h = h_u8(h, (uint32_t)done); h = h_u8(h, (uint32_t)done_exact); h = h_u8(h, (uint32_t)depth);
    h = h_u32(h, frame); h = h_u32(h, payload_len); h = h_u8(h, (uint32_t)terminates);
    if (!ok) return h;
    h = h_u32(h, c->n_choices > 65535u ? 65535u : c->n_choices);
    h = h_u32(h, c->finish);
    h = h_u8(h, c->has_usage);
    if (c->has_usage) { h = h_i64(h, c->prompt); h = h_i64(h, c->completion); h = h_i64(h, c->total); }
    h = h_str(h, r->text + c->content.off, c->content.len);
    h = h_u8(h, c->tool_calls_nonnil); h = h_u8(h, c->has_valid_tool_call);
    h = h_u32(h, c->tc_count > 65535u ? 65535u : c->tc_count);
    for (uint32_t k = 0; k < c->tc_count && k < 65535u; k++) {
        const orc_tc *t = &r->tcs[c->tc_first + k];
        h = h_i64(h, t->index);
        h = h_u8(h, t->has_id);   if (t->has_id) h = h_str(h, r->text + t->id.off, t->id.len);
        h = h_u8(h, t->has_type); if (t->has_type) h = h_str(h, r->text + t->type.off, t->type.len);
        h = h_u8(h, t->has_function);
        h = h_str(h, r->text + t->name.off, t->name.len);
        h = h_str(h, r->text + t->args.off, t->args.len);
    }
    return h;
}

static int depth_limited(const uint8_t *body, const orc_line *l) {
    return orc_json_scan(body + l->pay_off, l->pay_len, ORC_DEPTH_LIMIT) == ORC_JSON_DEPTH;
}

static void digest_one(orc_result *r, const uint8_t *body, size_t n, uint32_t mode, orc_digest *d, uint8_t *terminated, uint32_t *tail_len) {
    orc_result_clear(r);
    if (mode & 1u) orc_reframe_stream(r, body, n, 0);
    else orc_passthrough(r, body, n, (mode & 2u) != 0);
    for (size_t i = 0; i < r->n_lines; i++) {
        const orc_line *l = &r->lines[i];
        const orc_chunk *c = l->chunk != 0xFFFFFFFFu ? &r->chunks[l->chunk] : 0;
        const uint32_t ord = (uint32_t)d->n_frames;      /* the frame this line emits, if any */
        if (mode & 1u) {
            if (l->kind == ORC_L_EMITTED) {
                const int dl = depth_limited(body, l);
                const int term = !dl && c->json_ok && c->n_choices > 0 && (c->finish == ORC_FIN_STOP || c->finish == ORC_FIN_TOOL_CALLS);
                d->frames_h = h_str(d->frames_h, r->out + l->out_off, l->out_len); d->n_frames++; d->frame_bytes += l->out_len;
                d->recs_h = h_chunk(d->recs_h, r, c, 0, 0, dl, ord, l->pay_len, term); d->n_recs++;
            } else if (l->kind == ORC_L_DONE) {
                d->recs_h = h_chunk(d->recs_h, r, c, 1, 0, depth_limited(body, l), 0xFFFFFFFFu, l->pay_len, 0); d->n_recs++;
            } else if (l->kind == ORC_L_DONE_EXACT) { d->recs_h = h_chunk(d->recs_h, r, 0, 1, 1, 0, 0xFFFFFFFFu, l->pay_len, 0); d->n_recs++; }
        } else {
            d->frames_h = h_str(d->frames_h, r->out + l->out_off, l->out_len); d->n_frames++; d->frame_bytes += l->out_len;
            if (c) { d->recs_h = h_chunk(d->recs_h, r, c, 0, 0, depth_limited(body, l), ord, l->pay_len, 0); d->n_recs++; }
        }
    }
    *terminated = (uint8_t)((mode & 1u) ? r->terminated : 0);
    *tail_len = (uint32_t)r->tail_len;
}

typedef struct {
    const uint8_t *arena; const uint64_t *off; const uint32_t *len; const uint8_t *mode; size_t n;
    atomic_size_t *next; orc_digest *d; uint8_t *terminated; uint32_t *tail_len;
} cjob;

static void *cworker(void *p) {
    cjob *j = (cjob *)p;
    orc_result *r = orc_result_new();
    for (;;) {
        size_t s0 = atomic_fetch_add(j->next, 16);
        if (s0 >= j->n) break;
        size_t s1 = s0 + 16 < j->n ? s0 + 16 : j->n;
        for (size_t s = s0; s < s1; s++) digest_one(r, j->arena + j->off[s], j->len[s], j->mode[s], &j->d[s], &j->terminated[s], &j->tail_len[s]);
    }
    orc_result_free(r);
    return 0;
}

/* Oracle digests of n whole upstream bodies (mode bit0 R, bit1 parse). d must be orc_digest_init'ed. */
void orc_digest_streams(const uint8_t *arena, const uint64_t *off, const uint32_t *len, const uint8_t *mode, size_t n,
                        int n_threads, orc_digest *d, uint8_t *terminated, uint32_t *tail_len) {
    if (n_threads < 1) n_threads = 1;
    pthread_t *th = (pthread_t *)calloc((size_t)n_threads, sizeof *th);
    atomic_size_t next = 0;
    cjob j = { arena, off, len, mode, n, &next, d, terminated, tail_len };
    for (int t = 0; t < n_threads; t++) pthread_create(&th[t], 0, cworker, &j);
    for (int t = 0; t < n_threads; t++) pthread_join(th[t], 0);
    free(th);
}

/* ---------------------------------------------------------------- GPU side */
static inline const uint8_t *at(const sse_result *res, uint32_t off) {      /* sse_at(), restated so that liborc does not link the product */
    return off >= res->in_base ? res->in + (off - res->in_base) : res->out + off;
}
static inline const uint8_t *span(const sse_result *res, uint32_t off, int in_text) { return in_text ? res->text + off : at(res, off); }

/* ord: the linked frame's ordinal among the connection's frames (0xFFFFFFFF: none, 0xFFFFFFFE: outside the record's run) */
static uint64_t h_rec(uint64_t h, const sse_result *res, const sse_rec *rc, uint32_t ord, uint32_t *inexact) {
    const uint32_t fl = rc->flags;
    if (fl & SSE_F_TOO_LONG) (*inexact)++;
    h = h_u8(h, (fl & SSE_F_JSON_OK) != 0); h = h_u8(h, (fl & SSE_F_DONE_LINE) != 0); h = h_u8(h, (fl & SSE_F_DONE_EXACT) != 0);
    h = h_u8(h, (fl & SSE_F_DEPTH_LIMIT) != 0);
    h = h_u32(h, ord); h = h_u32(h, rc->payload_len); h = h_u8(h, (fl & SSE_F_TERMINATES) != 0);
    if (!(fl & SSE_F_JSON_OK)) return h;
    h = h_u32(h, rc->n_choices);
    h = h_u32(h, (fl & SSE_F_FINISH_MASK) >> SSE_F_FINISH_SHIFT);
    h = h_u8(h, (fl & SSE_F_HAS_USAGE) != 0);
    if (fl & SSE_F_HAS_USAGE) {
        const sse_usage *u = &res->usages[rc->usage];
        h = h_i64(h, u->prompt_tokens); h = h_i64(h, u->completion_tokens); h = h_i64(h, u->total_tokens);
    }
    h = h_str(h, span(res, rc->content_off, (fl & SSE_F_CONTENT_TEXT) != 0), rc->content_len);
    h = h_u8(h, (fl & SSE_F_TC_NONNIL) != 0); h = h_u8(h, (fl & SSE_F_TC_VALID) != 0);
    h = h_u32(h, rc->tc_count);
    uint32_t t = rc->tc_first;
    for (uint32_t k = 0; k < rc->tc_count; k++) {
        if (t == SSE_NONE || t >= res->n_tcs) { (*inexact) += 1u << 16; break; }      /* chain shorter than tc_count: never equal */
        const sse_tc *c = &res->tcs[t];
        h = h_i64(h, c->index);
        h = h_u8(h, (c->flags & SSE_TC_HAS_ID) != 0);
        if (c->flags & SSE_TC_HAS_ID) h = h_str(h, span(res, c->id_off, (c->flags & SSE_TC_ID_TEXT) != 0), c->id_len);
        h = h_u8(h, (c->flags & SSE_TC_HAS_TYPE) != 0);
        if (c->flags & SSE_TC_HAS_TYPE) h = h_str(h, span(res, c->type_off, (c->flags & SSE_TC_TYPE_TEXT) != 0), c->type_len);
        h = h_u8(h, (c->flags & SSE_TC_HAS_FUNC) != 0);
        h = h_str(h, span(res, c->name_off, (c->flags & SSE_TC_NAME_TEXT) != 0), c->name_len);
        h = h_str(h, span(res, c->args_off, (c->flags & SSE_TC_ARGS_TEXT) != 0), c->args_len);
        t = c->next;
    }
    return h;
}

/* Folds one batch result into the digests: segment i belongs to connection conn[i]. carry_len / seg_flags (per connection)
 * receive the segment's values (seg_flags OR-ed). Returns the number of segments folded. */
uint32_t orc_digest_result(const sse_result *res, const uint32_t *conn, orc_digest *d, uint32_t *carry_len, uint32_t *seg_flags) {
    for (uint32_t i = 0; i < res->n_segs; i++) {
        const sse_seg_result *sr = &res->segs[i];
        orc_digest *D = &d[conn[i]];
        const sse_run *run = &sr->run;
        for (;;) {
            const uint64_t fbase = D->n_frames;
            for (uint32_t f = 0; f < run->frame_count; f++) {
                const sse_frame *fr = &res->frames[run->frame_first + f];
                D->frames_h = h_str(D->frames_h, at(res, fr->off), fr->len); D->n_frames++; D->frame_bytes += fr->len;
            }
            for (uint32_t k = 0; k < run->rec_count; k++) {
                const sse_rec *rc = &res->recs[run->rec_first + k];
                const uint32_t ord = rc->frame == SSE_NONE ? SSE_NONE
                                   : rc->frame - run->frame_first < run->frame_count ? (uint32_t)(fbase + (rc->frame - run->frame_first))
                                   : 0xFFFFFFFEu;
                D->recs_h = h_rec(D->recs_h, res, rc, ord, &D->inexact); D->n_recs++;
            }
            if (run->next == SSE_NONE) break;
            run = &res->runs[run->next];
        }
        carry_len[conn[i]] = sr->carry_len;
        seg_flags[conn[i]] |= sr->flags;
    }
    return res->n_segs;
}

/* ---------------------------------------------------------------- structural check of one batch result */
typedef struct {
    const sse_result *res; const sse_seg *segs; uint32_t flags;
    uint32_t n_viol; char *msg; size_t msg_cap;
    uint8_t *frame_seen, *rec_seen, *run_seen, *tc_seen, *usage_seen, *frame_links;
} ck_state;

/* Counts a violation; the first one is described in msg as "<rule>: seg <i> run <r> index <k>: <detail>" (run -1: the run
 * inline in sse_seg_result, index -1: the rule is about the segment or run as a whole). */
static void viol(ck_state *c, const char *rule, uint32_t seg, int64_t run, int64_t idx, const char *fmt, ...) {
    if (c->n_viol++ == 0 && c->msg && c->msg_cap) {
        int k = snprintf(c->msg, c->msg_cap, "%s: seg %u run %lld index %lld: ", rule, seg, (long long)run, (long long)idx);
        if (k >= 0 && (size_t)k < c->msg_cap) {
            va_list ap; va_start(ap, fmt); vsnprintf(c->msg + k, c->msg_cap - (size_t)k, fmt, ap); va_end(ap);
        }
    }
}

static int in_seg_input(const sse_result *res, const sse_seg *sg, uint32_t off, uint32_t len) {
    if (off < res->in_base) return 0;
    const uint64_t o = (uint64_t)off - res->in_base;
    return o >= sg->in_off && o + len <= (uint64_t)sg->in_off + sg->in_len;
}

/* A span that is not in the text arena lies inside the payload bytes of the record's frame (win_len > 0: [win_off, win_off +
 * win_len)), or, for a record without a frame, inside the segment's input or the out arena's used bytes. */
static void check_span(ck_state *c, uint32_t s, int64_t run, int64_t ri, const char *what, uint32_t off, uint32_t len, int text,
                       int has_frame, uint64_t win_off, uint64_t win_len) {
    const sse_result *res = c->res;
    if (len == 0) return;
    if (text) {
        if ((uint64_t)off + len > res->text_bytes) viol(c, "span.text", s, run, ri, "%s [%u, +%u) past text_bytes %u", what, off, len, res->text_bytes);
        return;
    }
    if (has_frame) {
        if (off < win_off || (uint64_t)off + len > win_off + win_len)
            viol(c, "span.frame", s, run, ri, "%s [%u, +%u) outside the frame's payload [%llu, +%llu)", what, off, len,
                 (unsigned long long)win_off, (unsigned long long)win_len);
    } else if (!in_seg_input(res, &c->segs[s], off, len) && !(off < res->in_base && (uint64_t)off + len <= res->out_bytes)) {
        viol(c, "span.arena", s, run, ri, "%s [%u, +%u) neither in the segment's input nor in out_bytes %u", what, off, len, res->out_bytes);
    }
}

#define REC_KNOWN_FLAGS (0x03FFu | SSE_F_FINISH_MASK)
#define SEG_KNOWN_FLAGS (SSE_SEG_TERMINATED | SSE_SEG_FINISHED | SSE_SEG_LINE_TOO_LONG | SSE_SEG_DEAD | SSE_SEG_DEFERRED)

static void check_rec(ck_state *c, uint32_t s, int64_t run_id, const sse_run *run, uint32_t ri, uint32_t *last_link,
                      uint32_t *n_term, uint32_t *term_rec) {
    const sse_result *res = c->res;
    const sse_seg *sg = &c->segs[s];
    const sse_rec *rc = &res->recs[ri];
    const uint32_t fl = rc->flags, mode = sg->mode;
    const int mode_r = (mode & SSE_MODE_R) != 0;
    const uint32_t fin = (fl & SSE_F_FINISH_MASK) >> SSE_F_FINISH_SHIFT;
    if (fl & ~REC_KNOWN_FLAGS) viol(c, "rec.flags", s, run_id, ri, "unknown flag bits 0x%x", fl & ~REC_KNOWN_FLAGS);
    if (fl & SSE_F_TOO_LONG) viol(c, "rec.too_long", s, run_id, ri, "SSE_F_TOO_LONG is produced by no engine");
    if ((fl & SSE_F_DEPTH_LIMIT) && (fl & SSE_F_JSON_OK)) viol(c, "rec.depth", s, run_id, ri, "SSE_F_DEPTH_LIMIT with SSE_F_JSON_OK");
    if ((fl & SSE_F_DONE_EXACT) && (!(fl & SSE_F_DONE_LINE) || rc->payload_len != 6))
        viol(c, "rec.done_exact", s, run_id, ri, "SSE_F_DONE_EXACT needs SSE_F_DONE_LINE and payload_len 6 (flags 0x%x, payload_len %u)", fl, rc->payload_len);
    if (!(fl & SSE_F_JSON_OK) && ((fl & (SSE_F_HAS_USAGE | SSE_F_TC_NONNIL | SSE_F_TC_VALID | SSE_F_CONTENT_TEXT | SSE_F_FINISH_MASK)) ||
                                  rc->usage != SSE_NONE || rc->tc_count || rc->tc_first != SSE_NONE || rc->content_len))
        viol(c, "rec.not_ok", s, run_id, ri, "a record without SSE_F_JSON_OK carries decoded fields (flags 0x%x)", fl);
    /* the link */
    const sse_frame *fr = 0;
    if (rc->frame != SSE_NONE) {
        if (rc->frame - run->frame_first >= run->frame_count)
            viol(c, "link.range", s, run_id, ri, "frame %u outside the run's frames [%u, +%u)", rc->frame, run->frame_first, run->frame_count);
        else {
            fr = &res->frames[rc->frame];
            c->frame_links[rc->frame]++;
            if (*last_link != SSE_NONE && rc->frame <= *last_link)
                viol(c, "link.order", s, run_id, ri, "frame %u after frame %u in the same run", rc->frame, *last_link);
            *last_link = rc->frame;
        }
        if (fl & SSE_F_DONE_LINE) viol(c, "link.done", s, run_id, ri, "a swallowed [DONE] line linked to frame %u", rc->frame);
    } else if (!mode_r) viol(c, "link.missing", s, run_id, ri, "a mode P|PARSE record without a frame");
    /* payload length against the frame: "data: " + payload + "\n\n" (R), "data: " + payload + "\n" (P|PARSE) */
    uint64_t win_off = 0, win_len = 0;
    if (fr) {
        const uint32_t tail = mode_r ? 2u : 1u;
        if ((uint64_t)fr->len != (uint64_t)rc->payload_len + 6u + tail)
            viol(c, "payload.len", s, run_id, ri, "frame of %u bytes, payload_len %u (mode %u)", fr->len, rc->payload_len, mode);
        win_off = (uint64_t)fr->off + 6u;
        win_len = fr->len >= 6u + tail ? fr->len - 6u - tail : 0;
    }
    /* spans */
    if (rc->content_len == 0 && (fl & SSE_F_CONTENT_TEXT)) viol(c, "span.content_text", s, run_id, ri, "SSE_F_CONTENT_TEXT on empty content");
    check_span(c, s, run_id, ri, "content", rc->content_off, rc->content_len, (fl & SSE_F_CONTENT_TEXT) != 0, fr != 0, win_off, win_len);
    /* usage */
    if (((fl & SSE_F_HAS_USAGE) != 0) != (rc->usage != SSE_NONE))
        viol(c, "usage.flag", s, run_id, ri, "SSE_F_HAS_USAGE %d with usage %u", (fl & SSE_F_HAS_USAGE) != 0, rc->usage);
    if (rc->usage != SSE_NONE) {
        if (rc->usage >= res->n_usages) viol(c, "usage.range", s, run_id, ri, "usage %u >= n_usages %u", rc->usage, res->n_usages);
        else if (c->usage_seen[rc->usage]++) viol(c, "usage.shared", s, run_id, ri, "usage %u has two records", rc->usage);
    }
    /* tool-call chain */
    if ((rc->tc_count == 0) != (rc->tc_first == SSE_NONE))
        viol(c, "tc.first", s, run_id, ri, "tc_count %u with tc_first %u", rc->tc_count, rc->tc_first);
    else if (rc->tc_count) {
        uint32_t t = rc->tc_first, k = 0;
        const uint32_t want = rc->tc_count < 65535u ? rc->tc_count : 0xFFFFFFFFu;      /* saturated: walk to the end */
        int broken = 0;
        while (k < want && t != SSE_NONE) {
            if (t >= res->n_tcs) { viol(c, "tc.range", s, run_id, ri, "element %u of the chain is %u >= n_tcs %u", k, t, res->n_tcs); broken = 1; break; }
            if (c->tc_seen[t]++) { viol(c, "tc.shared", s, run_id, ri, "tool-call element %u is in two chains", t); broken = 1; break; }
            const sse_tc *e = &res->tcs[t];
            if (e->flags & SSE_TC_HAS_ID) check_span(c, s, run_id, ri, "tc.id", e->id_off, e->id_len, (e->flags & SSE_TC_ID_TEXT) != 0, fr != 0, win_off, win_len);
            if (e->flags & SSE_TC_HAS_TYPE) check_span(c, s, run_id, ri, "tc.type", e->type_off, e->type_len, (e->flags & SSE_TC_TYPE_TEXT) != 0, fr != 0, win_off, win_len);
            check_span(c, s, run_id, ri, "tc.name", e->name_off, e->name_len, (e->flags & SSE_TC_NAME_TEXT) != 0, fr != 0, win_off, win_len);
            check_span(c, s, run_id, ri, "tc.args", e->args_off, e->args_len, (e->flags & SSE_TC_ARGS_TEXT) != 0, fr != 0, win_off, win_len);
            t = e->next; k++;
        }
        if (!broken && want != 0xFFFFFFFFu) {
            if (k < want) viol(c, "tc.short", s, run_id, ri, "chain of %u elements, tc_count %u", k, want);
            else if (t != SSE_NONE) viol(c, "tc.end", s, run_id, ri, "chain goes on past tc_count %u (next %u)", want, t);
        } else if (!broken && k < 65535u) viol(c, "tc.short", s, run_id, ri, "saturated tc_count with a chain of %u elements", k);
    }
    /* termination: agent.go:235-242 on an emitted chunk */
    const int term = mode_r && (fl & SSE_F_JSON_OK) && rc->n_choices > 0 && (fin == SSE_FIN_STOP || fin == SSE_FIN_TOOL_CALLS) &&
                     !(fl & SSE_F_DONE_LINE) && rc->frame != SSE_NONE;
    if (term != ((fl & SSE_F_TERMINATES) != 0))
        viol(c, "term.flag", s, run_id, ri, "SSE_F_TERMINATES %d, expected %d (flags 0x%x, n_choices %u)", (fl & SSE_F_TERMINATES) != 0, term, fl, rc->n_choices);
    if (fl & SSE_F_TERMINATES) { (*n_term)++; *term_rec = ri; }
}

/* Structural check of one batch result against the submitted descriptors segs[0 .. res->n_segs) of an engine created with
 * `flags` (sse_config.flags) whose connections hold lines of at most max_line bytes (carry_slot_bytes, or the line pool's
 * max_line_bytes). Returns the number of violations; msg receives the first. */
uint32_t orc_check_result(const sse_result *res, const sse_seg *segs, uint32_t flags, uint32_t max_line, char *msg, size_t msg_cap) {
    ck_state c; memset(&c, 0, sizeof c);
    c.res = res; c.segs = segs; c.flags = flags; c.msg = msg; c.msg_cap = msg_cap;
    if (msg && msg_cap) msg[0] = 0;
    c.frame_seen = (uint8_t *)calloc((size_t)res->n_frames + 1, 1);
    c.frame_links = (uint8_t *)calloc((size_t)res->n_frames + 1, 1);
    c.rec_seen = (uint8_t *)calloc((size_t)res->n_recs + 1, 1);
    c.run_seen = (uint8_t *)calloc((size_t)res->n_runs + 1, 1);
    c.tc_seen = (uint8_t *)calloc((size_t)res->n_tcs + 1, 1);
    c.usage_seen = (uint8_t *)calloc((size_t)res->n_usages + 1, 1);
    if (!c.frame_seen || !c.frame_links || !c.rec_seen || !c.run_seen || !c.tc_seen || !c.usage_seen) abort();
    for (uint32_t s = 0; s < res->n_segs; s++) {
        const sse_seg *sg = &segs[s];
        const sse_seg_result *sr = &res->segs[s];
        const uint32_t sf = sr->flags;
        const int mode_r = (sg->mode & SSE_MODE_R) != 0, parse = mode_r || (sg->mode & SSE_MODE_PARSE);
        if (sf & ~SEG_KNOWN_FLAGS) viol(&c, "seg.flags", s, -1, -1, "unknown flag bits 0x%x", sf & ~SEG_KNOWN_FLAGS);
        if ((sf & SSE_SEG_LINE_TOO_LONG) && !(sf & SSE_SEG_DEAD)) viol(&c, "seg.flags", s, -1, -1, "LINE_TOO_LONG without DEAD (0x%x)", sf);
        if ((sf & SSE_SEG_FINISHED) && (sf & ~SSE_SEG_FINISHED)) viol(&c, "seg.flags", s, -1, -1, "FINISHED with other flags (0x%x)", sf);
        /* DESIGN.md §5 deviation 3: a line after the terminating chunk can fail the connection (LINE_TOO_LONG | DEAD) in the
         * batch the finalize stage then marks TERMINATED; DEAD with TERMINATED is allowed only that way */
        if ((sf & SSE_SEG_TERMINATED) && (sf & SSE_SEG_DEAD) && !(sf & SSE_SEG_LINE_TOO_LONG))
            viol(&c, "seg.flags", s, -1, -1, "DEAD with TERMINATED without LINE_TOO_LONG (0x%x)", sf);
        if (!(flags & SSE_FLAG_DEFER)) {
            if (sf & SSE_SEG_DEFERRED) viol(&c, "seg.deferred", s, -1, -1, "SSE_SEG_DEFERRED without SSE_FLAG_DEFER");
            if (sr->consumed != sg->in_len) viol(&c, "seg.consumed", s, -1, -1, "consumed %u of %u bytes without SSE_FLAG_DEFER", sr->consumed, sg->in_len);
        } else if (sr->consumed > sg->in_len) viol(&c, "seg.consumed", s, -1, -1, "consumed %u > in_len %u", sr->consumed, sg->in_len);
        if (sr->carry_len > max_line) viol(&c, "seg.carry", s, -1, -1, "carry_len %u > longest line %u", sr->carry_len, max_line);
        uint32_t n_term = 0, term_rec = SSE_NONE, last_rec = SSE_NONE, n_frames = 0, n_recs = 0;
        const sse_run *run = &sr->run;
        int64_t run_id = -1;
        for (;;) {
            const int frames_ok = run->frame_count == 0 || (uint64_t)run->frame_first + run->frame_count <= res->n_frames;
            const int recs_ok = run->rec_count == 0 || (uint64_t)run->rec_first + run->rec_count <= res->n_recs;
            if (!frames_ok) viol(&c, "run.frames", s, run_id, -1, "frames [%u, +%u) past n_frames %u", run->frame_first, run->frame_count, res->n_frames);
            if (!recs_ok) viol(&c, "run.recs", s, run_id, -1, "records [%u, +%u) past n_recs %u", run->rec_first, run->rec_count, res->n_recs);
            if (frames_ok) {
                n_frames += run->frame_count;
                for (uint32_t f = run->frame_first; f < run->frame_first + run->frame_count; f++) {
                    if (c.frame_seen[f]++) viol(&c, "frame.shared", s, run_id, f, "frame %u is in two runs", f);
                    const sse_frame *fr = &res->frames[f];
                    if (fr->off < res->in_base) {
                        if ((uint64_t)fr->off + fr->len > res->out_bytes)
                            viol(&c, "frame.out", s, run_id, f, "frame [%u, +%u) past out_bytes %u", fr->off, fr->len, res->out_bytes);
                    } else {
                        if (flags & SSE_FLAG_COPY_OUT) viol(&c, "frame.copy_out", s, run_id, f, "a zero-copy frame under SSE_FLAG_COPY_OUT");
                        if (!in_seg_input(res, sg, fr->off, fr->len))
                            viol(&c, "frame.in", s, run_id, f, "input span [%u, +%u) outside the segment's input [%u, +%u)",
                                 fr->off - res->in_base, fr->len, sg->in_off, sg->in_len);
                    }
                }
            }
            if (recs_ok) {
                n_recs += run->rec_count;
                if (!parse && run->rec_count) viol(&c, "rec.mode_p", s, run_id, run->rec_first, "records in mode P without PARSE");
                uint32_t last_link = SSE_NONE;
                for (uint32_t r = run->rec_first; r < run->rec_first + run->rec_count; r++) {
                    if (c.rec_seen[r]++) { viol(&c, "rec.shared", s, run_id, r, "record %u is in two runs", r); continue; }
                    if (frames_ok) check_rec(&c, s, run_id, run, r, &last_link, &n_term, &term_rec);
                    last_rec = r;
                }
                if (mode_r && frames_ok)
                    for (uint32_t f = run->frame_first; f < run->frame_first + run->frame_count; f++)
                        if (c.frame_links[f] != 1) viol(&c, "link.unique", s, run_id, f, "frame %u has %u records linked to it", f, c.frame_links[f]);
            }
            if (run->next == SSE_NONE) break;
            if (run->next >= res->n_runs) { viol(&c, "run.next", s, run_id, -1, "next %u >= n_runs %u", run->next, res->n_runs); break; }
            if (c.run_seen[run->next]++) { viol(&c, "run.shared", s, run_id, -1, "run %u is referenced twice", run->next); break; }
            run_id = run->next;
            run = &res->runs[run->next];
        }
        if ((sf & SSE_SEG_FINISHED) && (n_frames || n_recs))
            viol(&c, "seg.finished", s, -1, -1, "a FINISHED segment with %u frames and %u records", n_frames, n_recs);
        if (n_term > 1) viol(&c, "term.count", s, -1, term_rec, "%u terminating records", n_term);
        if (n_term && term_rec != last_rec) viol(&c, "term.last", s, -1, term_rec, "the terminating record is not the segment's last (%u)", last_rec);
        if ((n_term != 0) != ((sf & SSE_SEG_TERMINATED) != 0))
            viol(&c, "term.seg", s, -1, term_rec, "%u terminating records, SSE_SEG_TERMINATED %d", n_term, (sf & SSE_SEG_TERMINATED) != 0);
        if (n_term && sr->carry_len) viol(&c, "term.carry", s, -1, term_rec, "a terminated segment holds %u bytes", sr->carry_len);
        if (n_term && sr->consumed != sg->in_len) viol(&c, "term.consumed", s, -1, term_rec, "a terminated segment consumed %u of %u", sr->consumed, sg->in_len);
    }
    free(c.frame_seen); free(c.frame_links); free(c.rec_seen); free(c.run_seen); free(c.tc_seen); free(c.usage_seen);
    return c.n_viol;
}
