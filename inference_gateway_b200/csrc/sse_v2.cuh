// sse_v2.cuh -- the decode stage's table-driven automaton (v2_round / v2_action / v2_finish_line) and what it uses: the lane state,
// capture, tool-call element assembly, the per-warp counters (DTally). Shared by the lane decoder (sse_kernel2.cu) and the long-line
// decoder (sse_long.cu), which run it for one lane and one warp per line.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "sse_common.cuh"
#include "sse_tables.h"

namespace {

using namespace ssetab;

#ifndef SSE_ROUNDS
#define SSE_ROUNDS 2
#endif
#ifndef SSE_KSTEPS
#define SSE_KSTEPS 2
#endif
constexpr int ROUNDS = SSE_ROUNDS;   // rounds between refills / busy checks
#ifndef SSE_SKIPW
#define SSE_SKIPW 4
#endif
constexpr int SKIPW = SSE_SKIPW;     // 16-byte windows a lane may cross per step while inside a long string value
constexpr int KSTEPS = SSE_KSTEPS;   // plain automaton steps per round before the pending actions run

// ---- skeleton templates (see "templates" below): what the automaton records while it walks a line
constexpr int TS_WORDS = 4096;             // template store (32-bit words)
constexpr int NREC = 8, REC_MAX = 40;      // lanes recording at the same time; wildcards per template
constexpr int T_BUCKETS = 64;              // buckets by the last two payload bytes (+ one for templates that end in a wildcard)
enum : uint8_t { WK_END = 0, WK_STR = 1, WK_INT = 2 };
enum : uint8_t { OP_NONE = 0, OP_CONTENT, OP_FINISH, OP_TC_ID, OP_TC_TYPE, OP_TC_NAME, OP_TC_ARGS, OP_TC_INDEX,
                 OP_U_PROMPT, OP_U_COMPLETION, OP_U_TOTAL, OP_CHK_I64, OP_CHK_F32 };
struct TRecEv { uint32_t start, len; uint8_t kind, op; uint16_t pad; };
struct TRec { uint32_t n, nonsimple; TRecEv ev[REC_MAX]; };
struct TCtx {                      // per CTA, shared memory
    uint32_t store[TS_WORDS];
    uint32_t head[T_BUCKETS + 1];
    uint32_t used, rec_busy, build_lock, loaded;
    TRec rec[NREC];
};

struct LaneScratch {               // cold per-lane state (usage ints, the tool-call element being assembled)
    int64_t u_prompt, u_completion, u_total, tc_index;
    uint32_t tc_flags, tc_dec, tc_prev;   // tc_prev: the line's last tool-call record (valid once the lane's tc_first is set)
    uint32_t id_off, id_len, type_off, type_len, name_off, name_len, args_off, args_len;
    TRec *recp;                    // the automaton records this line's wildcards here (nullptr: not recording)
    uint32_t rec, frame, slot, plen;   // the work item: record index, frame index, segment, payload length (read at the line's end only)
};
template <bool REC>
__device__ __forceinline__ void rec_event(LaneScratch &S, uint32_t kind, uint32_t start, uint32_t len, uint32_t op) {
    TRec *R = S.recp;
    if (R->n < (uint32_t)REC_MAX) { TRecEv e; e.start = start; e.len = len; e.kind = (uint8_t)kind; e.op = (uint8_t)op; e.pad = 0; R->ev[R->n] = e; R->n++; }
    else R->nonsimple = 1;
}
template <bool REC>
__device__ __forceinline__ void rec_nonsimple(LaneScratch &S) { if (REC && S.recp) S.recp->nonsimple = 1; }
// per-string flags (cleared outside strings) and per-line flags
constexpr uint32_t SF_ESC = 1, SF_HI = 2, SF_BAD = 8, SF_STRMASK = SF_ESC | SF_HI | SF_BAD;
constexpr uint32_t SF_SYN = 0x100, SF_TYPE = 0x200, SF_DEPTH = 0x400, SF_GBAD = 0x800, SF_USAGE = 0x1000,
                   SF_TCNONNIL = 0x2000, SF_TCOPEN = 0x4000, SF_TCVALID = 0x8000, SF_CDEC = 0x10000, SF_RMODE = 0x20000, SF_CBAD = 0x40000, SF_CSET = 0x80000, SF_DONELINE = 0x100000;

struct Lane {
    uint32_t p, pe;                // out-arena offsets of the payload being decoded
    uint4 win;                     // the 16 bytes containing p
    uint32_t st, depth, skip, sd, cur, slen, sf, choices_count, n_choices, finish;
    unsigned long long ct, ct1, sstk;   // container-type bit stack (1 = array), 128 levels
    uint32_t content_off, content_len, tc_count, tc_first;
    bool busy;
};

// RO = false: the bytes were written by another warp of the SAME kernel (fused v2): L2 only. RO = true: the payload arenas are
// read-only for the whole decode kernel, so the window may be cached in L1 (SSE_LDWIN 1).
#ifndef SSE_LDWIN
#define SSE_LDWIN 1
#endif
template <bool RO>
__device__ __forceinline__ uint4 ldwin16(const uint8_t *base, uint32_t off) {
    const uint4 *p = reinterpret_cast<const uint4 *>(base + (off & ~15u));
    return (RO && SSE_LDWIN) ? __ldg(p) : __ldcg(p);
}
__device__ __forceinline__ bool lane_live(const Lane &L) {
    return L.sd >= 3 && ((L.sstk >> 10) & 31ull) == N_CHOICE && L.choices_count == 1;
}
__device__ __forceinline__ uint32_t lane_top(const Lane &L) { return (uint32_t)((L.sstk >> (5 * (L.sd - 1))) & 31ull); }
__device__ __forceinline__ void value_done(Lane &L) {
    if (L.depth == 0) { L.st = S_END; return; }
    const uint32_t d = L.depth - 1;
    const unsigned long long bits = d < 64 ? L.ct : L.ct1;
    L.st = ((bits >> (d & 63u)) & 1ull) ? (uint32_t)S_AFTA : (uint32_t)S_AFTO;
}

__device__ __forceinline__ uint32_t gload4(const uint8_t *base, uint32_t off) {
    const uint32_t *w = reinterpret_cast<const uint32_t *>(base + (off & ~3u));
    return __funnelshift_r(__ldg(w), __ldg(w + 1), (off & 3u) * 8u);
}
// 0x80 in every byte that is not '0'..'9' (exact for the lowest flagged byte only: a byte >= 0x80 may flag the one above it)
__device__ __forceinline__ uint32_t nondigit4(uint32_t w4) {
    return (~((w4 | 0x80808080u) - 0x30303030u) | (w4 + 0x46464646u) | w4) & 0x80808080u;
}
// name id of the unescaped string body [s, s + n) of the payload arena (name_lookup), | 0x100 when it has an upper-case letter
__device__ __noinline__ uint32_t body_name(const uint8_t *base, const DfaTables &T, uint32_t s, uint32_t n) {
    bool upper = false;
    const uint32_t id = name_lookup(T, n, [&](uint32_t i) { return gload4(base, s + i); }, upper);
    return id | (upper ? 0x100u : 0u);
}

// A captured string the decoder has to unquote [s, e) of the payload arena. dec: 1 = has escapes; 2 (or 3) = may also hold
// invalid UTF-8, which Go replaces by U+FFFD (1 byte -> 3). It gets a text-arena allocation of that bound (4-byte aligned) and
// goes on the lane's queue, whose decoded length the warp patches into *patch; when the queue is full the lane decodes it.
__device__ __noinline__ Span capture_text(const KParams &P, LaneJobs *J, uint32_t s, uint32_t e, int dec, uint32_t *patch) {
    Span r;
    const uint32_t raw = e - s;
    r.text = true; r.len = 0; r.off = 0;
    if (raw == 0) return r;
    const uint32_t bound = (((dec & 2) ? 3u * raw : raw) + 3u) & ~3u;
    const uint32_t o = atomicAdd(&P.ctr->text_bytes, bound);
    if (o + bound > P.cap_text) { sse_overflow(P.ctr, SSE_OVF_TEXT); return r; }
    r.off = o;
    if (J->n < (uint32_t)MAX_JOBS) {      // raw > 0 implies decoded > 0
        UnquoteJob &j = J->j[J->n++];
        j.s = s; j.e = e; j.dst = o; j.patch = patch;
        r.len = raw;
        return r;
    }
    r.len = json_unquote_write(P.out, (int)s, (int)e, P.text + o);
    return r;
}
// Span of a captured string: without escapes it is the payload's own bytes (no call, nothing through local memory)
__device__ __forceinline__ Span capture_v2(const KParams &P, LaneJobs *J, uint32_t s, uint32_t e, int dec, uint32_t *patch) {
    if (!dec) { Span r; r.off = s; r.len = e - s; r.text = false; return r; }
    return capture_text(P, J, s, e, dec, patch);
}
// The long-line kernel's unquote queue: long enough that every string to decode goes on it (it is drained every ROUNDS rounds,
// and a round captures at most one tool-call element, 4 strings; a line adds its content once).
constexpr int LONG_JOBS = 4 * ROUNDS + 1;
struct LongJobs { uint32_t n; uint32_t pad; UnquoteJob j[LONG_JOBS]; };
// capture_v2 for the long-line kernel: the same text-arena allocation, and the decode always queued for the warp
__device__ __noinline__ Span capture_v2(const KParams &P, LongJobs *J, uint32_t s, uint32_t e, int dec, uint32_t *patch) {
    Span r;
    if (!dec) { r.off = s; r.len = e - s; r.text = false; return r; }
    const uint32_t raw = e - s;
    r.text = true; r.len = 0; r.off = 0;
    if (raw == 0) return r;
    const uint32_t bound = (((dec & 2) ? 3u * raw : raw) + 3u) & ~3u;
    const uint32_t o = atomicAdd(&P.ctr->text_bytes, bound);
    if (o + bound > P.cap_text) { sse_overflow(P.ctr, SSE_OVF_TEXT); return r; }
    UnquoteJob &j = J->j[J->n++];
    j.s = s; j.e = e; j.dst = o; j.patch = patch;
    r.off = o; r.len = raw;
    return r;
}

template <class Q>
__device__ void v2_flush_tc(const KParams &P, Lane &L, LaneScratch &S, Q *J) {
    if ((S.tc_flags & SSE_TC_HAS_ID) || ((S.tc_flags & SSE_TC_HAS_FUNC) && (S.name_len || S.args_len))) L.sf |= SF_TCVALID;
    L.sf &= ~SF_TCOPEN;
    // a line that can no longer be JSON_OK never has its chain read: an element such as the number in [1,1,...] takes no sse_tc,
    // so every element allocated takes at least 3 payload bytes ("{},")
    if (L.sf & (SF_SYN | SF_TYPE)) return;
    uint32_t idx = atomicAdd(&P.ctr->n_tcs, 1u);
    if (idx >= P.cap_tcs) { sse_overflow(P.ctr, SSE_OVF_TCS); return; }
    sse_tc *rec = &P.tcs[idx];
    Span id = capture_v2(P, J, S.id_off, S.id_off + S.id_len, S.tc_dec & 3, &rec->id_len);
    Span ty = capture_v2(P, J, S.type_off, S.type_off + S.type_len, (S.tc_dec >> 2) & 3, &rec->type_len);
    Span nm = capture_v2(P, J, S.name_off, S.name_off + S.name_len, (S.tc_dec >> 4) & 3, &rec->name_len);
    Span ar = capture_v2(P, J, S.args_off, S.args_off + S.args_len, (S.tc_dec >> 6) & 3, &rec->args_len);
    sse_tc o;
    o.index = S.tc_index;
    o.flags = S.tc_flags | (id.text ? SSE_TC_ID_TEXT : 0) | (ty.text ? SSE_TC_TYPE_TEXT : 0) |
              (nm.text ? SSE_TC_NAME_TEXT : 0) | (ar.text ? SSE_TC_ARGS_TEXT : 0);
    o.next = SSE_NONE;
    o.id_off = id.off; o.id_len = id.len; o.type_off = ty.off; o.type_len = ty.len;
    o.name_off = nm.off; o.name_len = nm.len; o.args_off = ar.off; o.args_len = ar.len;
    *rec = o;            // queued unquote jobs overwrite the *_len fields when the warp drains them
    if (L.tc_first == SSE_NONE) L.tc_first = idx; else P.tcs[S.tc_prev].next = idx;
    S.tc_prev = idx;
}

template <class Q>
__device__ void v2_elem_begin(const KParams &P, Lane &L, LaneScratch &S, Q *J) {
    if (L.skip > 0) { L.cur = TY_SKIP; return; }
    uint32_t nd = lane_top(L);
    if (nd == A_CHOICES) { L.choices_count++; L.cur = TY_STRUCT | (N_CHOICE << 4); }
    else if (nd == A_TOOLCALLS) {
        L.cur = TY_STRUCT | (N_TC << 4);
        if (lane_live(L)) {
            if (L.sf & SF_TCOPEN) v2_flush_tc(P, L, S, J);
            L.sf |= SF_TCOPEN; L.tc_count++;
            S.tc_index = 0; S.tc_flags = 0; S.tc_dec = 0;
            S.id_off = S.id_len = S.type_off = S.type_len = S.name_off = S.name_len = S.args_off = S.args_len = 0;
        }
    }
    else if (nd == A_TOKLP) L.cur = TY_STRUCT | (N_TOKLP << 4);
    else if (nd == A_TOPLP) L.cur = TY_STRUCT | (N_TOPLP << 4);
    else L.cur = TY_INT;
}

// choices[0] starts anew: "choices":null, and the close of an empty "choices" array (decode.go array() sets a fresh slice of
// capacity 0, so a later "choices" array grows new, zeroed storage)
__device__ __forceinline__ void v2_choices_reset(Lane &L) {
    L.n_choices = 0; L.choices_count = 0; L.finish = SSE_FIN_NONE; L.content_off = L.content_len = 0;
    L.sf &= ~(SF_CDEC | SF_CBAD | SF_CSET | SF_TCNONNIL | SF_TCOPEN | SF_TCVALID);
    L.tc_count = 0; L.tc_first = SSE_NONE;
}

template <bool REC>
__device__ void v2_null(Lane &L, LaneScratch &S) {
    uint32_t ty = L.cur & 15u, tgt = (L.cur >> 9) & 15u;
    if (ty == TY_TS) { L.sf &= ~SF_GBAD; return; }
    // a reset of captured state is not something a template replays
    if (tgt == TG_CHOICES || (tgt == TG_USAGE && (L.sf & SF_USAGE)) || tgt == TG_TOOLCALLS || tgt == TG_TC_ID || tgt == TG_TC_TYPE || tgt == TG_TC_FUNCTION) rec_nonsimple<REC>(S);
    switch (tgt) {
    case TG_CHOICES: v2_choices_reset(L); break;
    case TG_USAGE: L.sf &= ~SF_USAGE; S.u_prompt = S.u_completion = S.u_total = 0; break;
    case TG_TOOLCALLS:
        if (lane_live(L)) { L.sf &= ~(SF_TCNONNIL | SF_TCOPEN | SF_TCVALID); L.tc_count = 0; L.tc_first = SSE_NONE; }
        break;
    case TG_TC_ID: if ((L.sf & SF_TCOPEN) && lane_live(L)) { S.tc_flags &= ~SSE_TC_HAS_ID; S.id_off = S.id_len = 0; S.tc_dec &= ~3u; } break;
    case TG_TC_TYPE: if ((L.sf & SF_TCOPEN) && lane_live(L)) { S.tc_flags &= ~SSE_TC_HAS_TYPE; S.type_off = S.type_len = 0; S.tc_dec &= ~12u; } break;
    case TG_TC_FUNCTION:
        if ((L.sf & SF_TCOPEN) && lane_live(L)) { S.tc_flags &= ~SSE_TC_HAS_FUNC; S.name_off = S.name_len = S.args_off = S.args_len = 0; S.tc_dec &= ~0xF0u; }
        break;
    default: break;
    }
}

template <bool REC>
__device__ void v2_number_end(const KParams &P, Lane &L, LaneScratch &S, uint32_t end) {
    const uint32_t ty = L.cur & 15u, tgt = (L.cur >> 9) & 15u;
    const bool is_int = L.st == S_NZERO || L.st == S_NINT;
    const uint32_t start = end - L.slen - 1;
    if (REC && S.recp && is_int) {
        uint32_t op = OP_NONE;
        if (ty == TY_INT) {
            op = OP_CHK_I64;
            if ((L.sf & SF_USAGE) && (tgt == TG_PROMPT || tgt == TG_COMPLETION || tgt == TG_TOTAL)) op = OP_U_PROMPT + (tgt - TG_PROMPT);
            else if (tgt == TG_TC_INDEX && (L.sf & SF_TCOPEN) && lane_live(L) && L.tc_count <= 16u) op = OP_TC_INDEX | ((L.tc_count - 1u) << 4);
        } else if (ty == TY_F32) op = OP_CHK_F32;
        rec_event<REC>(S, WK_INT, start, end - start, op);
    }
    if (ty == TY_INT) {
        if (!is_int) L.sf |= SF_TYPE;
        else if (end - start > 18 || tgt != TG_NONE) {
            int64_t v;
            if (!parse_i64(P.out, (int)start, (int)end, v)) L.sf |= SF_TYPE;
            else if (tgt == TG_PROMPT) S.u_prompt = v;
            else if (tgt == TG_COMPLETION) S.u_completion = v;
            else if (tgt == TG_TOTAL) S.u_total = v;
            else if (tgt == TG_TC_INDEX) { if ((L.sf & SF_TCOPEN) && lane_live(L)) S.tc_index = v; }
        }
    } else if (ty == TY_F32) { if (f32_overflows(P.out, (int)start, (int)end)) L.sf |= SF_TYPE; }
    else if (ty == TY_TS) L.sf |= SF_GBAD;
    else if (ty != TY_SKIP) L.sf |= SF_TYPE;
}

// returns true when the current byte has to be looked up again in the new state
template <bool REC, class Q>
__device__ bool v2_action(const KParams &P, const DfaTables &T, Lane &L, LaneScratch &S, Q *J, uint32_t t) {
    switch (t) {
    case A_OPEN_OBJ: case A_OPEN_ARR: {
        const bool arr = t == A_OPEN_ARR;
        if (L.depth >= 128) { L.sf |= SF_DEPTH | SF_SYN; L.p = L.pe - 1; L.st = S_END; return false; }
        if (L.depth < 64) L.ct = (L.ct & ~(1ull << L.depth)) | ((unsigned long long)arr << L.depth);
        else L.ct1 = (L.ct1 & ~(1ull << (L.depth - 64))) | ((unsigned long long)arr << (L.depth - 64));
        L.depth++;
        const uint32_t ty = L.cur & 15u;
        if (L.skip > 0 || ty == TY_SKIP) L.skip++;
        else {
            const uint32_t okmask = arr ? ((1u << TY_SLICE) | (1u << TY_PSLICE))
                                        : ((1u << TY_STRUCT) | (1u << TY_PSTRUCT) | (1u << TY_ROOT) | (1u << TY_GOOGLE));
            if (!((okmask >> ty) & 1u)) { L.sf |= (ty == TY_TS) ? SF_GBAD : SF_TYPE; L.skip++; }
            else {
                const uint32_t sub = (L.cur >> 4) & 31u, tgt = (L.cur >> 9) & 15u;
                const bool live = lane_live(L);
                L.sstk = (L.sstk & ~(31ull << (5 * L.sd))) | ((unsigned long long)sub << (5 * L.sd));
                L.sd++;
                if (tgt != TG_NONE) {
                    if (tgt == TG_USAGE) L.sf |= SF_USAGE;
                    else if (tgt == TG_TC_FUNCTION) { if (live && (L.sf & SF_TCOPEN)) S.tc_flags |= SSE_TC_HAS_FUNC; }
                    else if (tgt == TG_CHOICES) { if (L.n_choices || L.choices_count) rec_nonsimple<REC>(S); L.choices_count = 0; }
                    else if (tgt == TG_TOOLCALLS) {
                        if (live && (L.sf & SF_TCNONNIL)) rec_nonsimple<REC>(S);
                        if (live) { L.sf = (L.sf | SF_TCNONNIL) & ~(SF_TCOPEN | SF_TCVALID); L.tc_count = 0; L.tc_first = SSE_NONE; }
                    }
                }
                if (sub == N_GOOGLE) L.sf &= ~SF_GBAD;
            }
        }
        L.st = arr ? S_ARR0 : S_OBJ0;
        return false;
    }
    case A_CLOSE_OBJ: case A_CLOSE_ARR: {
        L.depth--;
        if (L.skip > 0) L.skip--;
        else {
            const uint32_t node = lane_top(L);
            L.sd--;
            if (node == A_CHOICES) { if (L.choices_count) L.n_choices = L.choices_count; else v2_choices_reset(L); }
            else if (node == A_TOOLCALLS) { if (lane_live(L) && (L.sf & SF_TCOPEN)) v2_flush_tc(P, L, S, J); }
            else if (node == N_GOOGLE) { if (L.sf & SF_GBAD) L.sf |= SF_TYPE; }
        }
        value_done(L);
        return false;
    }
    case A_KEY_END: {
        uint32_t cur = TY_SKIP;
        if (L.skip == 0) {
            const uint32_t node = lane_top(L);
            if (L.sf & (SF_ESC | SF_HI)) {   // escaped / non-ASCII key: unquote and fold like encoding/json does
                uint8_t tmp[72];
                uint32_t n = json_unquote(P.out, (int)(L.p - L.slen), (int)L.p, tmp, 64);
                int f = (n <= 64) ? match_field(c_schema, (int)node, tmp, (int)n) : -1;
                if (f >= 0) cur = c_schema.f[f].ty | ((uint32_t)c_schema.f[f].sub << 4) | ((uint32_t)c_schema.f[f].tgt << 9);
            } else {
                const uint32_t nm = body_name(P.out, T, L.p - L.slen, L.slen), name = nm & 0xFFu;
                if (name != 0xFFu) {
                    uint32_t f = T.field[node * NNAMES + name];
                    if ((f & FIELD_VALID) && !(node == N_GOOGLE && (nm & 0x100u))) cur = f & 0x1FFFu;
                }
            }
        }
        L.cur = cur;
        L.st = S_COLON;
        return false;
    }
    case A_VSTR_END: {
        const uint32_t ty = L.cur & 15u, tgt = (L.cur >> 9) & 15u;
        uint32_t op = OP_NONE;
        if (ty == TY_STR || ty == TY_PSTR) {
            if (tgt != TG_NONE && lane_live(L)) {
                const uint32_t start = L.p - L.slen, len = L.slen;
                const uint32_t d2 = ((L.sf & SF_ESC) ? 1u : 0u) | ((L.sf & SF_BAD) ? 2u : 0u);
                if (tgt == TG_CONTENT) op = OP_CONTENT; else if (tgt == TG_FINISH) op = OP_FINISH;
                else if ((L.sf & SF_TCOPEN) && (tgt == TG_TC_ID || tgt == TG_TC_TYPE || tgt == TG_NAME || tgt == TG_ARGS)) {
                    if (L.tc_count <= 16u) op = (tgt == TG_TC_ID ? OP_TC_ID : tgt == TG_TC_TYPE ? OP_TC_TYPE : tgt == TG_NAME ? OP_TC_NAME : OP_TC_ARGS) | ((L.tc_count - 1u) << 4);
                    else rec_nonsimple<REC>(S);
                }
                switch (tgt) {
                case TG_CONTENT:
                    L.content_off = start; L.content_len = len;
                    L.sf = (L.sf & ~(SF_CDEC | SF_CBAD)) | SF_CSET | ((d2 & 1u) ? SF_CDEC : 0u) | ((d2 & 2u) ? SF_CBAD : 0u);
                    break;
                case TG_FINISH:
                    if (len == 0) L.finish = SSE_FIN_NONE;
                    else if (!d2) {
                        // the lookup folds ASCII case (it matches keys); finish_reason values compare exactly, and all are lower-case
                        const uint32_t nm = body_name(P.out, T, start, len);      // 0x1xx: upper-case, no finish value
                        const uint32_t fv = nm < 0xFFu ? T.finmap[nm] : 0xFFu;
                        L.finish = fv != 0xFFu ? fv : (uint32_t)SSE_FIN_OTHER;
                    }
                    else {
                        uint8_t tmp[40];
                        uint32_t n = json_unquote(P.out, (int)start, (int)L.p, tmp, 32);
                        L.finish = (n <= 32) ? classify_finish(tmp, (int)n) : (uint32_t)SSE_FIN_OTHER;
                    }
                    break;
                case TG_TC_ID: if (L.sf & SF_TCOPEN) { S.tc_flags |= SSE_TC_HAS_ID; S.id_off = start; S.id_len = len; S.tc_dec = (S.tc_dec & ~3u) | d2; } break;
                case TG_TC_TYPE: if (L.sf & SF_TCOPEN) { S.tc_flags |= SSE_TC_HAS_TYPE; S.type_off = start; S.type_len = len; S.tc_dec = (S.tc_dec & ~12u) | (d2 << 2); } break;
                case TG_NAME: if (L.sf & SF_TCOPEN) { S.name_off = start; S.name_len = len; S.tc_dec = (S.tc_dec & ~0x30u) | (d2 << 4); } break;
                case TG_ARGS: if (L.sf & SF_TCOPEN) { S.args_off = start; S.args_len = len; S.tc_dec = (S.tc_dec & ~0xC0u) | (d2 << 6); } break;
                default: break;
                }
            }
        } else if (ty == TY_TS) L.sf &= ~SF_GBAD;
        else if (ty != TY_SKIP) L.sf |= SF_TYPE;
        if (REC && S.recp) rec_event<REC>(S, WK_STR, L.p - L.slen, L.slen, op);
        value_done(L);
        return false;
    }
    case A_BAD_STAY: L.sf |= SF_BAD; L.st = S_VSTR; return false;
    case A_BAD_REDO: L.sf |= SF_BAD; L.st = S_VSTR; return true;
    case A_NUM_END: v2_number_end<REC>(P, L, S, L.p); value_done(L); return true;
    case A_LIT_TRUE: case A_LIT_FALSE: {
        const uint32_t ty = L.cur & 15u;
        if (ty == TY_TS) L.sf |= SF_GBAD; else if (ty != TY_SKIP) L.sf |= SF_TYPE;
        value_done(L);
        return false;
    }
    case A_LIT_NULL: v2_null<REC>(L, S); value_done(L); return false;
    case A_ELEM_REDO: v2_elem_begin(P, L, S, J); L.st = S_VAL; return true;
    case A_COMMA_ARR: v2_elem_begin(P, L, S, J); L.st = S_VAL; return false;
    default:   // A_ERR
        L.sf |= SF_SYN; L.p = L.pe - 1; L.st = S_END;
        return false;
    }
}

// A line retires: final syntax check, record, termination bookkeeping (agent.go:205-242).
template <bool REC, class Q>
__device__ bool v2_finish_line(const KParams &P, Lane &L, LaneScratch &S, Q *J) {
    bool terminates = false;
    if (!(L.sf & SF_SYN)) {
        if (L.depth == 0 && (L.st == S_NZERO || L.st == S_NINT || L.st == S_NFRAC || L.st == S_NEXP)) {
            v2_number_end<REC>(P, L, S, L.pe);
            L.st = S_END;
        }
        if (L.st != S_END) L.sf |= SF_SYN;
    }
    sse_rec r;
    r.frame = S.frame; r.flags = 0; r.content_off = r.content_len = 0; r.tc_first = SSE_NONE; r.tc_count = 0; r.n_choices = 0;
    r.usage = SSE_NONE;
    if (L.sf & SF_DEPTH) r.flags |= SSE_F_DEPTH_LIMIT;
    if (L.sf & SF_DONELINE) r.flags |= SSE_F_DONE_LINE;      // swallowed by the reframe, parsed for agent.go:377-402
    if (!(L.sf & (SF_SYN | SF_TYPE))) {
        r.flags |= SSE_F_JSON_OK;
        r.n_choices = (uint16_t)min(L.n_choices, 0xFFFFu);
        if (L.sf & SF_USAGE) {
            uint32_t idx = atomicAdd(&P.ctr->n_usages, 1u);
            if (idx < P.cap_usages) {
                sse_usage u; u.prompt_tokens = S.u_prompt; u.completion_tokens = S.u_completion; u.total_tokens = S.u_total;
                P.usages[idx] = u; r.usage = idx; r.flags |= SSE_F_HAS_USAGE;
            } else sse_overflow(P.ctr, SSE_OVF_USAGES);
        }
        if (L.n_choices > 0) {
            Span ct = capture_v2(P, J, L.content_off, L.content_off + L.content_len, ((L.sf & SF_CDEC) ? 1 : 0) | ((L.sf & SF_CBAD) ? 2 : 0),
                                 &P.recs[S.rec].content_len);
            r.content_off = ct.len ? ct.off : 0; r.content_len = ct.len;
            if (ct.text && ct.len) r.flags |= SSE_F_CONTENT_TEXT;
            r.flags |= L.finish << SSE_F_FINISH_SHIFT;
            if (L.sf & SF_TCNONNIL) r.flags |= SSE_F_TC_NONNIL;
            if (L.sf & SF_TCVALID) r.flags |= SSE_F_TC_VALID;
            r.tc_first = L.tc_count ? L.tc_first : SSE_NONE;
            r.tc_count = (uint16_t)min(L.tc_count, 0xFFFFu);
            if ((L.sf & SF_RMODE) && (L.finish == SSE_FIN_STOP || L.finish == SSE_FIN_TOOL_CALLS)) {
                r.flags |= SSE_F_TERMINATES;
                terminates = true;
            }
        }
    }
    r.payload_len = S.plen;
    P.recs[S.rec] = r;
    L.busy = false;
    return terminates;
}

// ---- SSE_FLAG_COUNTERS (the counting instantiation only): a warp's decode counters, one per lane (WarpTally from CN_DECODE_FIRST),
// and the clock of its last mark. mark(k) charges the cycles since the previous mark to bucket k: the warp is converged there and
// lane 0's clock is the warp's.
struct DTally {
    WarpTally t;
    long long last;
    __device__ __forceinline__ void add(uint32_t k, unsigned long long x) { t.add(k - CN_DECODE_FIRST, x); }
    __device__ __forceinline__ void lanes(uint32_t k, uint32_t x) { add(k, __reduce_add_sync(FULL, x)); }   // sum over the lanes
    __device__ __forceinline__ void ballot(uint32_t k, bool x) { add(k, (uint32_t)__popc(__ballot_sync(FULL, x))); }
    __device__ __forceinline__ void mark(uint32_t k) {
        __syncwarp();
        const long long now = __shfl_sync(FULL, (long long)clock64(), 0);
        add(k, (unsigned long long)(now - last));
        last = now;
    }
};

// ---- stragglers inside a long string value. A lane skips at most SKIPW windows of a string per round, so a 4 KB value costs it
// 64 rounds while the lanes with shorter lines have retired and the warp runs almost empty; the length of a nearly empty launch (a
// steady-state tick) is exactly that walk. When at most SSE_COOP lanes of the warp (any number of them when the launch has fewer
// items than the grid has lanes: then latency is all there is) are still inside the plain bytes of a string after their own skip,
// the WHOLE warp finishes each of those strings: 32 lanes x 16 bytes = 512 contiguous bytes per step
// (coalesced, independent loads), the first lane that sees a '"', '\\', control or non-ASCII byte -- or the end of the payload --
// gives the stop. Same result as the per-lane skip: the position of the next special byte.
#ifndef SSE_COOP
#define SSE_COOP 8
#endif
__device__ __forceinline__ uint32_t first_special16_from0(const uint4 &v) {     // index of the first special byte of v, 16: none
    const uint32_t s0 = special_mask4(v.x), s1 = special_mask4(v.y), s2 = special_mask4(v.z), s3 = special_mask4(v.w);
    const unsigned long long lo = ((unsigned long long)s1 << 32) | s0, hi = ((unsigned long long)s3 << 32) | s2;
    return lo ? (uint32_t)(__ffsll((long long)lo) - 1) >> 3 : (hi ? 8u + ((uint32_t)(__ffsll((long long)hi) - 1) >> 3) : 16u);
}
template <bool RO, bool CNT>
__device__ __forceinline__ void coop_string_skip(const KParams &P, Lane &L, unsigned mm, DTally &C) {
    const uint32_t lane = lane_id();
    #pragma unroll 1
    while (mm) {
        const int src = __ffs(mm) - 1;
        mm &= mm - 1;
        uint32_t q = __shfl_sync(FULL, L.p, src);                 // 16-byte aligned: the lane's own skip stopped at a window border
        const uint32_t qe = __shfl_sync(FULL, L.pe, src);
        const uint32_t q0 = q;
        uint32_t pos;
        #pragma unroll 1
        for (;;) {
            if constexpr (CNT) C.add(CN_D_COOP_STEPS, 1);
            const uint32_t off = q + lane * 16u;
            uint32_t stop = 0xFFFFFFFFu;                         // where this lane's 16 bytes end the run (none: they are all plain)
            if (off >= qe) stop = qe;
            else {
                const uint32_t j = first_special16_from0(ldwin16<RO>(P.out, off));
                if (off + j >= qe) stop = qe; else if (j < 16u) stop = off + j;
            }
            const unsigned hm = __ballot_sync(FULL, stop != 0xFFFFFFFFu);
            if (hm) { pos = __shfl_sync(FULL, stop, __ffs(hm) - 1); break; }
            q += 512u;
        }
        if constexpr (CNT) { C.add(CN_D_COOP_STRINGS, 1); C.add(CN_D_COOP_BYTES, pos - q0); }
        if ((int)lane == src) {
            L.slen += pos - L.p; L.p = pos;
            if (L.p < L.pe) L.win = ldwin16<RO>(P.out, L.p);
        }
    }
}

// One round of the per-lane automaton: KSTEPS plain steps, then the pending action (if any) of every lane.
template <bool RO, bool REC, bool CNT, class Q>
__device__ __forceinline__ void v2_round(const KParams &P, const DfaTables &T, Lane &L, LaneScratch &S, Q *J, const uint32_t coop_max,
                                         DTally &C) {
    uint32_t pend = 0;                       // action | cls << 8 | in_str << 16 | in_tok << 17
    uint32_t n_win = 0, n_plain = 0, n_act = 0, p0 = 0;      // (CNT) this lane's windows of phase A, steps, v2_action calls
    if constexpr (CNT) { C.add(CN_D_WARP_ROUNDS, 1); C.ballot(CN_D_BUSY_LANE_ROUNDS, L.busy); p0 = L.p; }
    // phase A (once per round, only the lanes inside a string or a digit run): jump over the plain bytes -- to the next '"',
    // '\\', control or non-ASCII byte of a key or value string, or to the next non-digit of an integer, fraction or exponent --
    // up to SKIPW windows. The automaton would walk those bytes without changing its state or flags; the key's or value's
    // bytes are read again where its end needs them (A_KEY_END, finish_reason). Keeping it out of the step loop means a warp
    // whose lanes are not all in the same phase executes this path once per round, not once per step.
    bool more = false;                       // still inside the plain bytes of a string after SKIPW windows
    const bool str_run = L.st == S_VSTR || L.st == S_KSTR;
    if (L.p < L.pe && (str_run || L.st == S_NINT || L.st == S_NFRAC || L.st == S_NEXP)) {
        int w = 0;
        #pragma unroll 1
        for (; w < SKIPW; w++) {
            if constexpr (CNT) n_win++;
            const uint32_t i = L.p & 15u;
            uint32_t s0, s1, s2, s3;
            if (str_run) { s0 = special_mask4(L.win.x); s1 = special_mask4(L.win.y); s2 = special_mask4(L.win.z); s3 = special_mask4(L.win.w); }
            else { s0 = nondigit4(L.win.x); s1 = nondigit4(L.win.y); s2 = nondigit4(L.win.z); s3 = nondigit4(L.win.w); }
            if (i == 0 && (s0 | s1 | s2 | s3) == 0 && L.p + 16u <= L.pe) {      // a whole window of plain bytes
                L.p += 16u; L.slen += 16u;
                if (L.p >= L.pe) break;
                L.win = ldwin16<RO>(P.out, L.p);
                continue;
            }
            unsigned long long lo = ((unsigned long long)s1 << 32) | s0;
            unsigned long long hi = ((unsigned long long)s3 << 32) | s2;
            if (i < 8) lo &= ~0ull << (i * 8); else { lo = 0; hi &= ~0ull << ((i - 8) * 8); }
            const uint32_t j = lo ? (uint32_t)(__ffsll((long long)lo) - 1) >> 3 : (hi ? 8u + ((uint32_t)(__ffsll((long long)hi) - 1) >> 3) : 16u);
            const uint32_t n = min(j - i, L.pe - L.p);
            if (n == 0) break;
            L.p += n; L.slen += n;
            if ((L.p & 15u) != 0 || L.p >= L.pe) break;     // stopped at a special byte or at the end of the payload
            L.win = ldwin16<RO>(P.out, L.p);
        }
        more = str_run && w == SKIPW;
    }
    if constexpr (CNT) { C.lanes(CN_D_SKIP_WINDOWS, n_win); C.lanes(CN_D_SKIP_BYTES, L.p - p0); C.mark(CN_C_SKIP); }
    if (SSE_COOP) {
        const unsigned mm = __ballot_sync(FULL, more);
        if (mm && (uint32_t)__popc(mm) <= coop_max) coop_string_skip<RO, CNT>(P, L, mm, C);
    }
    if constexpr (CNT) C.mark(CN_C_COOP);
    // phase B: plain automaton steps
    #pragma unroll
    for (int k = 0; k < KSTEPS; k++) {
        if (L.p < L.pe && pend == 0) {
            const uint32_t wsel = (L.p >> 2) & 3u;
            const uint32_t w01 = (wsel & 1u) ? L.win.y : L.win.x, w23 = (wsel & 1u) ? L.win.w : L.win.z;
            const uint32_t w = (wsel & 2u) ? w23 : w01;
            const uint32_t c = (w >> ((L.p & 3u) * 8u)) & 0xFFu;
            const uint32_t e = T.clssym[c];
            const uint32_t cls = e & 63u;
            const bool in_str = L.st >= S_KSTR, in_tok = L.st >= S_NMINUS;
            const uint32_t t = T.tr[L.st * NCLS + cls];
            if (t < A_FIRST) {
                if constexpr (CNT) n_plain++;
                L.sf = in_str ? (L.sf | (e >> 13)) : (L.sf & ~SF_STRMASK);
                L.slen = in_tok ? L.slen + 1 : 0;
                L.st = t;
                L.p++;
                if ((L.p & 15u) == 0 && L.p < L.pe) L.win = ldwin16<RO>(P.out, L.p);
            } else pend = t | (cls << 8) | (in_str ? 0x10000u : 0u) | (in_tok ? 0x20000u : 0u);
        }
    }
    if (pend) {
        uint32_t t = pend & 0xFFu;
        const uint32_t cls = (pend >> 8) & 0xFFu;
        if constexpr (CNT) p0 = L.p;
        for (;;) {
            if constexpr (CNT) n_act++;
            if (!v2_action<REC>(P, T, L, S, J, t)) break;         // the action chose the next state
            t = T.tr[L.st * NCLS + cls];                     // redo: same byte, new state
            if (t < A_FIRST) { L.st = t; break; }
        }
        const bool in_str = (pend & 0x10000u) != 0;
        const uint32_t nf = (cls == C_BSLASH ? SF_ESC : 0u) | (cls >= C_H80 ? SF_HI : 0u);
        L.sf = in_str ? (L.sf | nf) : (L.sf & ~SF_STRMASK);
        if constexpr (CNT) p0 = L.p - p0;            // bytes a syntax or depth error jumped over (L.p = L.pe - 1)
        L.slen = (pend & 0x20000u) ? L.slen + 1 : 0;
        L.p++;
        if ((L.p & 15u) == 0 && L.p < L.pe) L.win = ldwin16<RO>(P.out, L.p);
    }
    if constexpr (CNT) {
        C.lanes(CN_D_PLAIN_STEPS, n_plain); C.lanes(CN_D_ACTIONS, pend ? 1u : 0u);
        C.lanes(CN_D_ACTION_REDOS, n_act ? n_act - 1u : 0u); C.lanes(CN_D_ABANDONED_BYTES, pend ? p0 : 0u);
        C.mark(CN_C_STEPS);
    }
}

} // namespace
