// sse_kernel2.cu -- stages 2-4 of the default pipeline: work-item sort, decode, finalize.
//
// The table-driven automaton (v2_round / v2_action / v2_finish_line): one lane per line steps a pushdown automaton over the
// payload it reads through a 16-byte register window. Syntax, type compatibility and field capture follow json.Unmarshal into
// CreateChatCompletionStreamResponse; the plain bytes of strings and digit runs are taken a window at a time, and a key is matched
// at its closing quote by a perfect hash of its case-folded bytes; rare cases (escaped keys,
// int/float range checks) fall to the sequential helpers of sse_common.cuh; strings that need unquoting are queued and decoded
// by the whole warp.
//
//   sse_bucket_{hist,scan,scatter}_kernel  counting sort of the produce stage's work items by (length, shape class)
//   sse_decode_kernel                      persistent, one CTA per SM: warps pull 32 sorted items and run the automaton
//   sse_finalize_kernel                    early termination (agent.go:235-242): cut a segment's runs after its terminating chunk
//   sse_decode_kernel<TPL=true>            the same with skeleton-template replay in front of the automaton (SSE_FLAG_TEMPLATES;
//                                          opt-in: measured slower, DESIGN.md 4.2)
//   sse_decode_kernel<TPL, CNT=true>       SSE_FLAG_COUNTERS: the same with per-warp counters and cycle marks (DTally)
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

// Span of a captured string: without escapes it is the payload's own bytes (no call, nothing through local memory); the
// rare decoded case goes through capture() (text-arena allocation + queued warp-cooperative unquote).
__device__ __forceinline__ Span capture_v2(const KParams &P, LaneJobs *J, uint32_t s, uint32_t e, int dec, uint32_t *patch) {
    if (!dec) { Span r; r.off = s; r.len = e - s; r.text = false; return r; }
    ParseCtx cx; cx.jobs = J; cx.sm = P.out; cx.P = &P; cx.S = nullptr; cx.emitted = true; cx.out_delta = 0;
    return capture(cx, (int)s, (int)e, dec, patch);
}

__device__ void v2_flush_tc(const KParams &P, Lane &L, LaneScratch &S, LaneJobs *J) {
    if ((S.tc_flags & SSE_TC_HAS_ID) || ((S.tc_flags & SSE_TC_HAS_FUNC) && (S.name_len || S.args_len))) L.sf |= SF_TCVALID;
    L.sf &= ~SF_TCOPEN;
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

__device__ void v2_elem_begin(const KParams &P, Lane &L, LaneScratch &S, LaneJobs *J) {
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

template <bool REC>
__device__ void v2_null(Lane &L, LaneScratch &S) {
    uint32_t ty = L.cur & 15u, tgt = (L.cur >> 9) & 15u;
    if (ty == TY_TS) { L.sf &= ~SF_GBAD; return; }
    // a reset of captured state is not something a template replays
    if (tgt == TG_CHOICES || (tgt == TG_USAGE && (L.sf & SF_USAGE)) || tgt == TG_TOOLCALLS || tgt == TG_TC_ID || tgt == TG_TC_TYPE || tgt == TG_TC_FUNCTION) rec_nonsimple<REC>(S);
    switch (tgt) {
    case TG_CHOICES:
        L.n_choices = 0; L.choices_count = 0; L.finish = SSE_FIN_NONE; L.content_off = L.content_len = 0;
        L.sf &= ~(SF_CDEC | SF_CBAD | SF_CSET | SF_TCNONNIL | SF_TCOPEN | SF_TCVALID);
        L.tc_count = 0; L.tc_first = SSE_NONE;
        break;
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
template <bool REC>
__device__ bool v2_action(const KParams &P, const DfaTables &T, Lane &L, LaneScratch &S, LaneJobs *J, uint32_t t) {
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
            if (node == A_CHOICES) L.n_choices = L.choices_count;
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
template <bool REC>
__device__ bool v2_finish_line(const KParams &P, Lane &L, LaneScratch &S, LaneJobs *J) {
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
template <bool RO, bool REC, bool CNT>
__device__ __forceinline__ void v2_round(const KParams &P, const DfaTables &T, Lane &L, LaneScratch &S, LaneJobs *J, const uint32_t coop_max,
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

// ---------------------------------------------------------------- split pipeline, stage 2: decode
// Persistent warps pull 32 work items at a time (lines of the same stream are adjacent, so the lanes of a batch walk
// near-identical structure in lockstep); no producer code and no line window in this kernel: small instruction
// footprint, shared memory only for the tables and the cold per-lane state.
#ifndef SSE_V3_WARPS
#define SSE_V3_WARPS 32
#endif
constexpr int V3_WARPS = SSE_V3_WARPS;

// ---------------------------------------------------------------- skeleton templates
// Consecutive chunks of a stream -- and the chunks of every other stream of the same provider -- differ only inside string
// values and integers: keys, punctuation and literals are byte for byte the same. A line the automaton has walked leaves a
// template in the CTA's cache (handed from launch to launch through KParams.tcache): its bytes outside those wildcards, in
// runs, and per wildcard what the parse did with it. A later line whose runs compare equal, and whose wildcards are again a
// well-formed string body / an integer, takes the automaton through exactly the same transitions: its record is the template's
// with its own spans, and the automaton does not have to run. The work items are sorted by shape, so the 32 lanes of a warp
// hold lines of the same template and walk it in step.
//   [0] next | bucket << 16        [1] skeleton bytes | flags << 16 | tc_count << 24     [2] static record flags
//   [3] n_choices | n_items << 16  [4] the last (up to 4) skeleton bytes  [5] their mask
//   n_items items (run length | wildcard kind << 16 | op << 24), 4 words of per-element tool-call flags when tc_count > 0,
//   then the runs (each starts on a word)
constexpr uint32_t T_LIT_MAX = 1024, TF_HAS_USAGE = 1, TF_SIMPLE = 2, T_HDR = 6;

// body of a string value from fp (just behind the opening quote): position of the closing quote, or SSE_NONE when the body
// is not well formed (control byte, bad escape, no closing quote). d2: bit 0 escapes, bit 1 invalid UTF-8.
// 0x80 in some byte of w iff w holds a '"', a '\\', a byte < 0x20 or a byte >= 0x80 (which byte: special_mask4)
__device__ __forceinline__ uint32_t special_any4(uint32_t w) {
    const uint32_t q = w ^ 0x22222222u, b = w ^ 0x5C5C5C5Cu;
    return (((q - 0x01010101u) & ~q) | ((b - 0x01010101u) & ~b) | ((w - 0x20202020u) & ~w) | w) & 0x80808080u;
}
// position of the first special byte of the 16-byte window v at or after byte i (16: none)
__device__ __forceinline__ uint32_t first_special16(const uint4 &v, uint32_t i) {
    const uint32_t s0 = special_mask4(v.x), s1 = special_mask4(v.y), s2 = special_mask4(v.z), s3 = special_mask4(v.w);
    unsigned long long lo = ((unsigned long long)s1 << 32) | s0, hi = ((unsigned long long)s3 << 32) | s2;
    if (i < 8) lo &= ~0ull << (i * 8); else { lo = 0; hi &= ~0ull << ((i - 8) * 8); }
    return lo ? (uint32_t)(__ffsll((long long)lo) - 1) >> 3 : (hi ? 8u + ((uint32_t)(__ffsll((long long)hi) - 1) >> 3) : 16u);
}
// body of a string value from fp (just behind the opening quote): position of the closing quote, or SSE_NONE when the body
// is not well formed (control byte, bad escape, no closing quote). Returns d2 (bit 0 escapes, bit 1 invalid UTF-8) in the
// two top bits of the result's companion word *d2p.
__device__ __noinline__ uint32_t t_scan_string(const uint8_t *base, uint32_t fp, uint32_t pe, uint32_t *d2p) {
    uint32_t p = fp, d2 = 0;
    while (p < pe) {
        uint4 v = __ldg(reinterpret_cast<const uint4 *>(base + (p & ~15u)));
        if ((p & 15u) == 0) {
            // whole windows of plain bytes: two loads in flight, one test per window
            uint4 v2 = __ldg(reinterpret_cast<const uint4 *>(base + p + 16u));
            while (!(special_any4(v.x) | special_any4(v.y) | special_any4(v.z) | special_any4(v.w))) {
                p += 16u;
                if (p >= pe) { *d2p = d2; return SSE_NONE; }
                v = v2;
                v2 = __ldg(reinterpret_cast<const uint4 *>(base + p + 16u));
            }
        }
        const uint32_t jb = first_special16(v, p & 15u);
        const uint32_t q = (p & ~15u) + jb;
        if (jb == 16u) { p = q; continue; }
        if (q >= pe) break;
        const uint32_t c = __ldg(base + q);
        if (c == '"') { *d2p = d2; return q; }
        if (c == '\\') {
            const uint32_t c2 = __ldg(base + q + 1);
            if (q + 2u <= pe && (c2 == '"' || c2 == '\\' || c2 == '/' || c2 == 'b' || c2 == 'f' || c2 == 'n' || c2 == 'r' || c2 == 't')) p = q + 2u;
            else if (c2 == 'u' && q + 6u <= pe && hex4(base + q + 2u) >= 0) p = q + 6u;
            else break;
            d2 |= 1u;
        } else if (c >= 0x80u) {
            const int k = utf8_valid_len(base + q, (int)(pe - q));
            if (k == 0) { d2 |= 2u; p = q + 1u; } else p = q + (uint32_t)k;      // invalid: the automaton flags it (A_BAD_*) and goes on byte by byte
        } else break;                                // control byte
    }
    *d2p = d2;
    return SSE_NONE;
}
// integer from fp: [-] 0 | [1-9][0-9]*; returns its end, or SSE_NONE
__device__ __forceinline__ uint32_t t_scan_int(const uint8_t *base, uint32_t fp, uint32_t pe) {
    uint32_t i = fp;
    if (i < pe && __ldg(base + i) == '-') i++;
    if (i >= pe) return SSE_NONE;
    const uint32_t d0 = __ldg(base + i);
    if (d0 == '0') return i + 1u;
    if (d0 - '1' > 8u) return SSE_NONE;
    i++;
    while (i + 4u <= pe && nondigit4(gload4(base, i)) == 0) i += 4u;
    while (i < pe && (uint32_t)__ldg(base + i) - '0' <= 9u) i++;
    return i;
}
__device__ __noinline__ uint32_t t_finish_code(const uint8_t *base, uint32_t s, uint32_t len, uint32_t d2) {
    if (len == 0) return SSE_FIN_NONE;
    uint8_t tmp[40];
    if (d2) { const uint32_t n = json_unquote(base, (int)s, (int)(s + len), tmp, 32); return (n <= 32) ? classify_finish(tmp, (int)n) : (uint32_t)SSE_FIN_OTHER; }
    if (len > 32u) return SSE_FIN_OTHER;
    for (uint32_t i = 0; i < len; i++) tmp[i] = __ldg(base + s + i);
    return classify_finish(tmp, (int)len);
}

__device__ __forceinline__ void t_elem_begin(const KParams &P, Lane &L, LaneScratch &S, LaneJobs *J, uint32_t static_flags) {
    if (L.sf & SF_TCOPEN) v2_flush_tc(P, L, S, J);
    L.sf |= SF_TCOPEN; L.tc_count++;
    S.tc_index = 0; S.tc_flags = static_flags; S.tc_dec = 0;
    S.id_off = S.id_len = S.type_off = S.type_len = S.name_off = S.name_len = S.args_off = S.args_len = 0;
}

// Walk the line [ps, pe) along template T. APPLY = false: compare the runs, scan the wildcards, take content / finish_reason
// (registers only); true: (after a successful compare) run every capture op into the lane state. SYNC: all lanes of the
// warp are in the call (act: this lane has a line and a candidate) and meet after every item. Returns false when the line
// does not fit. vflags: 0x80000000 an integer needs a range check (second walk).
template <bool APPLY, bool SYNC>
__device__ __forceinline__ bool t_walk(const KParams &P, const uint32_t *T, Lane &L, LaneScratch &S, LaneJobs *J, uint32_t ps, uint32_t pe,
                                       uint32_t &vflags, bool act) {
    const uint8_t *base = P.out;
    const uint32_t n_items = act ? T[3] >> 16 : 0u, tc_count = act ? T[1] >> 24 : 0u;
    const uint32_t *items = T + T_HDR;
    const uint8_t *tc_static = reinterpret_cast<const uint8_t *>(items + n_items);
    const uint32_t *lw = items + n_items + (tc_count ? 4u : 0u);
    uint32_t fp = ps;
    int cur_ord = -1;
    bool ok = act;
    if (!APPLY && act) { L.content_off = L.content_len = 0; L.finish = SSE_FIN_NONE; L.sf &= ~(SF_CDEC | SF_CBAD); }   // captures of an earlier candidate
    #pragma unroll 1
    for (uint32_t i = 0; ; i++) {
        const bool go = ok && i < n_items;
        if (SYNC) { if (!__any_sync(FULL, go)) break; } else if (!go) break;
        if (go) {
            const uint32_t it = items[i];
            const uint32_t lit = it & 0xFFFFu, kind = (it >> 16) & 0xFFu, op = it >> 24;
            if (!APPLY) {
                uint32_t diff = fp + lit > pe ? 1u : 0u;
                if (!diff) {
                    uint32_t j = 0;
                    #pragma unroll 4
                    for (; j + 4u <= lit; j += 4u) diff |= gload4(base, fp + j) ^ lw[j >> 2];
                    if (j < lit) diff |= (gload4(base, fp + j) ^ lw[j >> 2]) & ((1u << ((lit - j) * 8u)) - 1u);
                }
                if (diff) ok = false;
            }
            fp += lit; lw += (lit + 3u) >> 2;
            if (kind == WK_END) { if (!APPLY && fp != pe) ok = false; }
            else if (ok) {
                uint32_t end, d2 = 0;
                if (kind == WK_STR) end = t_scan_string(base, fp, pe, &d2); else end = t_scan_int(base, fp, pe);
                if (end == SSE_NONE) ok = false;
                else {
                    const uint32_t code = op & 15u, ord = op >> 4, len = end - fp;
                    if (!APPLY) {
                        if (code == OP_CONTENT) {
                            L.content_off = fp; L.content_len = len;
                            L.sf = (L.sf & ~(SF_CDEC | SF_CBAD)) | ((d2 & 1u) ? SF_CDEC : 0u) | ((d2 & 2u) ? SF_CBAD : 0u);
                        } else if (code == OP_FINISH) L.finish = t_finish_code(base, fp, len, d2);
                        else if ((code == OP_CHK_I64 || code == OP_CHK_F32) && len > 18u) vflags |= 0x80000000u;
                    } else if (code != OP_NONE) {
                        if (code >= OP_TC_ID && code <= OP_TC_INDEX)
                            while (cur_ord < (int)ord) { cur_ord++; t_elem_begin(P, L, S, J, tc_static[cur_ord]); }
                        int64_t v = 0;
                        switch (code) {
                        case OP_CONTENT:
                            L.content_off = fp; L.content_len = len;
                            L.sf = (L.sf & ~(SF_CDEC | SF_CBAD)) | ((d2 & 1u) ? SF_CDEC : 0u) | ((d2 & 2u) ? SF_CBAD : 0u);
                            break;
                        case OP_FINISH: L.finish = t_finish_code(base, fp, len, d2); break;
                        case OP_TC_ID: S.id_off = fp; S.id_len = len; S.tc_dec = (S.tc_dec & ~3u) | d2; break;
                        case OP_TC_TYPE: S.type_off = fp; S.type_len = len; S.tc_dec = (S.tc_dec & ~12u) | (d2 << 2); break;
                        case OP_TC_NAME: S.name_off = fp; S.name_len = len; S.tc_dec = (S.tc_dec & ~0x30u) | (d2 << 4); break;
                        case OP_TC_ARGS: S.args_off = fp; S.args_len = len; S.tc_dec = (S.tc_dec & ~0xC0u) | (d2 << 6); break;
                        case OP_TC_INDEX: if (parse_i64(base, (int)fp, (int)end, v)) S.tc_index = v; else L.sf |= SF_TYPE; break;
                        case OP_U_PROMPT: if (parse_i64(base, (int)fp, (int)end, v)) S.u_prompt = v; else L.sf |= SF_TYPE; break;
                        case OP_U_COMPLETION: if (parse_i64(base, (int)fp, (int)end, v)) S.u_completion = v; else L.sf |= SF_TYPE; break;
                        case OP_U_TOTAL: if (parse_i64(base, (int)fp, (int)end, v)) S.u_total = v; else L.sf |= SF_TYPE; break;
                        case OP_CHK_I64: if (len > 18u && !parse_i64(base, (int)fp, (int)end, v)) L.sf |= SF_TYPE; break;
                        case OP_CHK_F32: if (len > 18u && f32_overflows(base, (int)fp, (int)end)) L.sf |= SF_TYPE; break;
                        default: break;
                        }
                    }
                    fp = end;
                }
            }
        }
        if (SYNC) __syncwarp();
    }
    if (APPLY && act) {                                // elements without captured fields, and the last element
        while (cur_ord + 1 < (int)tc_count) { cur_ord++; t_elem_begin(P, L, S, J, tc_static[cur_ord]); }
        if (L.sf & SF_TCOPEN) v2_flush_tc(P, L, S, J);
    }
    return ok;
}

__device__ __forceinline__ uint32_t t_bucket(const uint8_t *base, uint32_t ps, uint32_t pe) {
    if (pe - ps < 2u) return 0u;
    return ((uint32_t)__ldg(base + pe - 1u) * 31u + (uint32_t)__ldg(base + pe - 2u)) & (uint32_t)(T_BUCKETS - 1);
}

// Walk the chains: every lane of the warp tries its next candidate in the same iteration (warp-uniform loop), so lanes that
// need more attempts do not fall out of step. off: first candidate per lane (0: none). Returns the template that fits.
__device__ __forceinline__ uint32_t t_find(const KParams &P, TCtx &X, Lane &L, LaneScratch &S, uint32_t off, uint32_t &vflags) {
    uint32_t found = 0;
    const uint32_t plen = L.pe - L.p;
    const uint32_t tail = plen >= 4u ? gload4(P.out, L.pe - 4u) : 0u;
    #pragma unroll 1
    while (__any_sync(FULL, off != 0u)) {
        // candidates whose last skeleton bytes differ from the line's are passed over right here
        while (off && (plen < 4u || ((tail ^ X.store[off + 4u]) & X.store[off + 5u]))) off = X.store[off] & 0xFFFFu;
        uint32_t vf = 0;
        const bool fit = t_walk<false, true>(P, X.store + off, L, S, nullptr, L.p, L.pe, vf, off != 0u);
        if (off) {
            if (fit) { found = off; off = 0; vflags = vf; }
            else off = X.store[off] & 0xFFFFu;
        }
    }
    return found;
}

// The automaton has just retired a line it recorded: turn the recording into a template (the caller holds the build lock).
__device__ __noinline__ void t_build(const KParams &P, TCtx &X, const TRec &R, uint32_t ps, uint32_t pe, uint32_t rec_static, uint32_t tflags,
                                     uint32_t n_choices, uint32_t tc_count, uint32_t tc_first) {
    const uint8_t *base = P.out;
    if (tc_count > 15u || pe - ps < 4u) return;
    const uint32_t n_items = R.n + 1u;
    uint32_t prev = ps, litw = 0, litb = 0;
    for (uint32_t i = 0; i < R.n; i++) {
        const uint32_t s = R.ev[i].start, e = s + R.ev[i].len;
        if (s < prev || e > pe || s - prev > 0xFFFFu) return;
        litw += (s - prev + 3u) >> 2; litb += s - prev; prev = e;
    }
    if (pe - prev > 0xFFFFu) return;
    litw += (pe - prev + 3u) >> 2; litb += pe - prev;
    if (litb > T_LIT_MAX) return;
    const uint32_t words = T_HDR + n_items + (tc_count ? 4u : 0u) + litw;
    const uint32_t off = X.used;
    if (off + words > (uint32_t)TS_WORDS) return;
    uint32_t *T = X.store + off;
    {
        const uint32_t endlit = pe - prev, tn = min(endlit, 4u);
        const uint32_t tmask = tn == 4u ? 0xFFFFFFFFu : tn == 0u ? 0u : ~((1u << ((4u - tn) * 8u)) - 1u);     // the high tn bytes of the last word
        T[4] = gload4(base, pe - 4u) & tmask; T[5] = tmask;
        bool simple = !(tflags & TF_HAS_USAGE) && tc_count == 0;
        for (uint32_t i = 0; i < R.n; i++) { const uint32_t c = R.ev[i].op & 15u; if (c != OP_NONE && c != OP_CONTENT && c != OP_FINISH && c != OP_CHK_I64 && c != OP_CHK_F32) simple = false; }
        if (simple) tflags |= TF_SIMPLE;
    }
    const uint32_t endlit = pe - prev;
    const uint32_t bucket = endlit >= 2u ? t_bucket(base, ps, pe) : (uint32_t)T_BUCKETS;      // ends in a wildcard: the catch-all chain
    T[1] = litb | (tflags << 16) | (tc_count << 24); T[2] = rec_static; T[3] = n_choices | (n_items << 16);
    uint32_t *items = T + T_HDR, *tcs = items + n_items, *lw = tcs + (tc_count ? 4u : 0u);
    if (tc_count) {
        uint32_t w4[4] = { 0, 0, 0, 0 }, t = tc_first, j = 0;
        for (; j < tc_count && t != SSE_NONE; j++) { w4[j >> 2] |= (P.tcs[t].flags & 7u) << ((j & 3u) * 8u); t = P.tcs[t].next; }
        // a chain shorter than tc_count: the tool-call arena was full (the batch is decoded again after it grows, SSE_FLAG_DEFER);
        // the flags of the missing elements are unknown, so no template
        if (j < tc_count) return;
        tcs[0] = w4[0]; tcs[1] = w4[1]; tcs[2] = w4[2]; tcs[3] = w4[3];
    }
    prev = ps;
    for (uint32_t i = 0; i < n_items; i++) {
        const bool last = i + 1u == n_items;
        const uint32_t s = last ? pe : R.ev[i].start;
        const uint32_t lit = s - prev;
        items[i] = lit | ((last ? (uint32_t)WK_END : (uint32_t)R.ev[i].kind) << 16) | ((last ? 0u : (uint32_t)R.ev[i].op) << 24);
        for (uint32_t j = 0; j < lit; j += 4u) {
            uint32_t v = gload4(base, prev + j);
            if (lit - j < 4u) v &= (1u << ((lit - j) * 8u)) - 1u;
            *lw++ = v;
        }
        prev = last ? pe : s + R.ev[i].len;
    }
    // the same skeleton may be there already (stored by another lane meanwhile): identical words
    for (uint32_t o = X.head[bucket]; o; o = X.store[o] & 0xFFFFu) {
        const uint32_t *U = X.store + o;
        bool same = true;
        for (uint32_t i = 1; i < words && same; i++) same = U[i] == T[i];
        if (same) return;
    }
    T[0] = (bucket << 16) | (X.head[bucket] & 0xFFFFu);
    __threadfence_block();
    X.used = off + words;
    X.head[bucket] = off;                                  // published: readers see a complete template
}

struct CtaSmem3 {
    DfaTables T;
    TCtx X;
    LaneScratch ls[V3_WARPS * 32];
    LaneJobs jobs[V3_WARPS * 32];
};
static_assert(sizeof(CtaSmem3) <= 227 * 1024, "shared memory budget");

// CNT: SSE_FLAG_COUNTERS (its own instantiation: with CNT = false every counting statement is compiled out)
template <bool TPL, bool CNT>
__global__ void __launch_bounds__(V3_WARPS * 32, 1)
sse_decode_kernel(const __grid_constant__ KParams P, const DfaTables *__restrict__ gT) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    CtaSmem3 &cs = *reinterpret_cast<CtaSmem3 *>(smem_raw);
    {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(gT);
        uint32_t *dst = reinterpret_cast<uint32_t *>(&cs.T);
        for (int i = threadIdx.x; i < (int)(sizeof(DfaTables) / 4); i += blockDim.x) dst[i] = src[i];
    }
    TCtx &X = cs.X;
    const bool templates = TPL && P.tcache != nullptr;
    {   // the templates learnt by earlier launches (a cache: results never depend on what it holds)
        uint32_t loaded = 1;
        if (templates) loaded = min(max(P.tcache[0], 1u), (uint32_t)TS_WORDS);
        for (uint32_t i = threadIdx.x; i <= (uint32_t)T_BUCKETS; i += blockDim.x) X.head[i] = loaded > 1u ? P.tcache[1u + i] : 0u;
        for (uint32_t i = threadIdx.x; i < loaded; i += blockDim.x) X.store[i] = loaded > 1u ? P.tcache[128u + i] : 0u;
        if (threadIdx.x == 0) { X.used = loaded; X.loaded = loaded; X.rec_busy = 0; X.build_lock = 0; }
    }
    __syncthreads();
    const DfaTables &T = cs.T;
    LaneScratch &S = cs.ls[threadIdx.x];
    LaneJobs *J = &cs.jobs[threadIdx.x];
    LaneJobs *Jw = &cs.jobs[threadIdx.x & ~31u];   // this warp's 32 queues
    J->n = 0;
    S.recp = nullptr;
    const uint32_t lane = lane_id();
    const uint32_t n_items = min(P.ctr->n_items, P.cap_items);
    // Items per warp and pull. A full batch (32) is right when there is more work than warps. A steady-state tick (one short
    // segment per connection) has fewer items than lanes in the grid: the kernel is then bound by the serial latency of a lane
    // walking its line with 2-3 warps per scheduler, so the items are spread over all warps (8 or 16 lanes each) instead.
    uint32_t batch = 32;
    {
        const uint32_t warps = gridDim.x * (uint32_t)V3_WARPS;
        if (n_items < 32u * warps) { const uint32_t per = (n_items + warps - 1u) / warps; batch = per <= 8u ? 8u : (per <= 16u ? 16u : 32u); }
    }

    const uint32_t coop_max = batch < 32u ? 32u : (uint32_t)SSE_COOP;      // see coop_string_skip

    Lane L; L.busy = false; L.p = L.pe = 0; L.win = make_uint4(0, 0, 0, 0);
    L.st = S_END; L.depth = L.skip = L.sd = 0; L.cur = 0; L.slen = 0; L.sf = 0; L.choices_count = L.n_choices = 0;
    L.finish = 0; L.ct = L.ct1 = L.sstk = 0; L.content_off = L.content_len = 0; L.tc_count = 0; L.tc_first = SSE_NONE;
    S.rec = S.frame = S.slot = S.plen = 0;

    DTally C;
    long long t_start = 0;
    if constexpr (CNT) {
        if (blockIdx.x == 0 && threadIdx.x == 0) P.cnt[CN_D_ITEMS_PER_PULL] = batch;
        C.t.v = 0;
        __syncwarp();
        t_start = C.last = __shfl_sync(FULL, (long long)clock64(), 0);
    }
    for (;;) {
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(&P.ctr->item_ticket, batch);
        base = __shfl_sync(FULL, base, 0);
        if (base >= n_items) break;
        const uint32_t idx = base + lane;
        const bool has = lane < batch && idx < n_items;
        if constexpr (CNT) { C.add(CN_D_PULLS, 1); C.ballot(CN_D_ITEMS, has); }
        if (has) {
            const uint4 it = P.items_sorted[idx];
            L.p = it.x; S.plen = it.y & 0x00FFFFFFu; L.pe = it.x + S.plen; S.rec = it.z; S.slot = it.w;   // slot: segment index
            S.frame = P.recs[it.z].frame;
            L.st = S_VAL; L.depth = L.skip = L.sd = 0; L.cur = TY_ROOT | (N_ROOT << 4); L.slen = 0;
            L.sf = ((it.y & 0x80000000u) ? SF_RMODE : 0u) | ((it.y & 0x40000000u) ? SF_DONELINE : 0u);
            L.choices_count = L.n_choices = 0; L.finish = SSE_FIN_NONE; L.ct = L.ct1 = L.sstk = 0;
            L.content_off = L.content_len = 0; L.tc_count = 0; L.tc_first = SSE_NONE;
            S.u_prompt = S.u_completion = S.u_total = 0;
            S.recp = nullptr;
            L.busy = true;
        }
        // ---- a cached skeleton? the chain of the line's bucket first, then the catch-all chain
        if (templates) {
            const bool cand = has && S.plen >= 4u;
            uint32_t vflags = 0, toff = 0;
            uint32_t first = cand ? X.head[t_bucket(P.out, L.p, L.pe)] : 0u;
            #pragma unroll 1
            for (int pass = 0; pass < 2; pass++) {
                const uint32_t f = t_find(P, X, L, S, first, vflags);
                if (f) toff = f;
                const bool miss = cand && !toff && pass == 0;
                first = miss ? X.head[T_BUCKETS] : 0u;
                if (!__any_sync(FULL, first != 0u)) break;
            }
            const uint32_t *Tm = X.store + toff;
            const bool simple = toff && ((Tm[1] >> 16) & TF_SIMPLE) && !(vflags & 0x80000000u);
            const bool full = toff && !simple;
            if (__any_sync(FULL, full)) {              // usage / tool-call / range-check ops: a second walk runs them
                if (full) {
                    L.tc_count = 0; L.tc_first = SSE_NONE; L.finish = SSE_FIN_NONE; L.content_off = L.content_len = 0;
                    L.sf &= ~(SF_CDEC | SF_CBAD);
                    if ((Tm[1] >> 16) & TF_HAS_USAGE) L.sf |= SF_USAGE;
                }
                uint32_t d = 0;
                t_walk<true, true>(P, Tm, L, S, J, L.p, L.pe, d, full);
            }
            if constexpr (CNT) {
                C.ballot(CN_D_TEMPLATE_LINES, toff != 0u); C.ballot(CN_D_LINES_FINISHED, toff != 0u);
                C.lanes(CN_D_TEMPLATE_BYTES, toff ? S.plen : 0u); C.ballot(CN_D_TEMPLATE_MISSES, cand && !toff);
            }
            if (toff) {                                  // the record is written, the lane retires
                L.n_choices = Tm[3] & 0xFFFFu;
                if (Tm[2] & SSE_F_TC_NONNIL) L.sf |= SF_TCNONNIL;
                L.st = S_END; L.depth = 0; L.p = L.pe;
                if (v2_finish_line<false>(P, L, S, J)) atomicMin(&P.seg_term[S.slot], S.rec);
                L.p = L.pe = 0;
            } else if (cand) {
                L.content_off = L.content_len = 0; L.finish = SSE_FIN_NONE; L.sf &= ~(SF_CDEC | SF_CBAD);      // (tried templates left captures behind)
                if (!(L.sf & SF_DONELINE) && X.used + 360u <= (uint32_t)TS_WORDS) {     // the automaton takes the line: let it record a template
                    uint32_t m = X.rec_busy;
                    while ((~m) & ((1u << NREC) - 1u)) {
                        const uint32_t b = (uint32_t)__ffs((~m) & ((1u << NREC) - 1u)) - 1u;
                        const uint32_t old = atomicCAS(&X.rec_busy, m, m | (1u << b));
                        if (old == m) { S.recp = &X.rec[b]; X.rec[b].n = 0; X.rec[b].nonsimple = 0; break; }
                        m = old;
                    }
                }
            }
        }
        if (L.busy && L.p < L.pe) L.win = ldwin16<true>(P.out, L.p);      // the automaton reads the payload through a 16-byte window
        if constexpr (CNT) C.mark(CN_C_PULL);
        for (;;) {
            const bool any_busy = __any_sync(FULL, L.busy);
            if (any_busy) {
                #pragma unroll 1
                for (int round = 0; round < ROUNDS; round++) {
                    v2_round<true, TPL, CNT>(P, T, L, S, J, coop_max, C);
                    if constexpr (CNT) C.ballot(CN_D_LINES_FINISHED, L.busy && L.p >= L.pe);
                    if (L.busy && L.p >= L.pe) {
                        const uint32_t ps = L.pe - S.plen, pe = L.pe;
                        if (v2_finish_line<TPL>(P, L, S, J)) atomicMin(&P.seg_term[S.slot], S.rec);   // agent.go:235-242, resolved in stage 3
                        if (TPL && S.recp) {            // keep the line's skeleton as a template (one lane builds at a time)
                            TRec *R = S.recp;
                            if (!R->nonsimple && !(L.sf & (SF_SYN | SF_TYPE | SF_DEPTH | SF_DONELINE)) && atomicCAS(&X.build_lock, 0u, 1u) == 0u) {
                                t_build(P, X, *R, ps, pe, SSE_F_JSON_OK | ((L.sf & SF_TCNONNIL) ? SSE_F_TC_NONNIL : 0u), (L.sf & SF_USAGE) ? TF_HAS_USAGE : 0u,
                                        L.n_choices, L.tc_count, L.tc_first);
                                __threadfence_block();
                                atomicExch(&X.build_lock, 0u);
                            }
                            atomicAnd(&X.rec_busy, ~(1u << (uint32_t)(R - X.rec)));
                            S.recp = nullptr;
                        }
                        L.p = L.pe = 0;
                    }
                    if constexpr (CNT) C.mark(CN_C_FINISH);
                }
            }
            // strings that need unquoting were queued by the lanes: decode them with the whole warp
            __syncwarp();
            unsigned jm = __ballot_sync(FULL, J->n > 0);
            while (jm) {
                const int leader = __ffs(jm) - 1;
                jm &= jm - 1;
                LaneJobs &LJ = Jw[leader];
                const uint32_t nj = LJ.n;
                for (uint32_t k = 0; k < nj; k++) {
                    const UnquoteJob jb = LJ.j[k];
                    if constexpr (CNT) { C.add(CN_D_UNQUOTE_JOBS, 1); C.add(CN_D_UNQUOTE_BYTES, jb.e - jb.s); }
                    warp_unquote(P.out, jb.s, jb.e, P.text + jb.dst, jb.patch);
                }
                __syncwarp();
                if ((int)lane == leader) LJ.n = 0;
            }
            __syncwarp();
            if constexpr (CNT) C.mark(CN_C_UNQUOTE);
            if (!any_busy) break;
        }
    }
    if constexpr (CNT) {
        __syncwarp();
        const long long t_end = __shfl_sync(FULL, (long long)clock64(), 0);
        C.add(CN_C_TOTAL, (unsigned long long)(t_end - t_start));
        C.t.flush(P.cnt + CN_DECODE_FIRST, CN_COUNT - CN_DECODE_FIRST);
    }
    // one CTA hands what it has learnt to the next launch (all CTAs see the same kinds of lines)
    if (templates && blockIdx.x == 0) {
        __syncthreads();
        const uint32_t used = min(X.used, (uint32_t)TS_WORDS);
        if (used > X.loaded) {
            for (uint32_t i = threadIdx.x; i < used; i += blockDim.x) P.tcache[128u + i] = X.store[i];
            for (uint32_t i = threadIdx.x; i <= (uint32_t)T_BUCKETS; i += blockDim.x) P.tcache[1u + i] = X.head[i];
            __threadfence();
            __syncthreads();
            if (threadIdx.x == 0) P.tcache[0] = used;
        }
    }
}



// ---------------------------------------------------------------- split pipeline, stage 1b: order the work items
// A decode warp takes 32 items and runs until the longest of them is done, so a batch of mixed lengths idles most lanes
// (payloads are lognormal 96..4096 B: in arrival order a batch is 34 % busy). Counting sort by payload length / 64, longest
// bucket first, and within a length bucket by shape class (provider hint x position of the line in its round): batches are then
// 94 % busy, their lanes stop at the same actions, and the long lines do not land on the tail of the kernel.
constexpr int N_BUCKETS = SSE_N_BUCKETS;
__device__ __forceinline__ uint32_t item_bucket(const KParams &P, uint32_t y) {
    const uint32_t cls = (y >> 24) & 31u;
    return (((uint32_t)SSE_LEN_BUCKETS - 1u - min((y & 0x00FFFFFFu) >> SSE_LEN_SHIFT, (uint32_t)SSE_LEN_BUCKETS - 1u)) << 5) | cls;
}
__global__ void sse_bucket_hist_kernel(const KParams P) {
    __shared__ uint32_t h[N_BUCKETS];
    for (int b = threadIdx.x; b < N_BUCKETS; b += blockDim.x) h[b] = 0;
    __syncthreads();
    const uint32_t n = min(P.ctr->n_items, P.cap_items);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        atomicAdd(&h[item_bucket(P, P.items[i].y)], 1u);
    __syncthreads();
    for (int b = threadIdx.x; b < N_BUCKETS; b += blockDim.x) if (h[b]) atomicAdd(&P.ctr->class_count[b], h[b]);
}
constexpr int SCAN_TPB = 1024, SCAN_PER = N_BUCKETS / SCAN_TPB;
static_assert(N_BUCKETS % SCAN_TPB == 0, "bucket count");
__global__ void __launch_bounds__(SCAN_TPB) sse_bucket_scan_kernel(const KParams P) {
    __shared__ uint32_t wsum[32];
    const uint32_t t = threadIdx.x, lane = t & 31u;
    uint32_t c[SCAN_PER], mine = 0;
    #pragma unroll
    for (int k = 0; k < SCAN_PER; k++) { c[k] = P.ctr->class_count[t * SCAN_PER + k]; mine += c[k]; }
    uint32_t incl = mine;
    for (int d = 1; d < 32; d <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, d); if ((int)lane >= d) incl += v; }
    if (lane == 31) wsum[t >> 5] = incl;
    __syncthreads();
    if (t < 32) {
        const uint32_t w = wsum[t];
        uint32_t wi = w;
        for (int d = 1; d < 32; d <<= 1) { const uint32_t v = __shfl_up_sync(FULL, wi, d); if ((int)lane >= d) wi += v; }
        wsum[t] = wi - w;
    }
    __syncthreads();
    uint32_t run = wsum[t >> 5] + incl - mine;
    #pragma unroll
    for (int k = 0; k < SCAN_PER; k++) { P.ctr->class_cursor[t * SCAN_PER + k] = run; run += c[k]; }
}
constexpr int SCATTER_TPB = 256, SCATTER_IPT = 8;   // one block places 2048 consecutive items
__global__ void __launch_bounds__(SCATTER_TPB) sse_bucket_scatter_kernel(const KParams P) {
    __shared__ uint32_t h[N_BUCKETS], base[N_BUCKETS];
    const uint32_t n = min(P.ctr->n_items, P.cap_items);
    for (uint32_t blk = blockIdx.x * (SCATTER_TPB * SCATTER_IPT); blk < n; blk += gridDim.x * (SCATTER_TPB * SCATTER_IPT)) {
        for (int b = threadIdx.x; b < N_BUCKETS; b += SCATTER_TPB) h[b] = 0;
        __syncthreads();
        uint4 it[SCATTER_IPT]; uint32_t rank[SCATTER_IPT];
        #pragma unroll
        for (int k = 0; k < SCATTER_IPT; k++) {
            const uint32_t i = blk + k * SCATTER_TPB + threadIdx.x;
            if (i < n) { it[k] = P.items[i]; rank[k] = atomicAdd(&h[item_bucket(P, it[k].y)], 1u); }
        }
        __syncthreads();
        for (int b = threadIdx.x; b < N_BUCKETS; b += SCATTER_TPB) if (h[b]) base[b] = atomicAdd(&P.ctr->class_cursor[b], h[b]);
        __syncthreads();
        #pragma unroll
        for (int k = 0; k < SCATTER_IPT; k++) {
            const uint32_t i = blk + k * SCATTER_TPB + threadIdx.x;
            if (i < n) {
                const uint32_t pos = base[item_bucket(P, it[k].y)] + rank[k];
                P.items_sorted[pos] = it[k];
            }
        }
        __syncthreads();
    }
}

// ---------------------------------------------------------------- split pipeline, stage 3: early termination
// One thread per segment: cut the segment's runs after the terminating chunk and mark the connection finished
// (everything after it is never read by the reference, mcp/agent.go:235-242 and :169). A finished segment has nothing left to
// resubmit: bytes its batch deferred (SSE_FLAG_DEFER) would be ignored, so the whole segment counts as consumed. Where the
// segment terminates does not depend on the tool-call, usage and text arenas, so this stage is complete even when the decode
// stage ran out of them (and is decoded again by sse_launch_decode).
template <bool CNT>
__global__ void sse_finalize_kernel(const __grid_constant__ KParams P) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= P.n_segs) return;
    const uint32_t trec = P.seg_term[s];
    if (trec == SSE_NONE) return;
    const uint32_t tframe = P.recs[trec].frame;
    sse_seg_result r = P.seg_results[s];
    sse_run *run = &r.run;
    for (;;) {
        if (trec >= run->rec_first && trec < run->rec_first + run->rec_count) {
            run->rec_count = trec - run->rec_first + 1;
            run->frame_count = tframe - run->frame_first + 1;
            run->next = SSE_NONE;
            break;
        }
        if (run->next == SSE_NONE) break;
        run = &P.runs[run->next];
    }
    r.flags = (r.flags | SSE_SEG_TERMINATED) & ~SSE_SEG_DEFERRED;
    r.carry_len = 0;
    r.consumed = P.segs[s].in_len;
    P.seg_results[s] = r;
    const uint32_t conn = P.segs[s].conn;
    // the produce stage kept reading after the terminating chunk and may have pooled a line that is never completed
    if (P.pool_pages && ((volatile PoolChain *)P.pool_chain)[conn].n_pages) {
        pool_lock(P.pool_hdr);
        if constexpr (CNT) atomicAdd(P.cnt + CN_P_POOL_PAGES_RETURNED, (unsigned long long)((volatile PoolChain *)P.pool_chain)[conn].n_pages);
        pool_release_locked(P, conn); pool_unlock(P.pool_hdr);
    }
    ConnState ns; ns.carry_len = 0; ns.flags = CONN_FINISHED;
    P.conns[conn] = ns;
}

// Line pool reset: conn < max_conns returns that connection's pages and clears its state (sse_reset_conn); conn == SSE_NONE
// rebuilds the free stack with every page free (sse_reset_all, context creation; the caller clears the connection states).
__global__ void sse_pool_reset_kernel(const __grid_constant__ KParams P, uint32_t conn) {
    if (conn != SSE_NONE) {
        if (blockIdx.x == 0 && threadIdx.x == 0) {
            pool_lock(P.pool_hdr); pool_release_locked(P, conn); pool_unlock(P.pool_hdr);
            ConnState z; z.carry_len = 0; z.flags = 0;
            P.conns[conn] = z;
        }
        return;
    }
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, nt = gridDim.x * blockDim.x;
    for (uint32_t i = tid; i < P.pool_pages; i += nt) P.pool_stack[i] = i;
    for (uint32_t i = tid; i < P.max_conns; i += nt) { PoolChain z; z.first = z.last = SSE_NONE; z.n_pages = 0; z.pad = 0; P.pool_chain[i] = z; }
    if (tid == 0) { P.pool_hdr->lock = 0; P.pool_hdr->n_free = P.pool_pages; }
}

DfaTables *g_tables_dev[16] = { nullptr };

} // namespace

int sse_v2_prepare(int device) {
    if (device < 0 || device >= 16) return (int)cudaErrorInvalidValue;
    if (g_tables_dev[device]) return 0;
    static Schema keep;   // field names must outlive build_tables
    cudaError_t e = cudaMemcpyFromSymbol(&keep, c_schema, sizeof keep);
    if (e != cudaSuccess) return (int)e;
    static ssetab::FieldSrc fs[N_FIELDS];
    int n = 0;
    for (int node = 0; node < N_COUNT; node++)
        for (int k = 0; k < keep.cnt[node]; k++) {
            const FieldDef &f = keep.f[keep.first[node] + k];
            fs[n].node = (uint8_t)node; fs[n].name = f.name; fs[n].ty = f.ty; fs[n].sub = f.sub; fs[n].tgt = f.tgt;
            n++;
        }
    static const char *fin_names[] = { "stop", "tool_calls", "length", "content_filter", "function_call" };
    static const uint8_t fin_vals[] = { SSE_FIN_STOP, SSE_FIN_TOOL_CALLS, SSE_FIN_LENGTH, SSE_FIN_CONTENT_FILTER, SSE_FIN_FUNCTION_CALL };
    static ssetab::DfaTables T;
    if (ssetab::build_tables(T, fs, n, fin_names, fin_vals, 5) != 0) return (int)cudaErrorInvalidValue;
    DfaTables *d = nullptr;
    e = cudaMalloc((void **)&d, sizeof T);
    if (e != cudaSuccess) return (int)e;
    e = cudaMemcpy(d, &T, sizeof T, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) return (int)e;
    e = cudaFuncSetAttribute(sse_decode_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CtaSmem3));
    if (e != cudaSuccess) return (int)e;
    e = cudaFuncSetAttribute(sse_decode_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CtaSmem3));
    if (e != cudaSuccess) return (int)e;
    e = cudaFuncSetAttribute(sse_decode_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CtaSmem3));
    if (e != cudaSuccess) return (int)e;
    e = cudaFuncSetAttribute(sse_decode_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CtaSmem3));
    if (e != cudaSuccess) return (int)e;
    g_tables_dev[device] = d;
    return 0;
}

// the decode kernel the context's flags select: templates (KParams.tcache) and counters (KParams.cnt)
static void launch_decode_kernel(const KParams &p, cudaStream_t st, int sm_count, int device) {
    const DfaTables *t = g_tables_dev[device];
    if (p.cnt) {
        if (p.tcache) sse_decode_kernel<true, true><<<sm_count, V3_WARPS * 32, sizeof(CtaSmem3), st>>>(p, t);
        else sse_decode_kernel<false, true><<<sm_count, V3_WARPS * 32, sizeof(CtaSmem3), st>>>(p, t);
    } else {
        if (p.tcache) sse_decode_kernel<true, false><<<sm_count, V3_WARPS * 32, sizeof(CtaSmem3), st>>>(p, t);
        else sse_decode_kernel<false, false><<<sm_count, V3_WARPS * 32, sizeof(CtaSmem3), st>>>(p, t);
    }
}

int sse_launch_decode_finalize(const KParams &p, void *stream, int sm_count, int device) {
    sse_bucket_hist_kernel<<<sm_count * 2, 512, 0, (cudaStream_t)stream>>>(p);
    sse_bucket_scan_kernel<<<1, SCAN_TPB, 0, (cudaStream_t)stream>>>(p);
    sse_bucket_scatter_kernel<<<sm_count * 2, SCATTER_TPB, 0, (cudaStream_t)stream>>>(p);
    launch_decode_kernel(p, (cudaStream_t)stream, sm_count, device);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return (int)e;
    const int tpb = 256;
    if (p.cnt) sse_finalize_kernel<true><<<(p.n_segs + tpb - 1) / tpb, tpb, 0, (cudaStream_t)stream>>>(p);
    else sse_finalize_kernel<false><<<(p.n_segs + tpb - 1) / tpb, tpb, 0, (cudaStream_t)stream>>>(p);
    return (int)cudaGetLastError();
}

// SSE_FLAG_DEFER, after the tool-call / usage / text arenas of a batch grew: the decode stage again over the items the sort left
// in items_sorted (the caller has reset the decode counters). Records are rewritten whole, so a second pass gives the records a
// single pass with large enough arenas gives.
int sse_launch_decode(const KParams &p, void *stream, int sm_count, int device) {
    launch_decode_kernel(p, (cudaStream_t)stream, sm_count, device);
    return (int)cudaGetLastError();
}

int sse_launch_pool_reset(const KParams &p, uint32_t conn, void *stream) {
    const uint32_t n = p.pool_pages > p.max_conns ? p.pool_pages : p.max_conns;
    const uint32_t grid = conn != SSE_NONE ? 1u : (n + 255u) / 256u < 1024u ? (n + 255u) / 256u : 1024u;
    sse_pool_reset_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(p, conn);
    return (int)cudaGetLastError();
}
