// sse_kernel2.cu -- stages 2-4 of the default pipeline: work-item sort, decode, finalize.
//
// The table-driven automaton (v2_round / v2_action / v2_finish_line, in sse_v2.cuh): one lane per line steps a pushdown automaton over the
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
#include "sse_v2.cuh"

namespace {

using namespace ssetab;

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
// Items of at least KParams.long_line payload bytes are kept out of the buckets: they go first, to items_sorted[0, n_long), for the
// long-line kernel, and the decode kernel's first ticket is n_long. Every other item keeps the place it has without them.
constexpr int N_BUCKETS = SSE_N_BUCKETS;
__device__ __forceinline__ bool item_long(const KParams &P, uint32_t y) { return P.long_line && (y & 0x00FFFFFFu) >= P.long_line; }
__device__ __forceinline__ uint32_t item_bucket(const KParams &P, uint32_t y) {
    const uint32_t cls = (y >> 24) & 31u;
    return (((uint32_t)SSE_LEN_BUCKETS - 1u - min((y & 0x00FFFFFFu) >> SSE_LEN_SHIFT, (uint32_t)SSE_LEN_BUCKETS - 1u)) << 5) | cls;
}
__global__ void sse_bucket_hist_kernel(const KParams P) {
    __shared__ uint32_t h[N_BUCKETS], n_long;
    for (int b = threadIdx.x; b < N_BUCKETS; b += blockDim.x) h[b] = 0;
    if (threadIdx.x == 0) n_long = 0;
    __syncthreads();
    const uint32_t n = min(P.ctr->n_items, P.cap_items);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t y = P.items[i].y;
        atomicAdd(item_long(P, y) ? &n_long : &h[item_bucket(P, y)], 1u);
    }
    __syncthreads();
    for (int b = threadIdx.x; b < N_BUCKETS; b += blockDim.x) if (h[b]) atomicAdd(&P.ctr->class_count[b], h[b]);
    if (threadIdx.x == 0 && n_long) atomicAdd(&P.ctr->n_long, n_long);
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
    const uint32_t n_long = P.ctr->n_long;
    if (t == 0 && n_long) P.ctr->item_ticket = n_long;
    uint32_t run = n_long + wsum[t >> 5] + incl - mine;
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
            if (i < n) {
                it[k] = P.items[i];
                rank[k] = item_long(P, it[k].y) ? atomicAdd(&P.ctr->long_cursor, 1u) : atomicAdd(&h[item_bucket(P, it[k].y)], 1u);
            }
        }
        __syncthreads();
        for (int b = threadIdx.x; b < N_BUCKETS; b += SCATTER_TPB) if (h[b]) base[b] = atomicAdd(&P.ctr->class_cursor[b], h[b]);
        __syncthreads();
        #pragma unroll
        for (int k = 0; k < SCATTER_IPT; k++) {
            const uint32_t i = blk + k * SCATTER_TPB + threadIdx.x;
            if (i < n) {
                const uint32_t pos = item_long(P, it[k].y) ? rank[k] : base[item_bucket(P, it[k].y)] + rank[k];
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

// Line pool growth: the pool's arrays were reallocated with pool_pages pages and the first old_pages copied over (page ids and
// chains are unchanged); the new pages go on top of the free stack. One block: every thread reads n_free before any writes it.
__global__ void sse_pool_extend_kernel(const __grid_constant__ KParams P, uint32_t old_pages, uint32_t grow) {
    const uint32_t n = P.pool_hdr->n_free;
    for (uint32_t i = threadIdx.x; i < P.pool_pages - old_pages; i += blockDim.x) P.pool_stack[n + i] = old_pages + i;
    __syncthreads();
    if (threadIdx.x == 0) { P.pool_hdr->n_free = n + (P.pool_pages - old_pages); P.pool_hdr->grow = grow; }
}

// Line pool trim, step 1 (one block; P holds the old arrays, the pool is idle and its `held` pages are all in chains): numbers
// the held pages densely in chain order. An exclusive scan of PoolChain.n_pages gives every connection its first new page, base;
// its chain is rewritten in place (first = base, last = base + n - 1, next'[i] = i + 1) and the old id of its k-th page goes to
// src[base + k]. src is the top `held` entries of the new free stack, above n_free, where nothing reads them once the copy is
// done; its bottom `pages - held` entries become the free pages [held, pages). Carry lengths, and so every connection's offset in
// its last page, are untouched.
__global__ void __launch_bounds__(1024) sse_pool_repack_chains_kernel(const __grid_constant__ KParams P, uint32_t *new_stack,
                                                                      uint32_t *new_next, uint32_t held, uint32_t pages, uint32_t grow) {
    __shared__ uint32_t warp_sum[32];
    const uint32_t t = threadIdx.x, lane = t & 31u, w = t >> 5;
    const uint32_t per = (P.max_conns + blockDim.x - 1) / blockDim.x;
    const uint32_t c0 = min(t * per, P.max_conns), c1 = min(c0 + per, P.max_conns);
    uint32_t n = 0;
    for (uint32_t c = c0; c < c1; c++) n += P.pool_chain[c].n_pages;
    uint32_t x = n;   // inclusive scan over the block: within the warp, then over the warp totals
    for (uint32_t d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(FULL, x, d); if (lane >= d) x += y; }
    if (lane == 31) warp_sum[w] = x;
    __syncthreads();
    if (w == 0) {
        uint32_t s = lane < (blockDim.x >> 5) ? warp_sum[lane] : 0u;
        for (uint32_t d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(FULL, s, d); if (lane >= d) s += y; }
        warp_sum[lane] = s;
    }
    __syncthreads();
    uint32_t base = x - n + (w ? warp_sum[w - 1] : 0u);
    uint32_t *src = new_stack + (pages - held);
    for (uint32_t c = c0; c < c1; c++) {
        PoolChain ch = P.pool_chain[c];
        if (!ch.n_pages) continue;
        uint32_t pg = ch.first;
        for (uint32_t k = 0; k < ch.n_pages; k++) {
            src[base + k] = pg;
            new_next[base + k] = k + 1 < ch.n_pages ? base + k + 1 : SSE_NONE;
            if (k + 1 < ch.n_pages) pg = P.pool_next[pg];
        }
        ch.first = base; ch.last = base + ch.n_pages - 1;
        P.pool_chain[c] = ch;
        base += ch.n_pages;
    }
    for (uint32_t i = t; i < pages - held; i += blockDim.x) new_stack[i] = held + i;
    if (t == 0) { P.pool_hdr->lock = 0; P.pool_hdr->n_free = pages - held; P.pool_hdr->grow = grow; }
}

// Line pool trim, step 2: new page i = old page src[i], for the held pages only, 16 bytes per load and store (page_bytes is a
// multiple of 16). A block copies whole pages, so no thread divides by the page size.
__global__ void __launch_bounds__(256) sse_pool_repack_copy_kernel(const uint4 *__restrict__ old_pool, uint4 *__restrict__ new_pool,
                                                                   const uint32_t *__restrict__ src, uint32_t held, uint32_t vecs_per_page) {
    for (uint32_t p = blockIdx.x; p < held; p += gridDim.x) {
        const uint4 *s = old_pool + (size_t)src[p] * vecs_per_page;
        uint4 *d = new_pool + (size_t)p * vecs_per_page;
        for (uint32_t v = threadIdx.x; v < vecs_per_page; v += blockDim.x) d[v] = s[v];
    }
}

DfaTables *g_tables_dev[16] = { nullptr };

} // namespace

int sse_build_tables(ssetab::DfaTables &T) {
    static_assert(ssetab::N_NODES == N_COUNT, "the field table has a row per schema node");
    static constexpr Schema S = c_schema;     // the host's copy, made at compile time (host code does not read constant memory)
    ssetab::FieldSrc fs[N_FIELDS];
    int n = 0;
    for (int node = 0; node < N_COUNT; node++)
        for (int k = 0; k < S.cnt[node]; k++) {
            const FieldDef &f = S.f[S.first[node] + k];
            fs[n].node = (uint8_t)node; fs[n].name = f.name; fs[n].ty = f.ty; fs[n].sub = f.sub; fs[n].tgt = f.tgt;
            n++;
        }
    // finish_reason values with a code of their own (common_types.go:33-39); any other non-empty value is SSE_FIN_OTHER
    static const char *const fin_names[] = { "stop", "tool_calls", "length", "content_filter", "function_call" };
    static const uint8_t fin_vals[] = { SSE_FIN_STOP, SSE_FIN_TOOL_CALLS, SSE_FIN_LENGTH, SSE_FIN_CONTENT_FILTER, SSE_FIN_FUNCTION_CALL };
    return ssetab::build_tables(T, fs, n, fin_names, fin_vals, 5);
}

int sse_v2_prepare(int device) {
    if (device < 0 || device >= 16) return (int)cudaErrorInvalidValue;
    if (g_tables_dev[device]) return 0;
    static ssetab::DfaTables T;
    if (sse_build_tables(T) != 0) return (int)cudaErrorInvalidValue;
    DfaTables *d = nullptr;
    cudaError_t e = cudaMalloc((void **)&d, sizeof T);
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
    const int el = sse_long_prepare(device);
    if (el != 0) return el;
    g_tables_dev[device] = d;
    return 0;
}

// the decode kernels the context's flags select: templates (KParams.tcache) and counters (KParams.cnt). The long-line kernel
// goes first, alone: the lane decoder fills every SM, so the two could not run side by side.
static void launch_decode_kernel(const KParams &p, cudaStream_t st, int sm_count, int device) {
    const DfaTables *t = g_tables_dev[device];
    if (p.long_line) sse_launch_long_decode(p, t, (void *)st, sm_count, device);
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

int sse_launch_pool_extend(const KParams &p, uint32_t old_pages, bool grow, void *stream) {
    sse_pool_extend_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(p, old_pages, grow ? 1u : 0u);
    return (int)cudaGetLastError();
}

int sse_launch_pool_repack(const KParams &p, uint8_t *pool, uint32_t *stack, uint32_t *next, uint32_t held, uint32_t pages, bool grow,
                           int sm_count, void *stream) {
    sse_pool_repack_chains_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(p, stack, next, held, pages, grow ? 1u : 0u);
    if (held) {
        const uint32_t grid = held < 8u * (uint32_t)sm_count ? held : 8u * (uint32_t)sm_count;   // 8 blocks of 256 fill an SM
        sse_pool_repack_copy_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const uint4 *)p.pool, (uint4 *)pool, stack + (pages - held),
                                                                            held, p.page_bytes / 16u);
    }
    return (int)cudaGetLastError();
}
