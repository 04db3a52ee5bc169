// sse_long.cu -- split pipeline, stage 2a: lines of at least SSE_LONG_LINE payload bytes, decoded by a warp each. Kept in its own
// translation unit so that the lane decoder (sse_kernel2.cu) is compiled exactly as without it.
#include <cuda_runtime.h>
#include <stdint.h>
#include "sse_v2.cuh"

namespace {

using namespace ssetab;

// A lane takes work item `it` (payload offset, length | mode bits, record, segment): the automaton at the start of a document.
__device__ __forceinline__ void lane_begin(const KParams &P, Lane &L, LaneScratch &S, const uint4 it) {
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

// ---------------------------------------------------------------- split pipeline, stage 2a: long lines, a warp each
// A work item of at least KParams.long_line payload bytes (items_sorted[0, n_long)) is decoded by a whole warp. Lane 0 runs the
// automaton as a decode lane does (v2_round, the other 31 lanes idle), and the warp takes over what costs a lane its time on such
// a line: the bodies of strings and digit runs (warp_jump), and the unquoting of every captured string that needs it (queued,
// one job per string, drained by warp_unquote_parallel every ROUNDS rounds). The records are those the lane decoder writes.
constexpr int LONG_WARPS = 4;                 // warps per CTA
constexpr uint32_t LONG_JUMP_MIN = 32;        // body bytes the automaton walks itself first: short strings and numbers stay with it
enum : uint32_t { J_NONE, J_VSTR, J_KSTR, J_DIGITS };

// 16-bit mask of the bytes of v that f flags (f: 0x80 in each flagged byte of a word, exact for every byte)
template <class F>
__device__ __forceinline__ uint32_t mask16(const uint4 &v, F f) {
    return gather4(f(v.x)) | (gather4(f(v.y)) << 4) | (gather4(f(v.z)) << 8) | (gather4(f(v.w)) << 12);
}
__device__ __forceinline__ uint32_t bs4(uint32_t w) { return zero_bytes(w ^ 0x5C5C5C5Cu); }
__device__ __forceinline__ uint32_t quote4(uint32_t w) { return zero_bytes(w ^ 0x22222222u); }
__device__ __forceinline__ uint32_t ctl4(uint32_t w) { return zero_bytes(w & 0xE0E0E0E0u); }
__device__ __forceinline__ uint32_t hi4(uint32_t w) { return w & 0x80808080u; }
__device__ __forceinline__ uint32_t nondigit4x(uint32_t w) {
    const uint32_t x = w ^ 0x30303030u;            // a digit becomes 0..9
    return (((x & 0x7F7F7F7Fu) + 0x76767676u) | x) & 0x80808080u;
}
// bytes k..k+3 of the 28-byte window W (k <= 20)
__device__ __forceinline__ uint32_t word_at(const uint32_t (&W)[7], uint32_t k) {
    const uint32_t i = k >> 2;
    uint32_t a = W[0], b = W[1];
    #pragma unroll
    for (uint32_t m = 1; m < 6u; m++) if (i == m) { a = W[m]; b = W[m + 1]; }
    return __funnelshift_r(a, b, (k & 3u) * 8u);
}
__device__ __forceinline__ bool hex4w(uint32_t w) {
    bool ok = true;
    #pragma unroll
    for (int b = 0; b < 4; b++) ok &= hexval((w >> (8 * b)) & 0xFFu) >= 0;
    return ok;
}
// utf8_valid_len of the bytes of w (avail of them in the payload)
__device__ __forceinline__ uint32_t utf8_len_w(uint32_t w, uint32_t avail) {
    const uint32_t c = w & 0xFFu, s1 = (w >> 8) & 0xFFu, s2 = (w >> 16) & 0xFFu, s3 = w >> 24;
    if (c < 0x80u) return 1;
    if (c >= 0xC2u && c <= 0xDFu) return (avail >= 2u && (s1 & 0xC0u) == 0x80u) ? 2u : 0u;
    if (c >= 0xE0u && c <= 0xEFu) {
        const uint32_t lo = c == 0xE0u ? 0xA0u : 0x80u, hi = c == 0xEDu ? 0x9Fu : 0xBFu;
        return (avail >= 3u && s1 >= lo && s1 <= hi && (s2 & 0xC0u) == 0x80u) ? 3u : 0u;
    }
    if (c >= 0xF0u && c <= 0xF4u) {
        const uint32_t lo = c == 0xF0u ? 0x90u : 0x80u, hi = c == 0xF4u ? 0x8Fu : 0xBFu;
        return (avail >= 4u && s1 >= lo && s1 <= hi && (s2 & 0xC0u) == 0x80u && (s3 & 0xC0u) == 0x80u) ? 4u : 0u;
    }
    return 0;
}

// The automaton is in S_VSTR (J_VSTR), S_KSTR (J_KSTR) or a digit run (J_DIGITS) at p: the warp finds where it has to step again,
// 512 bytes per step (16 per lane, the next step's loads in flight). A digit run ends at its first non-digit, a key body at its
// first '"', '\\', control or non-ASCII byte (what the automaton's own skip stops at). A value body goes on over every escape that
// is well formed and every valid UTF-8 sequence that ends by pe, and ends where the automaton would be in S_VSTR again: at the
// closing quote, a control byte, or the first byte of an escape or sequence the warp does not vouch for. Which backslashes start an
// escape comes from the parity of the backslash runs, carried from lane to lane and step to step; a valid sequence covers at
// most the first 3 bytes of the next lane (lead bytes are never continuation bytes, so each lane knows which sequences of its own
// reach over). Returns the position (warp-uniform); flags: the SF_ESC / SF_HI bits the automaton would have set on the way.
template <bool CNT>
__device__ __forceinline__ uint32_t warp_jump(const uint8_t *__restrict__ base, const uint32_t p, const uint32_t pe, const uint32_t kind,
                                              uint32_t &flags, DTally &C) {
    const uint32_t lane = lane_id();
    auto load = [&](uint32_t off) { return off < pe ? __ldg(reinterpret_cast<const uint4 *>(base + off)) : make_uint4(0u, 0u, 0u, 0u); };
    uint32_t q = p & ~15u, esc_in = 0, cov_in = 0, fl = 0, pos;
    uint4 v = load(q + lane * 16u);
    #pragma unroll 1
    for (;;) {
        if constexpr (CNT) C.add(CN_D_COOP_STEPS, 1);
        const uint32_t off = q + lane * 16u;
        const uint4 nv = load(off + 512u);
        const uint32_t lo = p > off ? min(p - off, 16u) : 0u, hi = pe > off ? min(pe - off, 16u) : 0u;
        const uint32_t live = ((1u << hi) - 1u) & ~((1u << lo) - 1u);       // this lane's bytes of [p, pe)
        uint32_t stop = hi < 16u ? 1u << hi : 0u;                              // pe
        uint32_t B = 0, H = 0;
        if (kind == J_DIGITS) stop |= mask16(v, nondigit4x) & live;
        else if (kind == J_KSTR) stop |= mask16(v, [](uint32_t w) { return bs4(w) | quote4(w) | ctl4(w) | hi4(w); }) & live;
        else {
            const uint32_t sp = mask16(v, [](uint32_t w) { return bs4(w) | quote4(w) | ctl4(w) | hi4(w); }) & live;
            if (!__any_sync(FULL, (sp | stop) != 0u)) {      // 512 plain bytes: no escape or sequence carries into the next step
                esc_in = 0; cov_in = 0;
                q += 512u;
                v = nv;
                continue;
            }
            B = mask16(v, bs4) & live; H = mask16(v, hi4) & live;
            uint32_t bad = mask16(v, ctl4) & live;
            // escapes: a backslash starts one unless an odd run of backslashes stands right before it. The run that ends a lane does
            // not depend on what comes before it unless it fills the lane.
            const uint32_t top = __clz(~(B << 16)) & 1u;
            const unsigned M = __ballot_sync(FULL, B != 0xFFFFu), O = __ballot_sync(FULL, top != 0u);
            const unsigned below = M & ((1u << lane) - 1u);
            const uint32_t cin = below ? (O >> (31u - __clz(below))) & 1u : esc_in;
            esc_in = M ? (O >> (31u - __clz(M))) & 1u : esc_in;
            uint32_t E = 0, S = 0;                                               // escaped bytes, escape starts
            if (B | cin) {
                uint32_t x = cin;
                #pragma unroll
                for (uint32_t j = 0; j < 16u; j++) { const uint32_t st = ((B >> j) & 1u) & (x ^ 1u); E |= x << j; S |= st << j; x = st; }
            }
            bad |= mask16(v, quote4) & live & ~E;
            uint32_t W[7] = { v.x, v.y, v.z, v.w, 0u, 0u, 0u };                // with the next 12 bytes: the next lane's, or the next step's
            {
                uint32_t a = __shfl_down_sync(FULL, v.x, 1), b = __shfl_down_sync(FULL, v.y, 1), c = __shfl_down_sync(FULL, v.z, 1);
                const uint32_t a0 = __shfl_sync(FULL, nv.x, 0), b0 = __shfl_sync(FULL, nv.y, 0), c0 = __shfl_sync(FULL, nv.z, 0);
                if (lane == 31u) { a = a0; b = b0; c = c0; }
                W[4] = a; W[5] = b; W[6] = c;
            }
            #pragma unroll 1
            for (uint32_t m = S; m; m &= m - 1u) {
                const uint32_t j = __ffs(m) - 1u, a = word_at(W, j + 1u), c1 = a & 0xFFu;
                const bool ok = c1 == 'u' ? off + j + 6u <= pe && hex4w(__funnelshift_r(a, word_at(W, j + 5u), 8u))
                                          : off + j + 2u <= pe && (c1 == '"' || c1 == '\\' || c1 == '/' || c1 == 'b' || c1 == 'f' ||
                                                                   c1 == 'n' || c1 == 'r' || c1 == 't');
                if (!ok) bad |= 1u << j;
            }
            uint32_t cov_out = 0;                                                // bytes of the next lane a sequence of this one covers
            #pragma unroll
            for (uint32_t j = 13; j < 16u; j++)
                if ((H >> j) & 1u) { const uint32_t k = utf8_len_w(word_at(W, j), pe - (off + j)); if (j + k > 16u) cov_out = j + k - 16u; }
            uint32_t cov = __shfl_up_sync(FULL, cov_out, 1);
            if (lane == 0) cov = cov_in;
            cov_in = __shfl_sync(FULL, cov_out, 31);
            #pragma unroll 1
            for (uint32_t m = H & ~((1u << cov) - 1u); m; m &= m - 1u) {
                const uint32_t j = __ffs(m) - 1u;
                if (j < cov) continue;
                const uint32_t k = utf8_len_w(word_at(W, j), pe - (off + j));
                if (!k) { bad |= 1u << j; break; }
                cov = j + k;
            }
            stop |= bad;
        }
        const uint32_t first = stop ? (uint32_t)__ffs(stop) - 1u : 16u;
        const unsigned sm = __ballot_sync(FULL, stop != 0u);
        if (kind == J_VSTR) {
            const uint32_t pre = first < 16u ? (1u << first) - 1u : 0xFFFFu;  // this lane's bytes before the stop
            const unsigned upto = sm ? (2u << (__ffs(sm) - 1)) - 1u : FULL;     // the lanes up to the one that stops
            if (__ballot_sync(FULL, (B & pre) != 0u) & upto) fl |= SF_ESC;
            if (__ballot_sync(FULL, (H & pre) != 0u) & upto) fl |= SF_HI;
        }
        if (sm) { pos = __shfl_sync(FULL, off + first, __ffs(sm) - 1); break; }
        q += 512u;
        v = nv;
    }
    flags = fl;
    if constexpr (CNT) { C.add(CN_D_COOP_STRINGS, 1); C.add(CN_D_COOP_BYTES, pos - p); }
    return pos;
}

struct LongSmem {
    DfaTables T;
    LaneScratch ls[LONG_WARPS];
    LongJobs jobs[LONG_WARPS];
};

// CNT: SSE_FLAG_COUNTERS. The counters add into the decode kernel's: a long line is one pull and one item, its jumps are
// cooperative strings / steps / bytes, its automaton rounds are warp rounds with one busy lane.
template <bool CNT>
__global__ void __launch_bounds__(LONG_WARPS * 32, 4)
sse_long_decode_kernel(const __grid_constant__ KParams P, const DfaTables *__restrict__ gT) {
    __shared__ __align__(16) LongSmem cs;
    {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(gT);
        uint32_t *dst = reinterpret_cast<uint32_t *>(&cs.T);
        for (int i = threadIdx.x; i < (int)(sizeof(DfaTables) / 4); i += blockDim.x) dst[i] = src[i];
    }
    __syncthreads();
    const DfaTables &T = cs.T;
    const uint32_t lane = lane_id();
    LaneScratch &S = cs.ls[threadIdx.x >> 5];            // lane 0's
    LongJobs *J = &cs.jobs[threadIdx.x >> 5];
    if (lane == 0) { J->n = 0; S.recp = nullptr; }
    const uint32_t n_long = P.ctr->n_long;

    Lane L; L.busy = false; L.p = L.pe = 0; L.win = make_uint4(0, 0, 0, 0);
    L.st = S_END; L.depth = L.skip = L.sd = 0; L.cur = 0; L.slen = 0; L.sf = 0; L.choices_count = L.n_choices = 0;
    L.finish = 0; L.ct = L.ct1 = L.sstk = 0; L.content_off = L.content_len = 0; L.tc_count = 0; L.tc_first = SSE_NONE;

    DTally C;
    long long t_start = 0;
    if constexpr (CNT) {
        C.t.v = 0;
        __syncwarp();
        t_start = C.last = __shfl_sync(FULL, (long long)clock64(), 0);
    }
    for (;;) {
        uint32_t idx = 0;
        if (lane == 0) idx = atomicAdd(&P.ctr->long_ticket, 1u);
        idx = __shfl_sync(FULL, idx, 0);
        if (idx >= n_long) break;
        if constexpr (CNT) { C.add(CN_D_PULLS, 1); C.add(CN_D_ITEMS, 1); }
        if (lane == 0) {
            lane_begin(P, L, S, P.items_sorted[idx]);
            if (L.p < L.pe) L.win = ldwin16<true>(P.out, L.p);
        }
        if constexpr (CNT) C.mark(CN_C_PULL);
        for (;;) {
            // lane 0 says whether the line goes on (0: done) and which jump the warp takes first (1 + J_*)
            uint32_t go = 0;
            if (lane == 0 && L.busy) {
                const uint32_t st = L.st;
                const uint32_t kind = st == S_VSTR ? J_VSTR : st == S_KSTR ? J_KSTR : (st == S_NINT || st == S_NFRAC || st == S_NEXP) ? J_DIGITS : J_NONE;
                go = 1u + ((L.p < L.pe && L.slen >= LONG_JUMP_MIN) ? kind : (uint32_t)J_NONE);
            }
            go = __shfl_sync(FULL, go, 0);
            if (!go) break;
            if (go - 1u != J_NONE) {
                const uint32_t p = __shfl_sync(FULL, L.p, 0), pe = __shfl_sync(FULL, L.pe, 0);
                uint32_t fl = 0;
                const uint32_t q = warp_jump<CNT>(P.out, p, pe, go - 1u, fl, C);
                if (lane == 0 && q != p) {
                    L.sf |= fl; L.slen += q - p; L.p = q;
                    if (q < pe) L.win = ldwin16<true>(P.out, q);
                }
            }
            if constexpr (CNT) C.mark(CN_C_COOP);
            #pragma unroll 1
            for (int round = 0; round < ROUNDS; round++) {
                v2_round<true, false, CNT>(P, T, L, S, J, 0u, C);
                const bool fin = L.busy && L.p >= L.pe;
                if constexpr (CNT) C.ballot(CN_D_LINES_FINISHED, fin);
                if (fin) {
                    if (v2_finish_line<false>(P, L, S, J)) atomicMin(&P.seg_term[S.slot], S.rec);   // agent.go:235-242, resolved in stage 3
                    L.p = L.pe = 0;
                }
                if constexpr (CNT) C.mark(CN_C_FINISH);
            }
            const uint32_t nj = __shfl_sync(FULL, lane == 0 ? J->n : 0u, 0);      // lane 0 fills the queue
            if (nj) {
                __syncwarp();
                for (uint32_t k = 0; k < nj; k++) {
                    const UnquoteJob jb = J->j[k];
                    if constexpr (CNT) { C.add(CN_D_UNQUOTE_JOBS, 1); C.add(CN_D_UNQUOTE_BYTES, jb.e - jb.s); }
                    warp_unquote_parallel(P.out, jb.s, jb.e, P.text + jb.dst, jb.patch);
                }
                __syncwarp();
                if (lane == 0) J->n = 0;
            }
            if constexpr (CNT) C.mark(CN_C_UNQUOTE);
        }
    }
    if constexpr (CNT) {
        __syncwarp();
        const long long t_end = __shfl_sync(FULL, (long long)clock64(), 0);
        C.add(CN_C_TOTAL, (unsigned long long)(t_end - t_start));
        C.t.flush(P.cnt + CN_DECODE_FIRST, CN_COUNT - CN_DECODE_FIRST);
    }
}

} // namespace

// The counting instantiation has the lower occupancy of the two; its CTAs per SM size the grid of both, which are then all resident.
int sse_long_prepare(LaunchState &ls) {
    int ctas = 0;
    const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, sse_long_decode_kernel<true>, LONG_WARPS * 32, 0);
    if (e != cudaSuccess) return (int)e;
    ls.long_ctas = ctas > 0 ? ctas : 1;
    return 0;
}

// Launched before the lane decoder, alone on the stream: the lane decoder fills every SM, so the two could not run side by side.
void sse_launch_long_decode(const KParams &p, void *stream, LaunchState &ls) {
    const int grid = ls.sm_count * ls.long_ctas;
    const DfaTables *tables = static_cast<const DfaTables *>(ls.tables);
    if (p.cnt) sse_long_decode_kernel<true><<<grid, LONG_WARPS * 32, 0, (cudaStream_t)stream>>>(p, tables);
    else sse_long_decode_kernel<false><<<grid, LONG_WARPS * 32, 0, (cudaStream_t)stream>>>(p, tables);
    ls.launches++;
}
