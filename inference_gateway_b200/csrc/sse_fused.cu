// sse_fused.cu -- the single-pass tile kernel (SSE_FLAG_KERNEL_FUSED): ONE pass over the input arena (plan kernel + fused
// tile kernel).
//
// A CTA owns a tile: up to 48 KiB (TILE) of consecutive connection segments (carry tail of the previous batch + new bytes),
// staged from HBM into shared memory by 1-D bulk copies (cp.async.bulk, one per segment, completion on an mbarrier).
// Everything the reference does per line happens on that tile, so the payload crosses HBM exactly once:
//
//   stage 1a  all warps, 512-byte slices, 16 bytes per lane: SWAR byte classification -> "stop" bitmap (1 bit per byte:
//             '"', '\\', '[', byte < 0x20, byte >= 0x80), gathered with dp4a
//   stage 1b  newline bits = stop bits whose byte is '\n'; block-wide scan -> line table in position order
//             (provider.go:322 ReadBytes('\n')); one thread per line classifies it: strings.TrimSpace, "data: ",
//             verbatim (mode P, routes.go:613) or reframe (mode R, agent.go:178-197); zero-copy decision
//   alloc     one atomicAdd per tile and result arena (records, materialised bytes, frames)
//   stage 2   one lane per line to decode: the json.Unmarshal automaton (sse_tables.h) over the tile. Inside a string it
//             jumps from stop bit to stop bit (a clean string costs two steps whatever its length); keys and
//             finish_reason values are matched by word compares against the struct-tag table; "[DONE]" (agent.go:181) is
//             looked for at the '[' stops it passes anyway; strings that need unquoting are decoded by the whole warp
//   finish    early termination (agent.go:235-242) cuts the segment's lines inside the CTA; frame table; the frames that
//             do not stand in the input as they must be sent go through the warp-cooperative serializer; unterminated
//             tails go back to the connection's carry slot (what bufio.Reader would hold)
//
// A segment that does not fit a tile (carry + bytes > TILE) is walked window by window by one CTA (restart at the
// unterminated line); a line longer than carry_slot_bytes (<= TILE - 32 = 49,120, sse_fused_max_line) fails the connection
// loudly.
// Pure integer/byte work, no tensor cores.
#include <cuda_runtime.h>
#include <stdint.h>
#include "sse_common.cuh"
#include "sse_tables.h"

namespace {

using namespace ssetab;

constexpr int F_THREADS = 512;
constexpr int F_WARPS = F_THREADS / 32;
constexpr int F_CTAS_PER_SM = 2;           // persistent: the grid is this many CTAs per SM, all resident
constexpr uint32_t TILE = 49152;
constexpr uint32_t TILE_PAD = 64;
constexpr uint32_t BM_WORDS = TILE / 32;
constexpr int MAX_TSEGS = 96;
constexpr int LCAP = F_THREADS;            // lines per round: one thread per line
constexpr int PLAN_GROUP = 1024;
constexpr int TS_WORDS = 3328;             // template store (32-bit words)
constexpr int NREC = 6, REC_MAX = 40;      // lanes recording a template at the same time; wildcards per template
constexpr int JQ_CAP = 64;
constexpr int W_STOPS = 96, W_STRUCT = 64;  // stop bytes / structural stops of a line the warp-per-line replay handles
struct FWarp { uint16_t spos[W_STOPS]; uint16_t sstop[W_STRUCT + 2]; uint32_t sdirty[(W_STRUCT + 8) / 4]; };   // sdirty: one byte per segment
struct FRes { uint16_t cpos, clen, toff, misc; };   // template captures of a line (misc: d2 | finish << 2 | done 32 | pending 64 | written 128)
struct FJob { uint32_t s, e, dst, pad; uint32_t *patch; };
struct FRecEv { uint16_t start, len; uint8_t kind, op; };
struct FRec { uint16_t n, nonsimple, n_str, n_arr; FRecEv ev[REC_MAX]; };           // segments packed into tiles by one warp of the plan kernel

// ---------------------------------------------------------------- tables (global -> shared at kernel start)
constexpr int HASH_BITS = 7;
struct FName { uint32_t w[5]; uint32_t len; };           // struct-tag name, zero padded
struct FFin { uint32_t w[4]; uint8_t len, val, pad[2]; };
constexpr int N_FIN = SSE_FIN_FUNCTION_CALL;             // finish_reason values with a code of their own: codes 1..N_FIN
struct FTables {
    uint16_t clssym[256];
    uint8_t tr[(NST * NCLS + 3) & ~3];
    uint32_t hash_mul;
    uint8_t hash[1 << HASH_BITS];                         // perfect hash of (first 4 bytes | 0x20202020, length) -> name id
    FName name[NNAMES];
    uint16_t field[N_NODES * NNAMES];                     // (struct, name id) -> ty | sub << 4 | tgt << 9 | FIELD_VALID
    FFin fin[N_FIN];                                      // fin[v - 1]: the finish_reason value whose code is v
};
static_assert(sizeof(FTables) % 4 == 0, "tables are copied as 32-bit words");

struct FSeg {                      // one segment of the tile (shared memory)
    uint32_t conn, mode, state;
    uint32_t data_off, in_pos, end;        // tile positions: first valid byte (carry), first input byte, one past the last byte
    uint32_t in_delta;                     // input arena offset = tile position + in_delta (positions >= in_pos)
    uint32_t term, dead;                   // this round: smallest terminating line / first dead line (SSE_NONE: none)
    uint32_t nruns, last_run;
    uint32_t rf0, fcnt, rr0, rcnt;         // this round's run
    uint32_t old_carry;
};
constexpr uint32_t FS_SKIP = 1, FS_TERM = 2, FS_DEAD = 4, FS_SKIP_DEAD = 8;

struct FLine {
    uint16_t start, nl, a, b;              // line [start, nl]; trimmed / payload bounds (see classify)
    uint16_t flags; uint8_t seg, pad;
    uint16_t rank_r, pad2;
    uint32_t out_off;                      // materialised bytes of this line in the out arena
};
constexpr uint16_t LF_KIND = 3, LF_PARSE = 4, LF_ZC = 8, LF_PREF = 16, LF_DONE = 32, LF_MAT = 64, LF_RMODE = 128, LF_JOB = 256;

struct FSmem {
    alignas(128) uint8_t tile[TILE + TILE_PAD];
    uint32_t stopbm[BM_WORDS + 4];
    uint32_t nlbm[BM_WORDS + 4];           // 1 bit per byte: '\n'
    FLine line[LCAP];
    uint16_t job[LCAP];
    uint16_t matlist[LCAP];                // lines of the round whose bytes have to be materialised
    FSeg seg[MAX_TSEGS];
    FTables T;
    uint32_t tstore[TS_WORDS];             // skeleton templates of this CTA (kept for the whole launch)
    uint32_t thead[W_STRUCT + 8];          // bucket (number of structural stops) -> newest template
    FRec rec[NREC];
    uint32_t ts_used, rec_busy, build_lock;
    FJob jq[JQ_CAP];                       // strings of this round that need unquoting
    FRes res[LCAP];                        // per decode job: what a template captured
    FWarp wsc[F_WARPS];                    // warp scratch of the replay
    uint32_t jq_n;
    alignas(8) unsigned long long mbar;
    uint32_t scan_a[F_WARPS], scan_b[F_WARPS];
    uint32_t bc[16];
};
static_assert(F_CTAS_PER_SM == 2 && sizeof(FSmem) <= 113 * 1024, "two CTAs per SM");

// ---------------------------------------------------------------- bulk copy + mbarrier (PTX)
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, unsigned long long *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_prefetch_l2(const void *src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------- out-of-line copies of shared helpers
// The steady-state path of this kernel has to fit the SM's 32 KB instruction cache (L1.5): everything that is big or rare
// is kept out of line, once.
__device__ __noinline__ void copy_s2g(uint8_t *__restrict__ g_dst, const uint8_t *__restrict__ sm_src, int n) { copy_s2g_vec(g_dst, sm_src, n); }
__device__ __noinline__ uint32_t trim_space_ab(const uint8_t *s, uint32_t a, uint32_t b) {     // strings.TrimSpace: a | b << 16
    int ia = (int)a, ib = (int)b;
    trim_space(s, ia, ib);
    return (uint32_t)ia | ((uint32_t)ib << 16);
}

// ---------------------------------------------------------------- block helpers
// exclusive prefix sums over the block (thread order); the totals come back too. Two barriers each.
__device__ __forceinline__ uint32_t warp_incl(uint32_t v, uint32_t lane) {
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t x = __shfl_up_sync(FULL, v, d); if ((int)lane >= d) v += x; }
    return v;
}
__device__ __noinline__ uint32_t block_scan1(FSmem &S, uint32_t a, uint32_t &ta) {
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    const uint32_t ia = warp_incl(a, lane);
    if (lane == 31) S.scan_a[w] = ia;
    __syncthreads();
    const uint32_t wa = warp_incl(lane < F_WARPS ? S.scan_a[lane] : 0u, lane);
    ta = __shfl_sync(FULL, wa, F_WARPS - 1);
    const uint32_t ba = __shfl_sync(FULL, wa, (int)(w ? w - 1u : 0u));
    __syncthreads();
    return (w ? ba : 0u) + ia - a;
}
__device__ __noinline__ void block_scan2(FSmem &S, uint32_t &a, uint32_t &b, uint32_t &ta, uint32_t &tb) {
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    const uint32_t ia = warp_incl(a, lane), ib = warp_incl(b, lane);
    if (lane == 31) { S.scan_a[w] = ia; S.scan_b[w] = ib; }
    __syncthreads();
    const uint32_t wa = warp_incl(lane < F_WARPS ? S.scan_a[lane] : 0u, lane), wb = warp_incl(lane < F_WARPS ? S.scan_b[lane] : 0u, lane);
    ta = __shfl_sync(FULL, wa, F_WARPS - 1); tb = __shfl_sync(FULL, wb, F_WARPS - 1);
    const uint32_t ba = __shfl_sync(FULL, wa, (int)(w ? w - 1u : 0u)), bb = __shfl_sync(FULL, wb, (int)(w ? w - 1u : 0u));
    __syncthreads();
    a = (w ? ba : 0u) + ia - a; b = (w ? bb : 0u) + ib - b;
}

// ---------------------------------------------------------------- stage 1a: stop bitmap
// 0x80 in every byte of w that is '"', '\\', '[', < 0x20 or >= 0x80 (exact)
__device__ __forceinline__ uint32_t stop_bits4(uint32_t w) {
    const uint32_t K80 = 0x80808080u, K01 = 0x01010101u;
    const uint32_t z1 = ((w ^ 0x22222222u) | K80) - K01;   // bit 7 clear iff the low 7 bits equal '"'
    const uint32_t z2 = ((w ^ 0x5C5C5C5Cu) | K80) - K01;
    const uint32_t z5 = ((w ^ 0x5B5B5B5Bu) | K80) - K01;
    const uint32_t z3 = (w & 0x7F7F7F7Fu) + 0x60606060u;   // bit 7 clear iff the low 7 bits are < 0x20
    return (~(z1 & z2 & z3 & z5) | w) & K80;
}
__device__ __forceinline__ uint32_t stop_mask16(const uint4 &v) {
    const uint32_t s0 = stop_bits4(v.x), s1 = stop_bits4(v.y), s2 = stop_bits4(v.z), s3 = stop_bits4(v.w);
    const uint32_t lo = __dp4a(s0, 0x08040201u, __dp4a(s1, 0x80402010u, 0u));   // 128 * (mask of 8 bytes)
    const uint32_t hi = __dp4a(s2, 0x08040201u, __dp4a(s3, 0x80402010u, 0u));
    return (lo | (hi << 8)) >> 7;
}
// 0x80 in every byte of w that is '\n' (exact)
__device__ __forceinline__ uint32_t nl_bits4(uint32_t w) {
    const uint32_t z = ((w ^ 0x0A0A0A0Au) | 0x80808080u) - 0x01010101u;
    return ~(z | w) & 0x80808080u;
}
__device__ __forceinline__ uint32_t nl_mask16(const uint4 &v) {
    const uint32_t lo = __dp4a(nl_bits4(v.x), 0x08040201u, __dp4a(nl_bits4(v.y), 0x80402010u, 0u));
    const uint32_t hi = __dp4a(nl_bits4(v.z), 0x08040201u, __dp4a(nl_bits4(v.w), 0x80402010u, 0u));
    return (lo | (hi << 8)) >> 7;
}
__device__ __forceinline__ void stage1a(FSmem &S, uint32_t fill) {
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    const uint32_t nsl = (fill + 511u) >> 9;
    uint16_t *bm16 = reinterpret_cast<uint16_t *>(S.stopbm);
    uint16_t *nl16 = reinterpret_cast<uint16_t *>(S.nlbm);
    for (uint32_t s = w; s < nsl; s += F_WARPS) {
        const uint32_t off = (s << 9) + lane * 16u;
        const uint4 v = *reinterpret_cast<const uint4 *>(S.tile + off);
        bm16[off >> 4] = (uint16_t)stop_mask16(v);
        nl16[off >> 4] = (uint16_t)nl_mask16(v);
    }
}

// first stop position >= p, or pe
__device__ __forceinline__ uint32_t next_stop(const FSmem &S, uint32_t p, uint32_t pe) {
    uint32_t w = p >> 5;
    uint32_t bits = S.stopbm[w] & (0xFFFFFFFFu << (p & 31u));
    #pragma unroll 1
    while (bits == 0) {
        w++;
        if ((w << 5) >= pe) return pe;
        bits = S.stopbm[w];
    }
    const uint32_t q = (w << 5) + (uint32_t)__ffs(bits) - 1u;
    return q < pe ? q : pe;
}
// strings.Contains(s[a:b], "[DONE]") through the stop bitmap
__device__ __noinline__ bool has_done_scan(const FSmem &S, uint32_t a, uint32_t b) {
    uint32_t p = a;
    while (p + 6u <= b) {
        const uint32_t q = next_stop(S, p, b);
        if (q + 6u > b) return false;
        if (is_done_at(S.tile + q)) return true;
        p = q + 1u;
    }
    return false;
}

// number of stop bytes in [a, b): two lines with the same count almost always have the same JSON shape
__device__ __forceinline__ uint32_t count_stops(const FSmem &S, uint32_t a, uint32_t b) {
    if (b <= a) return 0;
    uint32_t w = a >> 5;
    const uint32_t we = (b - 1u) >> 5;
    uint32_t bits = S.stopbm[w] & (0xFFFFFFFFu << (a & 31u));
    uint32_t n = 0;
    #pragma unroll 1
    for (; w < we; w++) { n += __popc(bits); bits = S.stopbm[w + 1]; }
    const uint32_t r = b & 31u;
    if (r) bits &= (1u << r) - 1u;
    return n + __popc(bits);
}

// Warp-cooperative unquote of a validated string body (decode.go unquoteBytes): 32 bytes per step. Plain bytes and the
// two-byte escapes (\" \\ \/ \b \f \n \r \t) are placed in parallel -- an escaping backslash is one that is preceded by an
// even number of backslashes; \uXXXX and non-ASCII bytes (kept, or U+FFFD when invalid) are done by lane 0 one at a time.
__device__ __noinline__ void warp_unquote2(const uint8_t *__restrict__ src, uint32_t s, uint32_t e, uint8_t *__restrict__ dst, uint32_t *patch) {
    const uint32_t lane = lane_id();
    const uint32_t lt = (1u << lane) - 1u;
    uint32_t i = s, n = 0;
    while (i < e) {
        const uint32_t idx = i + lane;
        const bool valid = idx < e;
        const uint32_t c = valid ? (uint32_t)src[idx] : 0x20u;
        const uint32_t nvalid = min(32u, e - i);
        const unsigned bs = __ballot_sync(FULL, valid && c == '\\');
        const unsigned hi = __ballot_sync(FULL, valid && c >= 0x80u);
        const uint32_t below = lane ? (bs << (32u - lane)) : 0u;
        const uint32_t run = (uint32_t)__clz((int)~below);                // consecutive backslashes right before this byte
        const bool escaped = (run & 1u) != 0;                         // the character an escaping backslash introduces
        const bool escaping = ((bs >> lane) & 1u) && !escaped;
        const unsigned um = __ballot_sync(FULL, valid && escaped && c == 'u');
        const unsigned em = __ballot_sync(FULL, escaping);
        uint32_t limit = nvalid;
        if (hi) limit = min(limit, (uint32_t)__ffs(hi) - 1u);
        if (um) limit = min(limit, (uint32_t)__ffs(um) - 2u);         // stop at the backslash of \uXXXX
        if (limit && ((em >> (limit - 1u)) & 1u)) limit--;            // an escape cut by the window: leave its backslash for the next step
        if (limit) {
            uint32_t m = c;
            if (escaped) m = c == 'b' ? 8u : c == 'f' ? 12u : c == 'n' ? 10u : c == 'r' ? 13u : c == 't' ? 9u : c;
            const bool outp = lane < limit && !escaping;
            const unsigned om = __ballot_sync(FULL, outp);
            if (outp) dst[n + __popc(om & lt)] = (uint8_t)m;
            n += __popc(om); i += limit;
            continue;
        }
        uint32_t ni = i, nn = n;                                      // one \uXXXX (pair) or one non-ASCII sequence
        if (lane == 0) {
            const uint32_t c0 = src[i];
            if (c0 == '\\') {
                ni = i + 2;
                uint32_t r = (uint32_t)hex4(src + ni);
                ni += 4;
                if (r >= 0xD800 && r < 0xE000) {
                    int r1 = -1;
                    if (ni + 6 <= e && src[ni] == '\\' && src[ni + 1] == 'u') r1 = hex4(src + ni + 2);
                    if (r < 0xDC00 && r1 >= 0xDC00 && r1 < 0xE000) { r = 0x10000 + ((r - 0xD800) << 10) + ((uint32_t)r1 - 0xDC00); ni += 6; }
                    else r = 0xFFFD;
                }
                nn += put_rune(dst, nn, r);
            } else {
                const int k = utf8_valid_len(src + i, (int)(e - i));
                if (k == 0) { nn += put_rune(dst, nn, 0xFFFD); ni = i + 1; }
                else { for (int q = 0; q < k; q++) dst[nn + q] = src[i + q]; nn += k; ni = i + k; }
            }
        }
        i = __shfl_sync(FULL, ni, 0); n = __shfl_sync(FULL, nn, 0);
    }
    if (lane == 0) *patch = n;
    __syncwarp();
}

// ---------------------------------------------------------------- stage 2: the decoder
// One lane per line. The lane state lives in registers: everything that touches it is inlined, the helpers that stay
// out of line take scalars. The walk is the byte automaton of sse_tables.h with shortcuts that are, by construction,
// sequences of its own steps: a string body is crossed by jumping from stop bit to stop bit; the quote that closes a
// clean string is dispatched without table lookups; the ':' after a key and the ',' after a value in an object are
// consumed in the same step; digit runs go four bytes at a time; "null" is taken as one token.
constexpr uint32_t SF_ESC = 1, SF_HI = 2, SF_BAD = 8, SF_STRMASK = 15;
constexpr uint32_t SF_SYN = 0x100, SF_TYPE = 0x200, SF_DEPTH = 0x400, SF_GBAD = 0x800, SF_USAGE = 0x1000,
                   SF_TCNONNIL = 0x2000, SF_TCOPEN = 0x4000, SF_TCVALID = 0x8000, SF_CDEC = 0x10000, SF_RMODE = 0x20000,
                   SF_CBAD = 0x40000, SF_CSET = 0x80000, SF_DONELINE = 0x100000;
constexpr uint32_t TCB_NAME = 0x100, TCB_ARGS = 0x200;   // decoded name / arguments are non-empty

struct FLane {
    uint32_t p, pe;
    uint32_t st, depth, skip, sd, cur, slen, sf, choices_count, n_choices, finish;
    unsigned long long ct, ct1, sstk;
    uint32_t content_pos, content_len, tc_count, tc_first, tc_prev, tc_cur, tcb, usage_idx;
    uint32_t rec, delta, plen, line;
    uint32_t rslot;                              // recording a template into S.rec[rslot] (SSE_NONE: no)
    bool busy;
};

enum : uint8_t { WK_END = 0, WK_STR = 1, WK_INT = 2 };      // template wildcards (see "skeleton templates" below)
enum : uint8_t { OP_NONE = 0, OP_CONTENT, OP_FINISH, OP_TC_ID, OP_TC_TYPE, OP_TC_NAME, OP_TC_ARGS, OP_TC_INDEX,
                 OP_U_PROMPT, OP_U_COMPLETION, OP_U_TOTAL, OP_CHK_I64, OP_CHK_F32 };
__device__ __forceinline__ void rec_event(FSmem &S, FLane &L, uint32_t kind, uint32_t start, uint32_t len, uint32_t op) {
    FRec &R = S.rec[L.rslot];
    if (R.n < REC_MAX) { FRecEv e; e.start = (uint16_t)start; e.len = (uint16_t)len; e.kind = (uint8_t)kind; e.op = (uint8_t)op; R.ev[R.n] = e; R.n++; }
    else R.nonsimple = 1;
}
__device__ __forceinline__ void rec_nonsimple(FSmem &S, FLane &L) { if (L.rslot != SSE_NONE) S.rec[L.rslot].nonsimple = 1; }

__device__ __forceinline__ bool fl_live(const FLane &L) { return L.sd >= 3 && ((L.sstk >> 10) & 31ull) == N_CHOICE && L.choices_count == 1; }
__device__ __forceinline__ uint32_t fl_top(const FLane &L) { return (uint32_t)((L.sstk >> (5 * (L.sd - 1))) & 31ull); }
__device__ __forceinline__ void fl_value_done(FLane &L) {
    if (L.depth == 0) { L.st = S_END; return; }
    const uint32_t d = L.depth - 1;
    const unsigned long long bits = d < 64 ? L.ct : L.ct1;
    L.st = ((bits >> (d & 63u)) & 1ull) ? (uint32_t)S_AFTA : (uint32_t)S_AFTO;
}

__device__ __noinline__ uint32_t f_text_alloc(const KParams &P, uint32_t bound) {
    const uint32_t o = atomicAdd(&P.ctr->text_bytes, bound);
    if (o + bound > P.cap_text) { sse_overflow(P.ctr, SSE_OVF_TEXT); return SSE_NONE; }
    return o;
}
// Captured string [s, s+len) of the tile. dec: bit 0 has escapes, bit 1 may hold invalid UTF-8 (-> U+FFFD, 1 byte -> 3).
// Without dec the span is the payload's own bytes in an arena. Otherwise a text-arena allocation; the unquote is
// deferred to the warp when the lane's job slot is free (patch receives the decoded length).
__device__ __forceinline__ Span f_capture(const KParams &P, FSmem &S, FLane &L, uint32_t s, uint32_t len, uint32_t dec, uint32_t *patch) {
    Span r;
    if (!dec) { r.off = s + L.delta; r.len = len; r.text = false; return r; }
    r.text = true; r.len = 0; r.off = 0;
    if (len == 0) return r;
    const uint32_t o = f_text_alloc(P, (((dec & 2u) ? 3u * len : len) + 3u) & ~3u);
    if (o == SSE_NONE) return r;
    r.off = o;
    if (patch) {              // decoded after the lines are through, one warp per string (process_window)
        const uint32_t qi = atomicAdd(&S.jq_n, 1u);
        if (qi < (uint32_t)JQ_CAP) {
            FJob jb; jb.s = s; jb.e = s + len; jb.dst = o; jb.patch = patch;
            S.jq[qi] = jb;
            r.len = len;      // patched by the job; raw > 0 implies decoded > 0
            return r;
        }
    }
    r.len = json_unquote_write(S.tile, (int)s, (int)(s + len), P.text + o);
    return r;
}

__device__ __forceinline__ void f_flush_tc(const KParams &P, FLane &L) {
    if ((L.tcb & SSE_TC_HAS_ID) || ((L.tcb & SSE_TC_HAS_FUNC) && (L.tcb & (TCB_NAME | TCB_ARGS)))) L.sf |= SF_TCVALID;
    L.sf &= ~SF_TCOPEN;
    if (L.tc_cur != SSE_NONE) P.tcs[L.tc_cur].flags = L.tcb & 0xFFu;
}

__device__ __noinline__ uint32_t f_tc_alloc(const KParams &P, uint32_t prev) {
    const uint32_t idx = atomicAdd(&P.ctr->n_tcs, 1u);
    if (idx >= P.cap_tcs) { sse_overflow(P.ctr, SSE_OVF_TCS); return SSE_NONE; }
    uint4 *q = reinterpret_cast<uint4 *>(&P.tcs[idx]);     // index 0, flags 0, next NONE, empty spans
    q[0] = make_uint4(0u, 0u, 0u, SSE_NONE); q[1] = make_uint4(0u, 0u, 0u, 0u); q[2] = make_uint4(0u, 0u, 0u, 0u);
    if (prev != SSE_NONE) P.tcs[prev].next = idx;
    return idx;
}
__device__ __noinline__ uint32_t f_usage_alloc(const KParams &P) {
    const uint32_t idx = atomicAdd(&P.ctr->n_usages, 1u);
    if (idx >= P.cap_usages) { sse_overflow(P.ctr, SSE_OVF_USAGES); return SSE_NONE; }
    sse_usage z; z.prompt_tokens = z.completion_tokens = z.total_tokens = 0;
    P.usages[idx] = z;
    return idx;
}

__device__ __forceinline__ void f_elem_begin(const KParams &P, FLane &L) {
    if (L.skip > 0) { L.cur = TY_SKIP; return; }
    const uint32_t nd = fl_top(L);
    if (nd == A_CHOICES) { L.choices_count++; L.cur = TY_STRUCT | (N_CHOICE << 4); }
    else if (nd == A_TOOLCALLS) {
        L.cur = TY_STRUCT | (N_TC << 4);
        if (fl_live(L)) {
            if (L.sf & SF_TCOPEN) f_flush_tc(P, L);
            L.sf |= SF_TCOPEN; L.tc_count++; L.tcb = 0;
            // a line that can no longer be JSON_OK never has its chain read: once the number in [1,1,...] has set SF_TYPE, the
            // elements after it take no sse_tc, so every element allocated but the first of a line takes 3 payload bytes ("{},")
            const uint32_t idx = (L.sf & (SF_SYN | SF_TYPE)) ? SSE_NONE : f_tc_alloc(P, L.tc_first == SSE_NONE ? SSE_NONE : L.tc_prev);
            if (idx != SSE_NONE) { if (L.tc_first == SSE_NONE) L.tc_first = idx; L.tc_prev = idx; }
            L.tc_cur = idx;
        }
    }
    else if (nd == A_TOKLP) L.cur = TY_STRUCT | (N_TOKLP << 4);
    else if (nd == A_TOPLP) L.cur = TY_STRUCT | (N_TOPLP << 4);
    else L.cur = TY_INT;
}

__device__ __forceinline__ void f_drop_tcs(FLane &L) {
    L.sf &= ~(SF_TCNONNIL | SF_TCOPEN | SF_TCVALID);
    L.tc_count = 0; L.tc_first = L.tc_prev = L.tc_cur = SSE_NONE; L.tcb = 0;
}
// a span is overwritten (repeated key, null): a queued unquote job must not patch its length later
__device__ __noinline__ void f_cancel_job(FSmem &S, uint32_t *patch) {
    const uint32_t n = min(S.jq_n, (uint32_t)JQ_CAP);
    for (uint32_t i = 0; i < n; i++) if (S.jq[i].patch == patch) S.jq[i].patch = nullptr;
}

// choices[0] starts anew: "choices":null, and the close of an empty "choices" array (decode.go array() sets a fresh slice of
// capacity 0, so a later "choices" array grows new, zeroed storage)
__device__ __forceinline__ void f_choices_reset(FLane &L) {
    L.n_choices = 0; L.choices_count = 0; L.finish = SSE_FIN_NONE; L.content_pos = L.content_len = 0;
    L.sf &= ~(SF_CDEC | SF_CBAD | SF_CSET);
    f_drop_tcs(L);
}

__device__ __forceinline__ void f_null(const KParams &P, FSmem &S, FLane &L) {
    const uint32_t ty = L.cur & 15u, tgt = (L.cur >> 9) & 15u;
    if (ty == TY_TS) { L.sf &= ~SF_GBAD; return; }
    if (tgt == TG_NONE || tgt == TG_FINISH || tgt == TG_CONTENT || tgt == TG_PROMPT || tgt == TG_COMPLETION || tgt == TG_TOTAL ||
        tgt == TG_TC_INDEX || tgt == TG_NAME || tgt == TG_ARGS) return;      // null leaves non-pointer fields untouched
    const bool tco = (L.sf & SF_TCOPEN) && fl_live(L) && L.tc_cur != SSE_NONE;
    if (tgt != TG_USAGE || (L.sf & SF_USAGE)) rec_nonsimple(S, L);     // a reset is not something a template replays
    switch (tgt) {
    case TG_CHOICES: f_choices_reset(L); break;
    case TG_USAGE: L.sf &= ~SF_USAGE; break;     // the line keeps its sse_usage slot: a later "usage":{} zeroes and reuses it
    case TG_TOOLCALLS: if (fl_live(L)) f_drop_tcs(L); break;
    case TG_TC_ID:
        if ((L.sf & SF_TCOPEN) && fl_live(L)) { L.tcb &= ~(SSE_TC_HAS_ID | SSE_TC_ID_TEXT); if (tco) { sse_tc *t = &P.tcs[L.tc_cur]; f_cancel_job(S, &t->id_len); t->id_off = t->id_len = 0; } }
        break;
    case TG_TC_TYPE:
        if ((L.sf & SF_TCOPEN) && fl_live(L)) { L.tcb &= ~(SSE_TC_HAS_TYPE | SSE_TC_TYPE_TEXT); if (tco) { sse_tc *t = &P.tcs[L.tc_cur]; f_cancel_job(S, &t->type_len); t->type_off = t->type_len = 0; } }
        break;
    case TG_TC_FUNCTION:
        if ((L.sf & SF_TCOPEN) && fl_live(L)) {
            L.tcb &= ~(SSE_TC_HAS_FUNC | SSE_TC_NAME_TEXT | SSE_TC_ARGS_TEXT | TCB_NAME | TCB_ARGS);
            if (tco) { sse_tc *t = &P.tcs[L.tc_cur]; f_cancel_job(S, &t->name_len); f_cancel_job(S, &t->args_len); t->name_off = t->name_len = t->args_off = t->args_len = 0; }
        }
        break;
    default: break;
    }
}

// the part of a number's end that needs the digits: range checks and captured integers. Returns SF_TYPE or 0.
__device__ __noinline__ uint32_t f_number_value(const KParams &P, const uint8_t *tile, uint32_t ty, uint32_t tgt, uint32_t start, uint32_t end,
                                                uint32_t usage_idx, uint32_t tc_idx) {
    if (ty == TY_F32) return f32_overflows(tile, (int)start, (int)end) ? SF_TYPE : 0u;
    int64_t v;
    if (!parse_i64(tile, (int)start, (int)end, v)) return SF_TYPE;
    if (tgt == TG_PROMPT || tgt == TG_COMPLETION || tgt == TG_TOTAL) {
        if (usage_idx != SSE_NONE) {
            sse_usage *u = &P.usages[usage_idx];
            if (tgt == TG_PROMPT) u->prompt_tokens = v; else if (tgt == TG_COMPLETION) u->completion_tokens = v; else u->total_tokens = v;
        }
    } else if (tgt == TG_TC_INDEX) { if (tc_idx != SSE_NONE) P.tcs[tc_idx].index = v; }
    return 0u;
}
// key / finish_reason bytes [s, s+len) as little-endian words, zero padded (len <= 20)
__device__ __forceinline__ void load_words(const FSmem &S, uint32_t s, uint32_t len, uint32_t k[5]) {
    const uint32_t *w = reinterpret_cast<const uint32_t *>(S.tile + (s & ~3u));
    const uint32_t sh = (s & 3u) * 8u;
    const uint32_t a0 = w[0], a1 = w[1], a2 = w[2], a3 = w[3], a4 = w[4], a5 = w[5];
    k[0] = __funnelshift_r(a0, a1, sh); k[1] = __funnelshift_r(a1, a2, sh); k[2] = __funnelshift_r(a2, a3, sh);
    k[3] = __funnelshift_r(a3, a4, sh); k[4] = __funnelshift_r(a4, a5, sh);
    #pragma unroll
    for (int i = 0; i < 5; i++) {
        const int rem = (int)len - 4 * i;          // bytes of word i that belong to the string
        if (rem <= 0) k[i] = 0; else if (rem < 4) k[i] &= (1u << (rem * 8)) - 1u;
    }
}

// (struct, key) -> packed field (ty | sub << 4 | tgt << 9), TY_SKIP if the struct has no such field.
// Exact match first, then encoding/json's case-insensitive match (decode.go: byExactName, then byFoldedName). The struct-tag
// name is found through a perfect hash of (first four bytes with the case bit set, length); the candidate is then compared
// word by word. A key that differs from the candidate in case bits only goes through the exact folding rules (key_eq).
__device__ __forceinline__ uint32_t f_match_key(const FSmem &S, uint32_t node, uint32_t s, uint32_t len) {
    if (len < 2u || len > 18u) return TY_SKIP;
    const uint32_t *w = reinterpret_cast<const uint32_t *>(S.tile + (s & ~3u));
    const uint32_t sh = (s & 3u) * 8u;
    uint32_t a = w[0], b = w[1];
    uint32_t k = __funnelshift_r(a, b, sh);
    if (len < 4u) k &= (1u << (len * 8u)) - 1u;
    const uint32_t h = ((k | 0x20202020u) * S.T.hash_mul + len * 0x9E3779B1u) >> (32 - HASH_BITS);
    const uint32_t nid = S.T.hash[h];
    if (nid == 0xFFu) return TY_SKIP;
    const FName &N = S.T.name[nid];
    if (N.len != len) return TY_SKIP;
    uint32_t diff = k ^ N.w[0];
    #pragma unroll
    for (int i = 1; i < 5; i++) {
        if ((int)len > 4 * i) {
            a = b; b = w[i + 1];
            uint32_t ki = __funnelshift_r(a, b, sh);
            const int rem = (int)len - 4 * i;
            if (rem < 4) ki &= (1u << (rem * 8)) - 1u;
            diff |= ki ^ N.w[i];
        }
    }
    if (diff == 0) { const uint32_t f = S.T.field[node * NNAMES + nid]; return (f & FIELD_VALID) ? (f & 0x1FFFu) : (uint32_t)TY_SKIP; }
    if ((diff & ~0x20202020u) == 0) {     // differs in case bits only: let the exact folding rules decide
        const int f = match_field(c_schema, (int)node, S.tile + s, (int)len);
        if (f >= 0) return c_schema.f[f].ty | ((uint32_t)c_schema.f[f].sub << 4) | ((uint32_t)c_schema.f[f].tgt << 9);
    }
    return TY_SKIP;
}
__device__ __noinline__ uint32_t f_match_key_slow(const FSmem &S, uint32_t node, uint32_t s, uint32_t e) {
    uint8_t tmp[72];     // escaped / non-ASCII key: unquote and fold like encoding/json does
    const uint32_t n = json_unquote(S.tile, (int)s, (int)e, tmp, 64);
    const int f = (n <= 64) ? match_field(c_schema, (int)node, tmp, (int)n) : -1;
    return f >= 0 ? (c_schema.f[f].ty | ((uint32_t)c_schema.f[f].sub << 4) | ((uint32_t)c_schema.f[f].tgt << 9)) : (uint32_t)TY_SKIP;
}
__device__ __noinline__ uint32_t f_match_finish(const FSmem &S, uint32_t s, uint32_t len, uint32_t dirty) {
    if (len == 0) return SSE_FIN_NONE;
    if (dirty) {
        uint8_t tmp[40];
        const uint32_t n = json_unquote(S.tile, (int)s, (int)(s + len), tmp, 32);
        return (n <= 32) ? classify_finish(tmp, (int)n) : (uint32_t)SSE_FIN_OTHER;
    }
    if (len < 4u || len > 14u) return SSE_FIN_OTHER;
    uint32_t k[5];
    load_words(S, s, len, k);
    #pragma unroll
    for (int i = 0; i < N_FIN; i++) {
        const FFin &F = S.T.fin[i];
        if (F.len == len && k[0] == F.w[0] && k[1] == F.w[1] && k[2] == F.w[2] && k[3] == F.w[3]) return F.val;
    }
    return SSE_FIN_OTHER;
}

// ---- the semantic actions (decode.go object / array / literalStore against the struct types)
__device__ __forceinline__ void f_open(const KParams &P, FSmem &S, FLane &L, bool arr) {
    if (L.rslot != SSE_NONE && arr) S.rec[L.rslot].n_arr++;
    if (L.depth >= 128) { L.sf |= SF_DEPTH | SF_SYN; L.p = L.pe - 1; L.st = S_END; return; }
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
            const bool live = fl_live(L);
            L.sstk = (L.sstk & ~(31ull << (5 * L.sd))) | ((unsigned long long)sub << (5 * L.sd));
            L.sd++;
            if (tgt != TG_NONE) {
                if (tgt == TG_USAGE) {
                    // a fresh CompletionUsage{}; a repeated key decodes into the same struct. One slot per line: after
                    // "usage":null the next object zeroes the line's slot instead of taking another (at most one usage per record)
                    if (L.usage_idx == SSE_NONE) L.usage_idx = f_usage_alloc(P);
                    else if (!(L.sf & SF_USAGE)) { sse_usage z; z.prompt_tokens = z.completion_tokens = z.total_tokens = 0; P.usages[L.usage_idx] = z; }
                    L.sf |= SF_USAGE;
                }
                else if (tgt == TG_TC_FUNCTION) { if (live && (L.sf & SF_TCOPEN)) L.tcb |= SSE_TC_HAS_FUNC; }
                else if (tgt == TG_CHOICES) { if (L.n_choices || L.choices_count) rec_nonsimple(S, L); L.choices_count = 0; }
                else if (tgt == TG_TOOLCALLS) { if (live) { if (L.sf & SF_TCNONNIL) rec_nonsimple(S, L); f_drop_tcs(L); L.sf |= SF_TCNONNIL; } }
            }
            if (sub == N_GOOGLE) L.sf &= ~SF_GBAD;
        }
    }
    L.st = arr ? S_ARR0 : S_OBJ0;
}
__device__ __forceinline__ void f_close(const KParams &P, FLane &L) {
    L.depth--;
    if (L.skip > 0) L.skip--;
    else {
        const uint32_t node = fl_top(L);
        L.sd--;
        if (node == A_CHOICES) { if (L.choices_count) L.n_choices = L.choices_count; else f_choices_reset(L); }
        else if (node == A_TOOLCALLS) { if (fl_live(L) && (L.sf & SF_TCOPEN)) f_flush_tc(P, L); }
        else if (node == N_GOOGLE) { if (L.sf & SF_GBAD) L.sf |= SF_TYPE; }
    }
    fl_value_done(L);
}
// a key [start, start+len) ended; dirty: it has escapes or non-ASCII bytes
__device__ __forceinline__ void f_key_end(FSmem &S, FLane &L, uint32_t start, uint32_t len, bool dirty) {
    uint32_t cur = TY_SKIP;
    if (L.skip == 0) {
        const uint32_t node = fl_top(L);
        cur = dirty ? f_match_key_slow(S, node, start, start + len) : f_match_key(S, node, start, len);
    }
    L.cur = cur;
    L.st = S_COLON;
    if (L.rslot != SSE_NONE) S.rec[L.rslot].n_str++;
}
// a string value [start, start+len) ended; d2: bit 0 escapes, bit 1 invalid UTF-8
__device__ __forceinline__ void f_vstr_end(const KParams &P, FSmem &S, FLane &L, uint32_t start, uint32_t len, uint32_t d2) {
    const uint32_t ty = L.cur & 15u, tgt = (L.cur >> 9) & 15u;
    uint32_t op = OP_NONE;
    if (ty == TY_STR || ty == TY_PSTR) {
        if (tgt != TG_NONE && fl_live(L)) {
            if (tgt == TG_CONTENT) {
                op = OP_CONTENT;
                L.content_pos = start; L.content_len = len;
                L.sf = (L.sf & ~(SF_CDEC | SF_CBAD)) | SF_CSET | ((d2 & 1u) ? SF_CDEC : 0u) | ((d2 & 2u) ? SF_CBAD : 0u);
            } else if (tgt == TG_FINISH) { L.finish = f_match_finish(S, start, len, d2); op = OP_FINISH; }
            else if (L.sf & SF_TCOPEN) {
                // the four strings of a tool-call element share one code path: field k of {id, type, name, arguments}
                const uint32_t k = tgt == TG_TC_ID ? 0u : tgt == TG_TC_TYPE ? 1u : tgt == TG_NAME ? 2u : tgt == TG_ARGS ? 3u : 4u;
                if (k < 4u) {
                    const uint32_t text_bit = SSE_TC_ID_TEXT << k;
                    L.tcb &= ~text_bit;
                    if (k == 0) L.tcb |= SSE_TC_HAS_ID; else if (k == 1) L.tcb |= SSE_TC_HAS_TYPE;
                    else if (k == 2) L.tcb = (L.tcb & ~TCB_NAME) | (len ? TCB_NAME : 0u);
                    else L.tcb = (L.tcb & ~TCB_ARGS) | (len ? TCB_ARGS : 0u);
                    if (L.tc_cur != SSE_NONE && L.tc_count <= 16u) op = (OP_TC_ID + k) | ((L.tc_count - 1u) << 4); else rec_nonsimple(S, L);
                    if (L.tc_cur != SSE_NONE) {
                        uint32_t *span = &P.tcs[L.tc_cur].id_off + 2u * k;     // {off, len} pairs are laid out in this order
                        f_cancel_job(S, span + 1);
                        const Span sp = f_capture(P, S, L, start, len, d2, span + 1);
                        span[0] = sp.off; span[1] = sp.len;
                        if (sp.text) L.tcb |= text_bit;
                    }
                }
            }
        }
    } else if (ty == TY_TS) L.sf &= ~SF_GBAD;
    else if (ty != TY_SKIP) L.sf |= SF_TYPE;
    fl_value_done(L);
    if (L.rslot != SSE_NONE) { S.rec[L.rslot].n_str++; rec_event(S, L, WK_STR, start, len, op); }
}
// a number [start, end) ended
__device__ __forceinline__ void f_number_end(const KParams &P, FSmem &S, FLane &L, uint32_t start, uint32_t end, bool is_int) {
    const uint32_t ty = L.cur & 15u, tgt = (L.cur >> 9) & 15u;
    if (L.rslot != SSE_NONE && is_int) {
        uint32_t op = OP_NONE;
        if (ty == TY_INT) {
            op = OP_CHK_I64;
            if ((L.sf & SF_USAGE) && L.usage_idx != SSE_NONE && (tgt == TG_PROMPT || tgt == TG_COMPLETION || tgt == TG_TOTAL)) op = OP_U_PROMPT + (tgt - TG_PROMPT);
            else if (tgt == TG_TC_INDEX && (L.sf & SF_TCOPEN) && fl_live(L) && L.tc_cur != SSE_NONE && L.tc_count <= 16u) op = OP_TC_INDEX | ((L.tc_count - 1u) << 4);
        } else if (ty == TY_F32) op = OP_CHK_F32;
        rec_event(S, L, WK_INT, start, end - start, op);
    }
    if (ty == TY_INT) {
        if (!is_int) L.sf |= SF_TYPE;
        else if (end - start > 18 || tgt != TG_NONE)
            L.sf |= f_number_value(P, S.tile, ty, tgt, start, end, L.usage_idx,
                                   ((L.sf & SF_TCOPEN) && fl_live(L)) ? L.tc_cur : SSE_NONE);
    } else if (ty == TY_F32) L.sf |= f_number_value(P, S.tile, ty, tgt, start, end, SSE_NONE, SSE_NONE);
    else if (ty == TY_TS) L.sf |= SF_GBAD;
    else if (ty != TY_SKIP) L.sf |= SF_TYPE;
}

// returns true when the current byte has to be looked up again in the new state
__device__ __forceinline__ bool f_action(const KParams &P, FSmem &S, FLane &L, uint32_t t) {
    switch (t) {
    case A_OPEN_OBJ: f_open(P, S, L, false); return false;
    case A_OPEN_ARR: f_open(P, S, L, true); return false;
    case A_CLOSE_OBJ: case A_CLOSE_ARR: f_close(P, L); return false;
    case A_KEY_END: f_key_end(S, L, L.p - L.slen, L.slen, (L.sf & (SF_ESC | SF_HI)) != 0); return false;
    case A_VSTR_END: f_vstr_end(P, S, L, L.p - L.slen, L.slen, ((L.sf & SF_ESC) ? 1u : 0u) | ((L.sf & SF_BAD) ? 2u : 0u)); return false;
    case A_BAD_STAY: L.sf |= SF_BAD; L.st = S_VSTR; return false;
    case A_BAD_REDO: L.sf |= SF_BAD; L.st = S_VSTR; return true;
    case A_NUM_END: f_number_end(P, S, L, L.p - L.slen - 1u, L.p, L.st == S_NZERO || L.st == S_NINT); fl_value_done(L); return true;
    case A_LIT_TRUE: case A_LIT_FALSE: {
        const uint32_t ty = L.cur & 15u;
        if (ty == TY_TS) L.sf |= SF_GBAD; else if (ty != TY_SKIP) L.sf |= SF_TYPE;
        fl_value_done(L);
        return false;
    }
    case A_LIT_NULL: f_null(P, S, L); fl_value_done(L); return false;
    case A_ELEM_REDO: f_elem_begin(P, L); L.st = S_VAL; return true;
    case A_COMMA_ARR: f_elem_begin(P, L); L.st = S_VAL; return false;
    default:   // A_ERR
        L.sf |= SF_SYN; L.p = L.pe - 1; L.st = S_END;
        return false;
    }
}

// four bytes at p (any alignment)
__device__ __forceinline__ uint32_t load4(const FSmem &S, uint32_t p) {
    const uint32_t *w = reinterpret_cast<const uint32_t *>(S.tile + (p & ~3u));
    return __funnelshift_r(w[0], w[1], (p & 3u) * 8u);
}
// 0x80 in every byte of w4 that is not '0'..'9'
__device__ __forceinline__ uint32_t nondigit4(uint32_t w4) {
    return (~((w4 | 0x80808080u) - 0x30303030u) | (w4 + 0x46464646u) | w4) & 0x80808080u;
}

// One byte of the table automaton (scanner.go grammar): used for everything the token shortcuts of f_step do not take --
// white space, escapes, non-ASCII bytes, '[' inside strings, fractions and exponents, true / false, errors.
__device__ __forceinline__ void f_byte(const KParams &P, FSmem &S, FLane &L, uint32_t c) {
    const uint32_t e = S.T.clssym[c];
    const uint32_t cls = e & 63u;
    const bool in_str = L.st >= S_KSTR, in_tok = L.st >= S_NMINUS;
    if (cls == C_LBRACK && (L.sf & SF_RMODE) && L.p + 6u <= L.pe && is_done_at(S.tile + L.p)) L.sf |= SF_DONELINE;   // agent.go:181
    uint32_t t = S.T.tr[L.st * NCLS + cls];
    if (t < A_FIRST) {
        L.sf = in_str ? (L.sf | ((e >> 13) & 3u)) : (L.sf & ~SF_STRMASK);
        L.slen = in_tok ? L.slen + 1 : 0;
        L.st = t;
        L.p++;
        return;
    }
    for (;;) {
        if (!f_action(P, S, L, t)) break;            // the action chose the next state
        t = S.T.tr[L.st * NCLS + cls];               // redo: same byte, new state
        if (t < A_FIRST) { L.st = t; break; }
    }
    const uint32_t nf = (cls == C_BSLASH ? SF_ESC : 0u) | (cls >= C_H80 ? SF_HI : 0u);
    L.sf = in_str ? (L.sf | nf) : (L.sf & ~SF_STRMASK);
    L.slen = in_tok ? L.slen + 1 : 0;
    L.p++;
}

// One step of a lane. At a token boundary the common tokens are taken whole -- each shortcut is exactly the sequence of
// f_byte steps it replaces, and applies only when the bytes are there for it; anything else falls through to f_byte:
//   key       '"' clean body '"' [':']           (S_OBJ0 / S_KEY -> S_COLON / S_VAL), and on into the value
//   string    '"' clean body '"' [',' in object] (S_VAL -> S_AFTO / S_AFTA / S_END -> S_KEY)
//   integer   [-] 0 | [1-9][0-9]*  followed by , } ]
//   null
//   ','  after a value in an object            (S_AFTO -> S_KEY)
// A clean body has no stop byte before its closing quote (no escape, control, non-ASCII byte or '[').
__device__ __forceinline__ void f_step(const KParams &P, FSmem &S, FLane &L) {
    if (L.p >= L.pe) return;
    uint32_t c = S.tile[L.p];
    const uint32_t st = L.st;
    if (st == S_VSTR || st == S_KSTR) {               // inside a string whose body is not clean
        // from stop byte to stop byte; well-formed escapes, valid UTF-8 sequences and '[' are crossed right here (each is the
        // sequence of plain f_byte steps it stands for), anything else is left to f_byte
        for (;;) {
            const uint32_t q = next_stop(S, L.p, L.pe);
            L.slen += q - L.p; L.p = q;
            if (q >= L.pe) return;                   // unterminated: the line ends inside the string (syntax error at finish)
            c = S.tile[q];
            uint32_t adv = 0;
            if (c == '\\') {
                const uint32_t c2 = S.tile[q + 1u];
                if (q + 2u <= L.pe && (c2 == '"' || c2 == '\\' || c2 == '/' || c2 == 'b' || c2 == 'f' || c2 == 'n' || c2 == 'r' || c2 == 't')) adv = 2;
                else if (c2 == 'u' && q + 6u <= L.pe && hex4(S.tile + q + 2u) >= 0) adv = 6;
                if (adv) L.sf |= SF_ESC;
            } else if (c == '[') {
                if ((L.sf & SF_RMODE) && q + 6u <= L.pe && is_done_at(S.tile + q)) L.sf |= SF_DONELINE;     // agent.go:181
                adv = 1;
            } else if (c >= 0x80u) {
                adv = st == S_KSTR ? 1u : (uint32_t)utf8_valid_len(S.tile + q, (int)(L.pe - q));    // keys are not validated by the automaton
                if (adv) L.sf |= SF_HI;
            }
            if (!adv) break;                         // closing quote, control byte, malformed escape or UTF-8
            L.p += adv; L.slen += adv;
            if (L.p >= L.pe) return;
        }
    } else if (st == S_KEY || st == S_OBJ0) {
        if (c == '"') {
            const uint32_t q = next_stop(S, L.p + 1u, L.pe);
            if (q < L.pe && S.tile[q] == '"') {
                f_key_end(S, L, L.p + 1u, q - L.p - 1u, false);
                L.p = q + 1u;
                if (L.p < L.pe && S.tile[L.p] == ':') { L.st = S_VAL; L.p++; }
                if (L.st != S_VAL || L.p >= L.pe) return;
                c = S.tile[L.p];
                goto value;
            }
        }
    } else if (st == S_VAL) {
value:
        if (c == '"') {
            const uint32_t q = next_stop(S, L.p + 1u, L.pe);
            if (q < L.pe && S.tile[q] == '"') {
                f_vstr_end(P, S, L, L.p + 1u, q - L.p - 1u, 0u);
                L.p = q + 1u;
                goto after_value;
            }
        } else if (c - '0' <= 9u || c == '-') {
            uint32_t i = L.p + (c == '-' ? 1u : 0u);
            const uint32_t d0 = S.tile[i];           // (the tile is padded: reading one byte past pe is harmless)
            bool ok = i < L.pe;
            if (d0 == '0') i++;
            else if (d0 - '1' <= 8u) {
                i++;
                while (i + 4u <= L.pe && nondigit4(load4(S, i)) == 0) i += 4u;
                while (i < L.pe && (uint32_t)S.tile[i] - '0' <= 9u) i++;
            } else ok = false;
            if (ok && i < L.pe) {
                const uint32_t d = S.tile[i];
                if (d == ',' || d == '}' || d == ']') {
                    f_number_end(P, S, L, L.p, i, true);
                    fl_value_done(L);
                    L.p = i;
                    goto after_value;
                }
            }
        } else if (c == 'n' && L.p + 4u <= L.pe && load4(S, L.p) == 0x6C6C756Eu) {
            f_null(P, S, L); fl_value_done(L);
            L.p += 4u;
            goto after_value;
        }
    } else if (st == S_AFTO) {
        if (c == ',') { L.st = S_KEY; L.p++; return; }
    }
    f_byte(P, S, L, c);
    return;
after_value:
    if (L.st == S_AFTO && L.p < L.pe && S.tile[L.p] == ',') { L.st = S_KEY; L.p++; }
}
// ---------------------------------------------------------------- skeleton templates
// Consecutive chunks of a stream -- and the chunks of every other stream of the same provider -- differ only inside string
// values and integers: keys, punctuation and literals are byte for byte the same. A line the automaton has parsed leaves a
// template in the CTA's cache: its structural stops (the quotes that open and close strings, and '[' outside strings), and
// for every segment between two of them either its bytes (keys, punctuation), "a string body", or "punctuation around an
// integer", plus what the parse did with the captured ones. A later line whose structural stops and segments compare equal,
// and whose string bodies / integers are well formed, takes the automaton through exactly the same transitions: its record
// is the template's with its own spans. The comparison is done by a whole warp per line -- one lane per stop, then one lane
// per segment, string parity and stop ranks by ballot -- so its cost does not depend on what the other lines look like.
// Lines that fit no template go to the automaton (one lane per line), which records a template for them.
constexpr uint32_t T_LIT_MAX = 1024;       // skeleton bytes per template
constexpr uint32_t TF_HAS_USAGE = 1;
constexpr uint32_t T_HDR = 7;              // header words
enum : uint32_t { SK_LIT = 0, SK_WILD = 1, SK_LITINT = 2, SK_LIT3 = 3 };   // SK_LIT3: up to 3 bytes, held in the segment word itself
// template in the store (32-bit words):
//   [0] next | n_struct << 16          [1] skeleton bytes | flags << 16 | tc_count << 24     [2] static record flags
//   [3] n_choices | n_ops << 16        [4],[5] bit j: structural stop j is '[' (else '"')
//   [6] content segment | finish_reason segment << 8 (0xFF: none)
//   n_struct + 1 segments: kind | len_a << 2 | len_b << 10 | byte offset into the literal pool << 18
//   n_ops ops: code | segment << 8 | tool-call ordinal << 16
//   4 words of per-element tool-call flags when tc_count > 0, then the literal pool

__device__ __forceinline__ uint32_t store_load4(const FSmem &S, const uint32_t *pool, uint32_t off) {
    const uint32_t *w = pool + (off >> 2);
    return __funnelshift_r(w[0], w[1], (off & 3u) * 8u);
}
// line bytes [a, a+len) == pool bytes [off, off+len)
__device__ __forceinline__ bool seg_equal(const FSmem &S, uint32_t a, const uint32_t *pool, uint32_t off, uint32_t len) {
    if (len <= 4u) return len == 0u || ((load4(S, a) ^ store_load4(S, pool, off)) & (0xFFFFFFFFu >> ((4u - len) * 8u))) == 0u;
    uint32_t diff = 0, j = 0;
    #pragma unroll 1
    for (; j + 4u <= len; j += 4u) diff |= load4(S, a + j) ^ store_load4(S, pool, off + j);
    if (j < len) diff |= (load4(S, a + j) ^ store_load4(S, pool, off + j)) & ((1u << ((len - j) * 8u)) - 1u);
    return diff == 0;
}
// integer [a, b): [-] 0 | [1-9][0-9]*
__device__ __forceinline__ bool int_ok(const FSmem &S, uint32_t a, uint32_t b) {
    if (a < b && S.tile[a] == '-') a++;
    if (a >= b) return false;
    const uint32_t d0 = S.tile[a];
    if (d0 == '0') return a + 1u == b;
    if (d0 - '1' > 8u) return false;
    a++;
    #pragma unroll 1
    while (a + 4u <= b) { if (nondigit4(load4(S, a))) return false; a += 4u; }
    if (a < b && (nondigit4(load4(S, a)) & (0xFFFFFFFFu >> ((4u - (b - a)) * 8u)))) return false;
    return true;
}
__device__ __noinline__ bool escape_ok(const FSmem &S, uint32_t p, uint32_t pe) {      // p: an escaping backslash
    const uint32_t c2 = S.tile[p + 1u];
    if (p + 2u <= pe && (c2 == '"' || c2 == '\\' || c2 == '/' || c2 == 'b' || c2 == 'f' || c2 == 'n' || c2 == 'r' || c2 == 't')) return true;
    return c2 == 'u' && p + 6u <= pe && hex4(S.tile + p + 2u) >= 0;
}
__device__ __noinline__ uint32_t backslash_run_before(const FSmem &S, uint32_t p, uint32_t lo) {
    uint32_t n = 0;
    while (p > lo && S.tile[p - 1u] == '\\') { n++; p--; }
    return n;
}

__device__ __noinline__ uint32_t f_tcs_alloc(const KParams &P, uint32_t n, const uint32_t *static_flags) {
    const uint32_t base = atomicAdd(&P.ctr->n_tcs, n);
    if (base + n > P.cap_tcs) { sse_overflow(P.ctr, SSE_OVF_TCS); return SSE_NONE; }
    const uint8_t *sf8 = reinterpret_cast<const uint8_t *>(static_flags);
    for (uint32_t j = 0; j < n; j++) {
        uint4 *q = reinterpret_cast<uint4 *>(&P.tcs[base + j]);
        q[0] = make_uint4(0u, 0u, (uint32_t)sf8[j], j + 1u < n ? base + j + 1u : SSE_NONE);
        q[1] = make_uint4(0u, 0u, 0u, 0u); q[2] = make_uint4(0u, 0u, 0u, 0u);
    }
    return base;
}

// The record of a retired line (agent.go:205-242 reads) from the lane's final state. Out of line: called from the template
// path and from the automaton.
__device__ __noinline__ void f_emit_record(const KParams &P, FSmem &S, uint32_t sf, uint32_t n_choices, uint32_t usage_idx, uint32_t content_pos,
                                           uint32_t content_len, uint32_t finish, uint32_t tc_count, uint32_t tc_first, uint32_t rec,
                                           uint32_t plen, uint32_t line, uint32_t delta) {
    sse_rec r;
    r.frame = SSE_NONE; r.flags = 0; r.content_off = r.content_len = 0; r.tc_first = SSE_NONE; r.tc_count = 0; r.n_choices = 0;
    r.usage = SSE_NONE;
    if (sf & SF_DEPTH) r.flags |= SSE_F_DEPTH_LIMIT;
    if (sf & SF_DONELINE) r.flags |= SSE_F_DONE_LINE;      // swallowed by the reframe, parsed for agent.go:377-402
    bool terminates = false;
    if (!(sf & (SF_SYN | SF_TYPE))) {
        r.flags |= SSE_F_JSON_OK;
        r.n_choices = (uint16_t)min(n_choices, 0xFFFFu);
        if ((sf & SF_USAGE) && usage_idx != SSE_NONE) { r.usage = usage_idx; r.flags |= SSE_F_HAS_USAGE; }
        if (n_choices > 0) {
            FLane C; C.delta = delta;
            const Span ct = f_capture(P, S, C, content_pos, content_len, ((sf & SF_CDEC) ? 1u : 0u) | ((sf & SF_CBAD) ? 2u : 0u),
                                      &P.recs[rec].content_len);
            r.content_off = ct.len ? ct.off : 0; r.content_len = ct.len;
            if (ct.text && ct.len) r.flags |= SSE_F_CONTENT_TEXT;
            r.flags |= finish << SSE_F_FINISH_SHIFT;
            if (sf & SF_TCNONNIL) r.flags |= SSE_F_TC_NONNIL;
            if (sf & SF_TCVALID) r.flags |= SSE_F_TC_VALID;
            r.tc_first = tc_count ? tc_first : SSE_NONE;
            r.tc_count = (uint16_t)min(tc_count, 0xFFFFu);
            if ((sf & SF_RMODE) && !(sf & SF_DONELINE) && (finish == SSE_FIN_STOP || finish == SSE_FIN_TOOL_CALLS)) {
                r.flags |= SSE_F_TERMINATES;
                terminates = true;
            }
        }
    }
    r.payload_len = plen;
    uint4 *q = reinterpret_cast<uint4 *>(&P.recs[rec]);
    q[0] = make_uint4(r.frame, r.flags, r.content_off, r.content_len);
    q[1] = make_uint4(r.tc_first, (uint32_t)r.tc_count | ((uint32_t)r.n_choices << 16), r.usage, r.payload_len);
    FLine &ln = S.line[line];
    if (sf & SF_DONELINE) ln.flags |= LF_DONE;
    if (terminates) atomicMin(&S.seg[ln.seg].term, line);
}

// does the string body [a, b) hold invalid UTF-8 (Go would write U+FFFD)? Escapes are skipped.
__device__ __noinline__ bool body_has_bad_utf8(const FSmem &S, uint32_t a, uint32_t b) {
    while (a < b) {
        const uint32_t c = S.tile[a];
        if (c == '\\') { a += 2u; continue; }
        if (c < 0x80u) { a++; continue; }
        const int k = utf8_valid_len(S.tile + a, (int)(b - a));
        if (k == 0) return true;
        a += (uint32_t)k;
    }
    return false;
}

// The automaton has just retired a line it recorded (slot rslot): turn the recording into a template.
__device__ __noinline__ void t_build(const KParams &P, FSmem &S, uint32_t rslot, uint32_t ps, uint32_t pe, uint32_t rec_static,
                                     uint32_t tflags, uint32_t n_choices, uint32_t tc_count, uint32_t tc_first) {
    const FRec &R = S.rec[rslot];
    if (tc_count > 15u || pe - ps < 2u) return;
    const uint32_t off = S.ts_used;                     // built in place behind the last template (the caller holds the build lock)
    if (off + 360u > (uint32_t)TS_WORDS) return;         // (a template is at most 7 + 65 + 24 + 4 + 257 words)
    uint32_t *T = S.tstore + off;
    uint32_t *segw = T + T_HDR;
    // ---- the structural stops of the line, and what stands between them
    uint32_t ns = 0, ev = 0, n_ops = 0, lit_used = 0, mask0 = 0, mask1 = 0, cseg = 0xFFu, fseg = 0xFFu;
    uint32_t opw[24];
    uint8_t lit[T_LIT_MAX];                             // (local scratch: building a template is rare)
    uint32_t seg_a = ps;                                // first byte of the segment that is open
    bool in_str = false, fail = false;
    uint32_t p = ps;
    for (;;) {
        const uint32_t q = p < pe ? next_stop(S, p, pe) : pe;
        const bool at_end = q >= pe;
        uint32_t c = at_end ? 0u : (uint32_t)S.tile[q];
        bool structural = at_end;
        if (!at_end) {
            if (in_str) { if (c == '"') structural = true; else if (c == '\\') { p = q + 2u; continue; } }
            else if (c == '"' || c == '[') structural = true;
            else { fail = true; break; }                // a stop byte outside strings that is not structural
            if (!structural) { p = q + 1u; continue; }
        }
        // segment [seg_a, q)
        const uint32_t a = seg_a, b = at_end ? pe : q, len = b - a;
        uint32_t word;
        if (ev < R.n && R.ev[ev].kind == WK_STR && R.ev[ev].start == a && (uint32_t)R.ev[ev].start + R.ev[ev].len == b && in_str) {
            word = SK_WILD;
            const uint32_t op = R.ev[ev].op, code = op & 15u;
            if (code == OP_CONTENT) cseg = ns; else if (code == OP_FINISH) fseg = ns;
            else if (code != OP_NONE) { if (n_ops < 24u) opw[n_ops++] = code | (ns << 8) | ((op >> 4) << 16); else fail = true; }
            ev++;
        } else if (ev < R.n && R.ev[ev].kind == WK_INT && R.ev[ev].start >= a && (uint32_t)R.ev[ev].start + R.ev[ev].len <= b && !in_str) {
            const uint32_t ia = R.ev[ev].start, ib = ia + R.ev[ev].len, pre = ia - a, suf = b - ib;
            if (pre > 255u || suf > 255u || lit_used + pre + suf > T_LIT_MAX) { fail = true; break; }
            word = SK_LITINT | (pre << 2) | (suf << 10) | (lit_used << 18);
            for (uint32_t i = 0; i < pre; i++) lit[lit_used++] = S.tile[a + i];
            for (uint32_t i = 0; i < suf; i++) lit[lit_used++] = S.tile[ib + i];
            const uint32_t op = R.ev[ev].op, code = op & 15u;
            // (range checks are not ops: the replay leaves integers of more than 18 digits to the automaton)
            if (code != OP_NONE && code != OP_CHK_I64 && code != OP_CHK_F32) { if (n_ops < 24u) opw[n_ops++] = code | (ns << 8) | ((op >> 4) << 16); else fail = true; }
            ev++;
            if (ev < R.n && R.ev[ev].start < b) { fail = true; break; }     // a second wildcard in the same segment
        } else {
            if (ev < R.n && R.ev[ev].start < b) { fail = true; break; }     // a wildcard that does not line up with a segment
            if (len > 255u || lit_used + len > T_LIT_MAX) { fail = true; break; }
            if (len <= 3u) {
                word = SK_LIT3 | (len << 2);
                for (uint32_t i = 0; i < len; i++) word |= (uint32_t)S.tile[a + i] << (8u + 8u * i);
            } else {
                word = SK_LIT | (len << 2) | (lit_used << 18);
                for (uint32_t i = 0; i < len; i++) lit[lit_used++] = S.tile[a + i];
            }
        }
        segw[ns] = word;
        if (at_end) break;
        if (ns >= 63u) { fail = true; break; }
        if (c == '[') { if (ns < 32u) mask0 |= 1u << ns; else mask1 |= 1u << (ns - 32u); }
        else in_str = !in_str;
        ns++;
        seg_a = q + 1u; p = q + 1u;
    }
    if (fail || in_str || ev != R.n) return;
    const uint32_t n_struct = ns;
    const uint32_t words = T_HDR + (n_struct + 1u) + n_ops + (tc_count ? 4u : 0u) + ((lit_used + 3u) >> 2) + 1u;
    if (off + words > (uint32_t)TS_WORDS) return;
    uint32_t *opsw = segw + n_struct + 1u, *tcs = opsw + n_ops, *pool = tcs + (tc_count ? 4u : 0u);
    for (uint32_t i = 0; i < n_ops; i++) opsw[i] = opw[i];
    if (tc_count) {
        uint32_t w4[4] = { 0, 0, 0, 0 }, t = tc_first;
        for (uint32_t j = 0; j < tc_count && t != SSE_NONE; j++) { w4[j >> 2] |= (P.tcs[t].flags & 7u) << ((j & 3u) * 8u); t = P.tcs[t].next; }
        tcs[0] = w4[0]; tcs[1] = w4[1]; tcs[2] = w4[2]; tcs[3] = w4[3];
    }
    for (uint32_t i = 0; i < lit_used; i += 4u) {
        uint32_t v = 0;
        for (uint32_t b = 0; b < 4u && i + b < lit_used; b++) v |= (uint32_t)lit[i + b] << (8u * b);
        pool[i >> 2] = v;
    }
    pool[(lit_used + 3u) >> 2] = 0;                        // (unaligned pool reads look one word ahead)
    T[1] = lit_used | (tflags << 16) | (tc_count << 24); T[2] = rec_static; T[3] = n_choices | (n_ops << 16);
    T[4] = mask0; T[5] = mask1; T[6] = cseg | (fseg << 8);
    // the same skeleton may have been stored by another lane meanwhile: identical words
    for (uint32_t o = S.thead[n_struct]; o; o = S.tstore[o] & 0xFFFFu) {
        const uint32_t *U = S.tstore + o;
        bool same = true;
        for (uint32_t i = 1; i < words && same; i++) same = U[i] == T[i];
        if (same) return;
    }
    T[0] = (n_struct << 16) | (S.thead[n_struct] & 0xFFFFu);
    __threadfence_block();
    S.ts_used = off + words;
    S.thead[n_struct] = off;                               // published: readers see a complete template
}

// A line retires: final syntax check, record, termination bookkeeping (agent.go:205-242).
__device__ __forceinline__ void f_finish_line(const KParams &P, FSmem &S, FLane &L) {
    if (!(L.sf & SF_SYN)) {
        if (L.depth == 0 && (L.st == S_NZERO || L.st == S_NINT || L.st == S_NFRAC || L.st == S_NEXP)) {
            f_number_end(P, S, L, L.pe - L.slen - 1u, L.pe, L.st == S_NZERO || L.st == S_NINT);
            L.st = S_END;
        }
        if (L.st != S_END) L.sf |= SF_SYN;
    }
    // a syntax error stops the walk: the rest of the payload has not been looked at for "[DONE]" (agent.go:181)
    if ((L.sf & SF_SYN) && (L.sf & SF_RMODE) && !(L.sf & SF_DONELINE) && has_done_scan(S, L.pe - L.plen, L.pe)) L.sf |= SF_DONELINE;
    f_emit_record(P, S, L.sf, L.n_choices, L.usage_idx, L.content_pos, L.content_len, L.finish, L.tc_count, L.tc_first, L.rec, L.plen,
                  L.line, L.delta);
    L.busy = false;
    if (L.rslot != SSE_NONE) {      // the automaton recorded this line: keep its skeleton as a template
        const FRec &R = S.rec[L.rslot];
        // one lane builds at a time (a second one, most likely holding the same skeleton, just drops its recording)
        if (!R.nonsimple && !(L.sf & (SF_SYN | SF_TYPE | SF_DEPTH | SF_DONELINE)) && atomicCAS(&S.build_lock, 0u, 1u) == 0u) {
            t_build(P, S, L.rslot, L.pe - L.plen, L.pe, SSE_F_JSON_OK | ((L.sf & SF_TCNONNIL) ? SSE_F_TC_NONNIL : 0u),
                    ((L.sf & SF_USAGE) && L.usage_idx != SSE_NONE) ? TF_HAS_USAGE : 0u, L.n_choices, L.tc_count, L.tc_first);
            __threadfence_block();
            atomicExch(&S.build_lock, 0u);
        }
        atomicAnd(&S.rec_busy, ~(1u << L.rslot));
        L.rslot = SSE_NONE;
    }
}

// lane state for the line of decode job j
__device__ __forceinline__ void lane_setup(const KParams &P, const FSmem &S, FLane &L, uint32_t j, uint32_t rb) {
    const uint32_t k = S.job[j];
    const FLine ln = S.line[k];
    const FSeg &sg = S.seg[ln.seg];
    const uint32_t pay_s = (ln.flags & LF_PREF) ? ln.a + 6u : ln.a;
    L.p = pay_s; L.pe = ln.b; L.plen = L.pe - L.p; L.line = k;
    L.rec = rb + ln.rank_r;
    const uint32_t src_s = (ln.flags & LF_RMODE) ? ln.a : ln.start;
    L.delta = (ln.flags & LF_ZC) ? P.in_base + sg.in_delta : ln.out_off - src_s;
    L.st = S_VAL; L.depth = L.skip = L.sd = 0; L.cur = TY_ROOT | (N_ROOT << 4); L.slen = 0;
    L.sf = ((ln.flags & LF_RMODE) ? SF_RMODE : 0u) | ((ln.flags & LF_DONE) ? SF_DONELINE : 0u);
    L.choices_count = L.n_choices = 0; L.finish = SSE_FIN_NONE; L.ct = L.ct1 = L.sstk = 0;
    L.content_pos = L.content_len = 0; L.tc_count = 0; L.tc_first = L.tc_prev = L.tc_cur = SSE_NONE; L.tcb = 0;
    L.usage_idx = SSE_NONE; L.rslot = SSE_NONE;
    L.busy = true;
}

// A template with usage / tool-call / range-check ops has fitted (rare lines: first tool-call chunk, usage chunk): one lane
// runs the ops and writes the record. Out of line: not part of the steady-state code.
__device__ __noinline__ void replay_ops(const KParams &P, FSmem &S, FWarp &W, const uint16_t *SS, bool clean, const uint32_t *T, uint32_t k, uint32_t j, uint32_t rb,
                                        uint32_t ps, uint32_t pe, uint32_t n_struct, uint32_t cpos, uint32_t clen, uint32_t d2, uint32_t fin, bool done) {
    const FLine ln = S.line[k];
    const bool rmode = (ln.flags & LF_RMODE) != 0;
    const uint32_t n_ops = T[3] >> 16, tc_count = T[1] >> 24, tflags = (T[1] >> 16) & 0xFFu;
    const FSeg &sg = S.seg[ln.seg];
    const uint32_t src_s = rmode ? ln.a : ln.start;
    const uint32_t delta = (ln.flags & LF_ZC) ? P.in_base + sg.in_delta : ln.out_off - src_s;
    uint32_t sf = (rmode ? SF_RMODE : 0u) | (done ? SF_DONELINE : 0u) | ((d2 & 1u) ? SF_CDEC : 0u) | ((d2 & 2u) ? SF_CBAD : 0u);
    uint32_t usage_idx = SSE_NONE, tc_base = SSE_NONE, tc_dyn = 0;
    const uint32_t *opsw = T + T_HDR + n_struct + 1u, *tc_static = opsw + n_ops;
    if (tflags & TF_HAS_USAGE) { usage_idx = f_usage_alloc(P); sf |= SF_USAGE; }
    if (tc_count) tc_base = f_tcs_alloc(P, tc_count, tc_static);
    FLane C; C.delta = delta;
    for (uint32_t i = 0; i < n_ops; i++) {
        const uint32_t code = opsw[i] & 0xFFu, s = (opsw[i] >> 8) & 0xFFu, ord = opsw[i] >> 16;
        uint32_t a = s == 0 ? ps : (uint32_t)SS[s - 1u] + 1u, b = s == n_struct ? pe : (uint32_t)SS[s];
        if (code >= OP_TC_INDEX) {                    // an integer: inside the segment's punctuation
            const uint32_t sw = T[T_HDR + s];
            a += (sw >> 2) & 0xFFu; b -= (sw >> 10) & 0xFFu;
        }
        switch (code) {
        case OP_TC_ID: case OP_TC_TYPE: case OP_TC_NAME: case OP_TC_ARGS:
            if (tc_base != SSE_NONE) {
                const uint32_t kf = code - OP_TC_ID, dd = clean ? 0u : (W.sdirty[s >> 2] >> ((s & 3u) * 8u)) & 0xFFu;
                const uint32_t e2 = (dd & 1u) | (((dd & 2u) && body_has_bad_utf8(S, a, b)) ? 2u : 0u);
                sse_tc *t = &P.tcs[tc_base + ord];
                uint32_t *span = &t->id_off + 2u * kf;
                f_cancel_job(S, span + 1);
                const Span sp = f_capture(P, S, C, a, b - a, e2, span + 1);
                span[0] = sp.off; span[1] = sp.len;
                const uint32_t text_bit = SSE_TC_ID_TEXT << kf;
                t->flags = (t->flags & ~text_bit) | (sp.text ? text_bit : 0u);
                if (kf >= 2u) { const uint32_t bb = 1u << (2u * ord + (kf - 2u)); tc_dyn = (b > a) ? (tc_dyn | bb) : (tc_dyn & ~bb); }
            }
            break;
        case OP_TC_INDEX: sf |= f_number_value(P, S.tile, TY_INT, TG_TC_INDEX, a, b, SSE_NONE, tc_base != SSE_NONE ? tc_base + ord : SSE_NONE); break;
        case OP_U_PROMPT: sf |= f_number_value(P, S.tile, TY_INT, TG_PROMPT, a, b, usage_idx, SSE_NONE); break;
        case OP_U_COMPLETION: sf |= f_number_value(P, S.tile, TY_INT, TG_COMPLETION, a, b, usage_idx, SSE_NONE); break;
        case OP_U_TOTAL: sf |= f_number_value(P, S.tile, TY_INT, TG_TOTAL, a, b, usage_idx, SSE_NONE); break;
        case OP_CHK_I64: if (b - a > 18u) sf |= f_number_value(P, S.tile, TY_INT, TG_NONE, a, b, SSE_NONE, SSE_NONE); break;
        case OP_CHK_F32: if (b - a > 18u) sf |= f_number_value(P, S.tile, TY_F32, TG_NONE, a, b, SSE_NONE, SSE_NONE); break;
        default: break;
        }
    }
    if (T[2] & SSE_F_TC_NONNIL) sf |= SF_TCNONNIL;
    const uint8_t *st8 = reinterpret_cast<const uint8_t *>(tc_static);
    for (uint32_t q = 0; q < tc_count; q++)
        if ((st8[q] & SSE_TC_HAS_ID) || ((st8[q] & SSE_TC_HAS_FUNC) && ((tc_dyn >> (2u * q)) & 3u))) sf |= SF_TCVALID;
    f_emit_record(P, S, sf, T[3] & 0xFFFFu, usage_idx, cpos, clen, fin, tc_base != SSE_NONE ? tc_count : 0u, tc_base, rb + ln.rank_r,
                  pe - ps, k, delta);
    FRes rs; rs.cpos = rs.clen = rs.toff = 0; rs.misc = 128u;      // done: nothing left for the record pass
    S.res[j] = rs;
}

// ---- warp-per-line replay
// One warp, one line. Returns true when a template fitted: the line's captures are then in S.res[job] (content and
// finish_reason only) for the lane-per-line record pass, or -- templates with usage / tool-call / range-check ops -- the
// record has been written right here by lane 0.
__device__ __noinline__ bool warp_replay(const KParams &P, FSmem &S, uint32_t j, uint32_t rb) {
    const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
    const uint32_t lt = (1u << lane) - 1u;
    FWarp &W = S.wsc[wid];
    const uint32_t k = S.job[j];
    const FLine ln = S.line[k];
    if (ln.flags & LF_DONE) return false;         // swallowed "[DONE]" lines: their flag is not part of a template
    const uint32_t ps = (ln.flags & LF_PREF) ? ln.a + 6u : ln.a, pe = ln.b;
    const bool rmode = (ln.flags & LF_RMODE) != 0;
    if (pe <= ps) return false;
    // ---- 1. the stop bytes of the payload, in order
    uint32_t n_stops = 0;
    const uint32_t w_end = (pe - 1u) >> 5;
    #pragma unroll 1
    for (uint32_t wb = ps >> 5; wb <= w_end; wb += 32u) {
        const uint32_t w = wb + lane;
        uint32_t bits = w <= w_end ? S.stopbm[w] : 0u;
        const uint32_t wpos = w << 5;
        if (wpos < ps) bits &= 0xFFFFFFFFu << (ps - wpos);
        if (w == w_end && (pe & 31u)) bits &= (1u << (pe & 31u)) - 1u;
        const uint32_t cnt = __popc(bits), incl = warp_incl(cnt, lane);
        uint32_t base = n_stops + incl - cnt;
        #pragma unroll
        for (int q = 0; q < 3; q++)                    // (a 32-byte word rarely holds more than three stops)
            if (bits) {
                const uint32_t b = (uint32_t)__ffs(bits) - 1u;
                bits &= bits - 1u;
                if (base < (uint32_t)W_STOPS) W.spos[base] = (uint16_t)(wpos + b);
                base++;
            }
        #pragma unroll 1
        while (bits) {
            const uint32_t b = (uint32_t)__ffs(bits) - 1u;
            bits &= bits - 1u;
            if (base < (uint32_t)W_STOPS) W.spos[base] = (uint16_t)(wpos + b);
            base++;
        }
        n_stops += __shfl_sync(FULL, incl, 31);
    }
    if (n_stops > (uint32_t)W_STOPS) return false;
    __syncwarp();
    // ---- 2a. the usual line: every stop is a quote or a '[' outside strings -- all of them structural, nothing to validate
    const uint16_t *SS = W.spos;
    bool clean = true;
    {
        uint32_t par = 0;
        bool odd = false;
        #pragma unroll 1
        for (uint32_t r0 = 0; r0 < n_stops; r0 += 32u) {
            const uint32_t i = r0 + lane;
            const bool have = i < n_stops;
            const uint32_t c = have ? (uint32_t)S.tile[W.spos[i]] : (uint32_t)'"';
            const unsigned qm = __ballot_sync(FULL, have && c == '"');
            const bool inside = ((par + __popc(qm & lt)) & 1u) != 0;
            if (have && c != '"' && (c != '[' || inside)) odd = true;
            par ^= __popc(qm) & 1u;
        }
        clean = !__any_sync(FULL, odd) && !par && n_stops <= (uint32_t)W_STRUCT;
    }
    uint32_t parity = 0, n_struct = clean ? n_stops : 0u;
    bool bad = false, done = false;
    if (!clean) {
    SS = W.sstop;
    if (lane < (uint32_t)(W_STRUCT + 8) / 4u) W.sdirty[lane] = 0;
    __syncwarp();
    // ---- 2b. which stops are structural (string parity by ballot); are the others harmless?
    #pragma unroll 1
    for (uint32_t r0 = 0; r0 < n_stops; r0 += 32u) {
        const uint32_t i = r0 + lane;
        const bool have = i < n_stops;
        const uint32_t p = have ? (uint32_t)W.spos[i] : ps;
        const uint32_t c = have ? (uint32_t)S.tile[p] : 0u;
        uint32_t run = 0;
        if (have && (c == '"' || c == '\\') && p > ps && S.tile[p - 1u] == '\\') run = backslash_run_before(S, p, ps);
        const bool is_q = have && c == '"' && !(run & 1u);
        const unsigned qm = __ballot_sync(FULL, is_q);
        const bool inside = ((parity + __popc(qm & lt)) & 1u) != 0;       // inside a string before this stop
        const bool brk = have && c == '[' && !inside;
        const unsigned sm = __ballot_sync(FULL, is_q || brk);
        const uint32_t segi = n_struct + __popc(sm & lt);                  // structural stops before this one = its segment
        if (have && !is_q && !brk) {
            if (!inside) bad = true;                                       // a stray byte between tokens: the automaton's business
            else if (c < 0x20u) bad = true;
            else if (c == '\\') {
                if (!(run & 1u) && !escape_ok(S, p, pe)) bad = true;      // an escaping backslash: what follows must be an escape
                if (segi < (uint32_t)W_STRUCT + 2u) atomicOr(&W.sdirty[segi >> 2], 1u << ((segi & 3u) * 8u));
            } else if (c >= 0x80u) { if (segi < (uint32_t)W_STRUCT + 2u) atomicOr(&W.sdirty[segi >> 2], 2u << ((segi & 3u) * 8u)); }
            else if (c == '[') { if (rmode && p + 6u <= pe && is_done_at(S.tile + p)) done = true; }
        }
        if (is_q || brk) { if (segi < (uint32_t)W_STRUCT) W.sstop[segi] = (uint16_t)p; }
        n_struct += __popc(sm);
        parity ^= __popc(qm) & 1u;
    }
    if (__any_sync(FULL, bad) || parity || n_struct > (uint32_t)W_STRUCT) return false;
    done = __any_sync(FULL, done);
    __syncwarp();
    }
    // ---- 3. a template with these structural stops and segments?
    uint32_t off = S.thead[n_struct];
    const uint32_t *T = nullptr;
    #pragma unroll 1
    for (; off; off = S.tstore[off] & 0xFFFFu) {
        const uint32_t *U = S.tstore + off;
        const uint32_t *segw = U + T_HDR;
        const uint32_t n_ops = U[3] >> 16, tc_count = U[1] >> 24;
        const uint32_t *pool = segw + n_struct + 1u + n_ops + (tc_count ? 4u : 0u);
        bool ok = true;
        #pragma unroll 1
        for (uint32_t s0 = 0; s0 <= n_struct; s0 += 32u) {
            const uint32_t s = s0 + lane;
            if (s <= n_struct) {
                const uint32_t a = s == 0 ? ps : (uint32_t)SS[s - 1u] + 1u, b = s == n_struct ? pe : (uint32_t)SS[s], len = b - a;
                if (s < n_struct) {
                    const uint32_t isb = S.tile[b] == '[' ? 1u : 0u;
                    if (isb != (((s < 32u ? U[4] : U[5]) >> (s & 31u)) & 1u)) ok = false;
                }
                const uint32_t sw = segw[s], kind = sw & 3u, la = (sw >> 2) & 0xFFu, lb = (sw >> 10) & 0xFFu, lo = sw >> 18;
                if (kind == SK_LIT3) {
                    const uint32_t l3 = (sw >> 2) & 3u;
                    if (len != l3 || (l3 && ((load4(S, a) ^ (sw >> 8)) & (0xFFFFFFu >> ((3u - l3) * 8u))))) ok = false;
                }
                else if (kind == SK_LIT) { if (len != la || !seg_equal(S, a, pool, lo, la)) ok = false; }
                else if (kind == SK_LITINT) {     // (an integer of more than 18 digits needs a range check: the automaton's business)
                    if (len <= la + lb || len > la + lb + 18u || !seg_equal(S, a, pool, lo, la) || !seg_equal(S, b - lb, pool, lo + la, lb) || !int_ok(S, a + la, b - lb)) ok = false;
                }
            }
        }
        if (__all_sync(FULL, ok)) { T = U; break; }
    }
    if (!T) return false;
    // ---- 4. the captures
    const uint32_t cseg = T[6] & 0xFFu, fseg = (T[6] >> 8) & 0xFFu, n_ops = T[3] >> 16, tc_count = T[1] >> 24, tflags = (T[1] >> 16) & 0xFFu;
    if (lane == 0) {
        uint32_t cpos = 0, clen = 0, d2 = 0, fin = SSE_FIN_NONE;
        if (cseg != 0xFFu) {
            cpos = (uint32_t)SS[cseg - 1u] + 1u; clen = (uint32_t)SS[cseg] - cpos;
            const uint32_t dd = clean ? 0u : (W.sdirty[cseg >> 2] >> ((cseg & 3u) * 8u)) & 0xFFu;
            d2 = (dd & 1u) | (((dd & 2u) && body_has_bad_utf8(S, cpos, cpos + clen)) ? 2u : 0u);
        }
        if (fseg != 0xFFu) {
            const uint32_t fp = (uint32_t)SS[fseg - 1u] + 1u, fl = (uint32_t)SS[fseg] - fp;
            const uint32_t dd = clean ? 0u : (W.sdirty[fseg >> 2] >> ((fseg & 3u) * 8u)) & 0xFFu;
            fin = f_match_finish(S, fp, fl, dd ? 1u : 0u);
        }
        if (n_ops == 0 && !(tflags & TF_HAS_USAGE) && tc_count == 0) {
            FRes rs; rs.cpos = (uint16_t)cpos; rs.clen = (uint16_t)clen; rs.toff = (uint16_t)(T - S.tstore);
            rs.misc = (uint16_t)(d2 | (fin << 2) | (done ? 32u : 0u) | 64u);
            S.res[j] = rs;
        } else {
            replay_ops(P, S, W, SS, clean, T, k, j, rb, ps, pe, n_struct, cpos, clen, d2, fin, done);
        }
    }
    __syncwarp();
    return true;
}

// Automaton path of stage 2: the lanes whose line no template took.
__device__ __noinline__ void stage2_automaton(const KParams &P, FSmem &S, bool has, uint32_t j, uint32_t rb) {
    FLane L;
    L.busy = false; L.p = L.pe = 0; L.plen = 0; L.sf = 0; L.rslot = SSE_NONE; L.line = 0; L.rec = 0; L.delta = 0;
    L.st = S_END; L.depth = L.skip = L.sd = 0; L.cur = 0; L.slen = 0; L.choices_count = L.n_choices = 0; L.finish = 0;
    L.ct = L.ct1 = L.sstk = 0; L.content_pos = L.content_len = 0; L.tc_count = 0; L.tc_first = L.tc_prev = L.tc_cur = SSE_NONE;
    L.tcb = 0; L.usage_idx = SSE_NONE;
    if (has) {
        lane_setup(P, S, L, j, rb);
        if ((P.flags & SSE_FLAG_TEMPLATES) && !(L.sf & SF_DONELINE) && S.ts_used + 360u <= (uint32_t)TS_WORDS) {
            uint32_t m = S.rec_busy;                 // record a template while the automaton walks the line
            while ((~m) & ((1u << NREC) - 1u)) {
                const uint32_t b = (uint32_t)__ffs((~m) & ((1u << NREC) - 1u)) - 1u;
                const uint32_t old = atomicCAS(&S.rec_busy, m, m | (1u << b));
                if (old == m) { L.rslot = b; FRec &R = S.rec[b]; R.n = 0; R.nonsimple = 0; R.n_str = 0; R.n_arr = 0; break; }
                m = old;
            }
        }
    }
    while (__any_sync(FULL, L.busy)) {
        #pragma unroll 1
        for (int r = 0; r < 4; r++) {
            f_step(P, S, L);
            if (L.busy && L.p >= L.pe) f_finish_line(P, S, L);
        }
    }
}

// Stage 2 of a round: (a) every warp takes lines one at a time through the templates; (b) the lines no template took go
// through the automaton, one lane per line; (c) after a block barrier (process_window) one thread per line writes the records
// of the lines whose captures (a) left in S.res.
__device__ void stage2(const KParams &P, FSmem &S, uint32_t n_jobs, uint32_t rb) {
    const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
    #pragma unroll 1
    for (uint32_t j = wid; j < n_jobs; j += F_WARPS) {
        bool hit = false;
        if ((P.flags & SSE_FLAG_TEMPLATES)) hit = warp_replay(P, S, j, rb);
        if (!hit && lane == 0) { FRes z; z.cpos = z.clen = z.toff = 0; z.misc = 0; S.res[j] = z; }
    }
    __syncwarp();
    // the lines no template took: lane i has this warp's i-th line
    const uint32_t mj = wid + F_WARPS * lane;
    const bool miss = mj < n_jobs && S.res[mj].misc == 0;
    if (__any_sync(FULL, miss)) stage2_automaton(P, S, miss, mj, rb);
}

// (c): records of the lines whose template captures are content / finish_reason only. One thread per job.
__device__ __forceinline__ void stage2_records(const KParams &P, FSmem &S, uint32_t n_jobs, uint32_t rb) {
    for (uint32_t j = threadIdx.x; j < n_jobs; j += F_THREADS) {
        const FRes rs = S.res[j];
        if (!(rs.misc & 64u)) continue;
        const uint32_t k = S.job[j];
        const FLine ln = S.line[k];
        const FSeg &sg = S.seg[ln.seg];
        const bool rmode = (ln.flags & LF_RMODE) != 0;
        const uint32_t ps = (ln.flags & LF_PREF) ? ln.a + 6u : ln.a, src_s = rmode ? ln.a : ln.start;
        const uint32_t delta = (ln.flags & LF_ZC) ? P.in_base + sg.in_delta : ln.out_off - src_s;
        const uint32_t *T = S.tstore + rs.toff;
        const uint32_t d2 = rs.misc & 3u;
        const uint32_t sf = (rmode ? SF_RMODE : 0u) | ((rs.misc & 32u) ? SF_DONELINE : 0u) | ((d2 & 1u) ? SF_CDEC : 0u) | ((d2 & 2u) ? SF_CBAD : 0u) |
                            ((T[2] & SSE_F_TC_NONNIL) ? SF_TCNONNIL : 0u);
        f_emit_record(P, S, sf, T[3] & 0xFFFFu, SSE_NONE, rs.cpos, rs.clen, (rs.misc >> 2) & 7u, 0u, SSE_NONE, rb + ln.rank_r, ln.b - ps, k, delta);
    }
}

// ---------------------------------------------------------------- one window of the tile: stage 1a .. finish of its rounds
// S.seg[0..nseg) describe the regions; fill = end of the last region. Returns through the segment table.
__device__ __noinline__ void process_window(const KParams &P, FSmem &S, uint32_t first_seg, uint32_t nseg, uint32_t fill) {
    const uint32_t tid = threadIdx.x, lane = tid & 31u, w = tid >> 5;
    const bool zero_copy = !(P.flags & SSE_FLAG_COPY_OUT);
    stage1a(S, fill);
    __syncthreads();

    uint32_t r_start = 0;
    #pragma unroll 1
    for (;;) {   // rounds of up to LCAP lines
        // ---------------- stage 1b: newline bits of this thread's 128 bytes, line table
        uint32_t nlm[4], cnt = 0;
        #pragma unroll
        for (int j = 0; j < 4; j++) {
            const uint32_t wi = tid * 4u + (uint32_t)j, wpos = wi << 5;
            uint32_t m = 0;
            if (wpos < fill && wpos + 32u > r_start) {
                m = S.nlbm[wi];
                if (wpos + 32u > fill) m &= (1u << (fill - wpos)) - 1u;
                if (wpos < r_start) m &= 0xFFFFFFFFu << (r_start - wpos);
            }
            nlm[j] = m; cnt += __popc(m);
        }
        uint32_t total;
        const uint32_t base = block_scan1(S, cnt, total);
        {
            uint32_t idx = base;
            #pragma unroll
            for (int j = 0; j < 4; j++) {
                uint32_t m = nlm[j];
                const uint32_t wpos = (tid * 4u + (uint32_t)j) << 5;
                #pragma unroll 1
                while (m) {
                    const uint32_t b = (uint32_t)__ffs(m) - 1u;
                    m &= m - 1u;
                    if (idx < (uint32_t)LCAP) S.line[idx].nl = (uint16_t)(wpos + b);
                    idx++;
                }
            }
        }
        const uint32_t n_lines = min(total, (uint32_t)LCAP);
        if (tid < nseg) { FSeg &sg = S.seg[tid]; sg.term = SSE_NONE; sg.dead = SSE_NONE; sg.rf0 = SSE_NONE; sg.rr0 = SSE_NONE; sg.fcnt = 0; sg.rcnt = 0; }
        if (tid == 0) { S.bc[9] = 0; S.jq_n = 0; }    // materialised lines, unquote jobs of this round
        __syncthreads();
        if (n_lines == 0) break;

        // ---------------- classify: one thread per line
        const uint32_t k = tid;
        uint32_t kind = K_DROP, lflags = 0, mat = 0, flen = 0, my_seg = 0;
        if (k < n_lines) {
            const uint32_t nl = S.line[k].nl;
            uint32_t lo = 0, hi = nseg;             // last segment with data_off <= nl
            #pragma unroll 1
            while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (S.seg[mid].data_off <= nl) lo = mid; else hi = mid; }
            my_seg = lo;
            const FSeg &sg = S.seg[lo];
            const uint32_t prev_end = k > 0 ? (uint32_t)S.line[k - 1].nl + 1u : r_start;
            const uint32_t start = max(prev_end, sg.data_off);
            uint32_t mode = sg.mode;
            if (mode & SSE_MODE_R) mode |= SSE_MODE_PARSE;
            int a = (int)start, b = (int)nl + 1;
            if (sg.state & (FS_SKIP | FS_TERM | FS_DEAD)) kind = K_DROP;
            else if (nl + 1u - start > P.carry_slot) { atomicMin(&S.seg[lo].dead, k); kind = K_DROP; }   // the line with its '\n', as the produce kernel counts it
            else if (mode & SSE_MODE_R) {
                lflags |= LF_RMODE;
                { const uint32_t ab = trim_space_ab(S.tile, (uint32_t)a, (uint32_t)b); a = (int)(ab & 0xFFFFu); b = (int)(ab >> 16); }   // agent.go:178-179
                const bool pref = is_data_prefix(S.tile + a, b - a);               // agent.go:186
                if (pref && b - a > 6) {                                           // agent.go:190-197; "[DONE]" is found by the decoder
                    kind = K_EMIT; lflags |= LF_PARSE | LF_PREF | LF_JOB; flen = (uint32_t)(b - a) + 2u;
                    if (b - a == 12 && is_done_at(S.tile + a + 6)) { kind = K_DONE_EXACT; lflags = (lflags & ~LF_JOB) | LF_DONE; flen = 0; }   // agent.go:394-396
                    else if (zero_copy && b == (int)nl && (uint32_t)a >= sg.in_pos && nl + 1u < sg.end && S.tile[nl + 1u] == '\n') lflags |= LF_ZC;
                    else mat = flen;
                } else if (b > a && has_done_scan(S, (uint32_t)a, (uint32_t)b)) {  // swallowed, still parsed (agent.go:182, :377-402)
                    kind = K_DONE; lflags |= LF_PARSE | LF_DONE | LF_JOB | (pref ? LF_PREF : 0);
                    if (zero_copy && (uint32_t)a >= sg.in_pos) lflags |= LF_ZC; else mat = (uint32_t)(b - a);
                }
            } else {
                kind = K_EMIT; flen = nl + 1u - start;                             // routes.go:613 verbatim
                if (zero_copy && start >= sg.in_pos) lflags |= LF_ZC; else mat = flen;
                if ((mode & SSE_MODE_PARSE) && is_data_prefix(S.tile + start, (int)(nl + 1u - start))) { lflags |= LF_PARSE | LF_PREF | LF_JOB; b = (int)nl; }
            }
            FLine &ln = S.line[k];
            ln.start = (uint16_t)start; ln.a = (uint16_t)a; ln.b = (uint16_t)b; ln.seg = (uint8_t)lo;
        }
        __syncthreads();
        // ---------------- allocate records, decode jobs and materialised bytes (one atomicAdd each per round)
        if (k < n_lines && k >= S.seg[my_seg].dead) { kind = K_DROP; lflags &= LF_RMODE; mat = 0; flen = 0; }
        uint32_t vrj = ((lflags & LF_PARSE) ? 1u : 0u) | ((lflags & LF_JOB) ? 0x10000u : 0u), vb = mat;
        uint32_t tot_rj, tot_b;
        block_scan2(S, vrj, vb, tot_rj, tot_b);
        const uint32_t vr = vrj & 0xFFFFu, tot_r = tot_rj & 0xFFFFu, tot_j = tot_rj >> 16;
        if (mat) S.matlist[atomicAdd(&S.bc[9], 1u)] = (uint16_t)k;
        if (tid == 0) {
            uint32_t rb = 0, ob = 0, ovf = 0;
            if (tot_r) rb = atomicAdd(&P.ctr->n_recs, tot_r);
            if (tot_b) ob = atomicAdd(&P.ctr->out_bytes, (tot_b + 15u) & ~15u);
            if (rb + tot_r > P.cap_recs || (tot_b && ob + tot_b + 16u > P.cap_out)) { sse_overflow(P.ctr, SSE_OVF_OUT); ovf = 1; }
            S.bc[1] = rb; S.bc[2] = ob; S.bc[3] = ovf;
        }
        __syncthreads();
        const uint32_t rb = S.bc[1], ob = S.bc[2];
        if (S.bc[3]) return;                      // the batch is reported as overflowed: stop touching result arenas
        // template bucket of a line to decode: its number of stop bytes (stage 2)
        if (k < n_lines && (lflags & LF_JOB)) {
            const FLine &ln = S.line[k];
            S.line[k].pad = (uint8_t)min(count_stops(S, (lflags & LF_PREF) ? ln.a + 6u : ln.a, ln.b), 255u);
        }
        if (k < n_lines) {
            FLine &ln = S.line[k];
            ln.flags = (uint16_t)(kind | lflags | (mat ? LF_MAT : 0));
            ln.rank_r = (uint16_t)vr; ln.out_off = ob + vb;
            if (lflags & LF_JOB) S.job[vrj >> 16] = (uint16_t)k;
            if (kind == K_DONE_EXACT) {
                sse_rec r; r.frame = SSE_NONE; r.flags = SSE_F_DONE_LINE | SSE_F_DONE_EXACT; r.content_off = r.content_len = 0;
                r.tc_first = SSE_NONE; r.tc_count = 0; r.n_choices = 0; r.usage = SSE_NONE; r.payload_len = 6;
                P.recs[rb + vr] = r;
            }
        }
        __syncthreads();
        // ---------------- decode
        stage2(P, S, tot_j, rb);
        __syncthreads();
        stage2_records(P, S, tot_j, rb);
        __syncthreads();
        #pragma unroll 1
        for (uint32_t i = w; i < min(S.jq_n, (uint32_t)JQ_CAP); i += F_WARPS) {      // unquote jobs: one warp per string
            const FJob jb = S.jq[i];
            if (jb.patch) warp_unquote2(S.tile, jb.s, jb.e, P.text + jb.dst, jb.patch);
        }
        // ---------------- frames (after early termination is known), record -> frame links, runs
        uint32_t vf = 0, tot_f;
        bool in_cut = false;
        if (k < n_lines) {
            const FSeg &sg = S.seg[my_seg];
            const uint32_t cut = min(sg.term == SSE_NONE ? SSE_NONE : sg.term + 1u, sg.dead);
            in_cut = k < cut;
            kind = S.line[k].flags & LF_KIND;
            lflags = S.line[k].flags;
            vf = (in_cut && kind == K_EMIT && !(lflags & LF_DONE)) ? 1u : 0u;
        }
        vf = block_scan1(S, vf, tot_f);
        if (tid == 0) {
            uint32_t fb = 0, ovf = 0;
            if (tot_f) fb = atomicAdd(&P.ctr->n_frames, tot_f);
            if (fb + tot_f > P.cap_frames) { sse_overflow(P.ctr, SSE_OVF_OUT); ovf = 1; }
            S.bc[1] = fb; S.bc[3] = ovf;
        }
        __syncthreads();
        if (S.bc[3]) return;
        const uint32_t fb = S.bc[1];
        if (k < n_lines && in_cut) {
            const FLine ln = S.line[k];
            FSeg &sg = S.seg[my_seg];
            const bool emit = kind == K_EMIT && !(lflags & LF_DONE);
            if (emit) {
                const uint32_t src_s = (lflags & LF_RMODE) ? ln.a : ln.start;
                sse_frame f; f.len = (lflags & LF_RMODE) ? (uint32_t)(ln.b - ln.a) + 2u : (uint32_t)ln.nl + 1u - ln.start;
                f.off = (lflags & LF_ZC) ? P.in_base + sg.in_delta + src_s : ln.out_off;
                P.frames[fb + vf] = f;
                atomicMin(&sg.rf0, fb + vf); atomicAdd(&sg.fcnt, 1u);
            }
            if (lflags & LF_PARSE) {
                if (emit) P.recs[rb + ln.rank_r].frame = fb + vf;
                atomicMin(&sg.rr0, rb + ln.rank_r); atomicAdd(&sg.rcnt, 1u);
            }
        }
        // ---------------- serializer: lines whose bytes do not stand in the input as they must be sent
        #pragma unroll 1
        for (uint32_t i = w; i < S.bc[9]; i += F_WARPS) {
            const FLine ln = S.line[S.matlist[i]];
            uint8_t *dst = P.out + ln.out_off;
            if (!(ln.flags & LF_RMODE)) copy_s2g(dst, S.tile + ln.start, (int)ln.nl + 1 - (int)ln.start);
            else if ((ln.flags & LF_KIND) == K_DONE && !(ln.flags & LF_PREF)) copy_s2g(dst, S.tile + ln.a, (int)ln.b - (int)ln.a);
            else {
                const int body = (int)ln.b - (int)ln.a;        // "data: " + payload is contiguous in the tile
                copy_s2g(dst, S.tile + ln.a, body);
                if (lane < 2) dst[body + lane] = (uint8_t)'\n';
            }
        }
        __syncthreads();
        // ---------------- this round's run of every segment; connection state
        if (tid < nseg) {
            FSeg &sg = S.seg[tid];
            const uint32_t gs = first_seg + tid;
            if (sg.fcnt || sg.rcnt) {
                sse_run r; r.frame_first = sg.fcnt ? sg.rf0 : 0; r.frame_count = sg.fcnt; r.rec_first = sg.rcnt ? sg.rr0 : 0; r.rec_count = sg.rcnt; r.next = SSE_NONE;
                if (sg.nruns == 0) P.seg_results[gs].run = r;
                else {
                    const uint32_t idx = atomicAdd(&P.ctr->n_runs, 1u);
                    if (idx >= P.cap_runs) sse_overflow(P.ctr, SSE_OVF_RUNS);
                    else {
                        P.runs[idx] = r;
                        if (sg.nruns == 1) P.seg_results[gs].run.next = idx; else P.runs[sg.last_run].next = idx;
                        sg.last_run = idx;
                    }
                }
                sg.nruns++;
            }
            if (sg.term != SSE_NONE && sg.term < sg.dead) sg.state |= FS_TERM;
            else if (sg.dead != SSE_NONE) sg.state |= FS_DEAD;
        }
        if (total <= (uint32_t)LCAP) { __syncthreads(); break; }
        r_start = (uint32_t)S.line[LCAP - 1].nl + 1u;
        __syncthreads();
    }
}

// last '\n' of [lo, hi) + 1, or lo if there is none (the unterminated tail starts there)
__device__ __noinline__ uint32_t tail_start(const FSmem &S, uint32_t lo, uint32_t hi) {
    if (hi <= lo) return lo;
    int w = (int)((hi - 1u) >> 5);
    const int w0 = (int)(lo >> 5);
    for (; w >= w0; w--) {
        uint32_t bits = S.stopbm[w];
        const uint32_t wpos = (uint32_t)w << 5;
        if (wpos + 32u > hi) bits &= (hi - wpos >= 32u) ? 0xFFFFFFFFu : ((1u << (hi - wpos)) - 1u);
        if (wpos < lo) bits &= 0xFFFFFFFFu << (lo - wpos);
        while (bits) {
            const uint32_t b = 31u - (uint32_t)__clz(bits);
            if (S.tile[wpos + b] == '\n') return wpos + b + 1u;
            bits &= ~(1u << b);
        }
    }
    return lo;
}

// Final state of a segment whose bytes have all been through a window: carry tail, connection state, result.
// Called by a whole warp.
__device__ __noinline__ void finish_segment(const KParams &P, FSmem &S, uint32_t first_seg, uint32_t i) {
    const uint32_t lane = threadIdx.x & 31u;
    FSeg &sg = S.seg[i];
    const uint32_t gs = first_seg + i;
    uint32_t carry = 0, flags = 0, cflags = 0;
    if (sg.state & FS_SKIP) { carry = sg.old_carry; flags = (sg.state & FS_SKIP_DEAD) ? SSE_SEG_DEAD : SSE_SEG_FINISHED; }
    else if (sg.state & FS_TERM) { flags = SSE_SEG_TERMINATED; cflags = CONN_FINISHED; }
    else if (sg.state & FS_DEAD) { flags = SSE_SEG_LINE_TOO_LONG | SSE_SEG_DEAD; cflags = CONN_DEAD; }
    else {
        uint32_t ts = 0;
        if (lane == 0) ts = tail_start(S, sg.data_off, sg.end);
        ts = __shfl_sync(FULL, ts, 0);
        const uint32_t tl = sg.end - ts;
        if (tl > P.carry_slot) { flags = SSE_SEG_LINE_TOO_LONG | SSE_SEG_DEAD; cflags = CONN_DEAD; }
        else {
            carry = tl;
            if (tl) {   // stored so that it ENDS at a 16-byte boundary of the slot: the next batch stages it with one aligned bulk copy
                uint8_t *slot = P.carry + (size_t)sg.conn * P.carry_slot;
                const uint32_t pad = (16u - (tl & 15u)) & 15u;
                copy_s2g(slot + pad, S.tile + ts, (int)tl);
            }
        }
    }
    if (lane == 0) {
        if (!(sg.state & FS_SKIP)) { ConnState ns; ns.carry_len = carry; ns.flags = cflags; P.conns[sg.conn] = ns; }
        sse_seg_result *r = &P.seg_results[gs];
        if (sg.nruns == 0) { sse_run z; z.frame_first = z.frame_count = z.rec_first = z.rec_count = 0; z.next = SSE_NONE; r->run = z; }
        r->carry_len = carry; r->flags = flags; r->consumed = P.segs[gs].in_len;
    }
}

__device__ __forceinline__ void wait_tile(FSmem &S, uint32_t &phase, uint32_t total) {
    if (total == 0) return;
    while (!mbar_try_wait(&S.mbar, phase)) { }
    phase ^= 1u;
}

// A segment that does not fit a tile (carry + bytes): one CTA walks it window by window; a window starts at the line the
// previous one left unterminated. (S.bc[4..7]: input offset, input end, carry length, connection.) Returns the barrier phase.
__device__ __noinline__ uint32_t big_segment(const KParams &P, FSmem &S, uint32_t first, uint32_t phase) {
    const uint32_t tid = threadIdx.x, w = tid >> 5;
    uint32_t src = S.bc[4];
    const uint32_t in_end = S.bc[5];
    uint32_t cl = S.bc[6];
    const uint32_t conn = S.bc[7];
    uint32_t front = 0;                   // bytes of the first loaded vector that belong to an earlier line
    for (;;) {
        const uint32_t Aw = (cl + 15u) & ~15u;
        const uint32_t room = TILE - Aw;
        const uint32_t nbytes = min(in_end - src, room);
        const uint32_t ldw = (nbytes + 15u) & ~15u;
        const uint32_t tot = Aw + ldw;
        if (tid == 0) {
            FSeg &sg = S.seg[0];
            sg.data_off = cl ? Aw - cl : front; sg.in_pos = Aw; sg.end = Aw + nbytes; sg.in_delta = src - Aw;
        }
        fence_proxy_async();
        if (tid == 0) {
            mbar_expect_tx(&S.mbar, tot);
            if (Aw) bulk_g2s(S.tile, P.carry + (size_t)conn * P.carry_slot, Aw, &S.mbar);
            if (ldw) bulk_g2s(S.tile + Aw, P.in + src, ldw, &S.mbar);
        }
        __syncthreads();
        wait_tile(S, phase, tot);
        if (tid == 0) {
            const uint32_t d0 = cl ? Aw - cl : front;
            for (uint32_t q = 0; q < d0; q++) S.tile[q] = 0;
            if (!cl) for (uint32_t q = Aw; q < Aw + front; q++) S.tile[q] = 0;
            for (uint32_t q = Aw + nbytes; q < tot; q++) S.tile[q] = 0;
        }
        __syncthreads();
        process_window(P, S, first, 1, tot);
        __syncthreads();
        const uint32_t st = S.seg[0].state;
        const bool last = src + nbytes >= in_end;
        if ((st & (FS_TERM | FS_DEAD)) || last) break;
        if (tid == 0) S.bc[8] = tail_start(S, S.seg[0].data_off, S.seg[0].end);
        __syncthreads();
        const uint32_t ts = S.bc[8];
        if (ts == S.seg[0].data_off) {        // a whole window without '\n': the line is longer than carry_slot_bytes can be
            if (tid == 0) S.seg[0].state |= FS_DEAD;
            __syncthreads();
            break;
        }
        const uint32_t X = ts + S.seg[0].in_delta;    // input offset of the unterminated line (ts >= in_pos here)
        __syncthreads();
        src = X & ~15u; front = X & 15u; cl = 0;
    }
    if (w == 0) finish_segment(P, S, first, 0);
    __syncthreads();
    return phase;
}

__global__ void __launch_bounds__(F_THREADS, F_CTAS_PER_SM)
sse_fused_kernel(const __grid_constant__ KParams P, const FTables *__restrict__ gT) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    FSmem &S = *reinterpret_cast<FSmem *>(smem_raw);
    const uint32_t tid = threadIdx.x, lane = tid & 31u, w = tid >> 5;
    {
        const uint32_t *src = reinterpret_cast<const uint32_t *>(gT);
        uint32_t *dst = reinterpret_cast<uint32_t *>(&S.T);
        for (int i = tid; i < (int)(sizeof(FTables) / 4); i += F_THREADS) dst[i] = src[i];
    }
    if (tid == 0) { mbar_init(&S.mbar, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); S.rec_busy = 0; S.build_lock = 0; }
    if (tid < W_STRUCT + 8) S.thead[tid] = 0;
    // the templates learnt by earlier launches (a cache: results never depend on what it holds)
    uint32_t t_loaded = 1;
    if (P.tcache) {
        t_loaded = min(max(P.tcache[0], 1u), (uint32_t)TS_WORDS);
        if (t_loaded > 1u) {
            for (uint32_t i = tid; i < (uint32_t)W_STRUCT + 8u; i += F_THREADS) S.thead[i] = P.tcache[1u + i];
            for (uint32_t i = tid; i < t_loaded; i += F_THREADS) S.tstore[i] = P.tcache[257u + i];
        }
    }
    __syncthreads();
    if (tid == 0) S.ts_used = t_loaded;
    __syncthreads();
    uint32_t phase = 0;
    const uint32_t n_tiles = min(P.ctr->n_tiles, P.cap_tiles);

    if (tid == 0) S.bc[0] = atomicAdd(&P.ctr->ticket, 1u);
    __syncthreads();
    uint32_t t_next = S.bc[0];
    for (;;) {
        const uint32_t t = t_next;
        if (t >= n_tiles) break;
        __syncthreads();
        if (tid == 0) S.bc[0] = atomicAdd(&P.ctr->ticket, 1u);       // tickets are taken one tile ahead ...
        __syncthreads();
        t_next = S.bc[0];
        if (t_next < n_tiles) {                                         // ... so that the next tile's bytes are on their way to L2
            const uint2 tn = P.tiles[t_next];
            if (tid < tn.y) {
                const sse_seg nx = P.segs[tn.x + tid];
                if (nx.in_len) bulk_prefetch_l2(P.in + nx.in_off, (nx.in_len + 15u) & ~15u);
            }
        }
        const uint2 td = P.tiles[t];
        const uint32_t first = td.x, nseg = td.y;

        // ---------------- layout of the tile: [carry, right-aligned to 16][segment bytes, padded to 16] per segment
        uint32_t size = 0, A = 0, ld = 0, clen = 0;
        sse_seg sd; sd.conn = 0; sd.in_off = 0; sd.in_len = 0; sd.mode = 0;
        bool skip = false, skip_dead = false;
        if (tid < nseg) {
            sd = P.segs[first + tid];
            const ConnState cs = P.conns[sd.conn];
            skip = (cs.flags & (CONN_FINISHED | CONN_DEAD)) != 0; skip_dead = (cs.flags & CONN_DEAD) != 0;
            clen = cs.carry_len;
            if (!skip) { A = (clen + 15u) & ~15u; ld = (sd.in_len + 15u) & ~15u; size = A + ld; }
        }
        uint32_t total;
        const uint32_t reg = block_scan1(S, size, total);
        const bool big = total > TILE;            // only a single-segment tile can exceed the tile (plan kernel)
        if (tid < nseg) {
            FSeg &sg = S.seg[tid];
            sg.conn = sd.conn; sg.mode = sd.mode; sg.state = skip ? (FS_SKIP | (skip_dead ? FS_SKIP_DEAD : 0u)) : 0u;
            sg.data_off = reg + A - (skip ? 0u : clen); sg.in_pos = reg + A; sg.end = reg + A + (skip ? 0u : sd.in_len);
            sg.in_delta = sd.in_off - (reg + A);
            sg.nruns = 0; sg.last_run = SSE_NONE; sg.old_carry = clen;
            sg.term = sg.dead = SSE_NONE; sg.rf0 = sg.rr0 = SSE_NONE; sg.fcnt = sg.rcnt = 0;
        }
        if (!big) {
            if (total) {
                fence_proxy_async();
                if (tid == 0) mbar_expect_tx(&S.mbar, total);
                __syncthreads();
                if (tid < nseg && !skip) {
                    if (A) bulk_g2s(S.tile + reg, P.carry + (size_t)sd.conn * P.carry_slot, A, &S.mbar);
                    if (ld) bulk_g2s(S.tile + reg + A, P.in + sd.in_off, ld, &S.mbar);
                }
                wait_tile(S, phase, total);
                if (tid < nseg && !skip) {       // no stray '\n' in the alignment pads
                    for (uint32_t q = reg; q < reg + A - clen; q++) S.tile[q] = 0;
                    for (uint32_t q = reg + A + sd.in_len; q < reg + A + ld; q++) S.tile[q] = 0;
                }
            }
            __syncthreads();
            if (total) process_window(P, S, first, nseg, total);
            __syncthreads();
            for (uint32_t i = w; i < nseg; i += F_WARPS) finish_segment(P, S, first, i);
            __syncthreads();
            continue;
        }

        // ---------------- a segment larger than the tile: windows, restarting at the unterminated line
        __syncthreads();
        if (tid == 0) { S.bc[4] = sd.in_off; S.bc[5] = sd.in_off + sd.in_len; S.bc[6] = clen; S.bc[7] = sd.conn; }
        __syncthreads();
        phase = big_segment(P, S, first, phase);
    }
    // one CTA hands what it has learnt to the next launch (all CTAs see the same kinds of lines)
    if (P.tcache && blockIdx.x == 0) {
        __syncthreads();
        const uint32_t used = min(S.ts_used, (uint32_t)TS_WORDS);
        if (used > t_loaded) {
            for (uint32_t i = tid; i < used; i += F_THREADS) P.tcache[257u + i] = S.tstore[i];
            for (uint32_t i = tid; i < (uint32_t)W_STRUCT + 8u; i += F_THREADS) P.tcache[1u + i] = S.thead[i];
            __threadfence();
            __syncthreads();
            if (tid == 0) P.tcache[0] = used;
        }
    }
}

// ---------------------------------------------------------------- plan kernel: pack consecutive segments into tiles
// One warp per PLAN_GROUP segments, greedy: a tile closes when the next segment's region (carry + bytes, 16-byte padded)
// does not fit, or at MAX_TSEGS segments. A segment larger than a tile gets a tile of its own (windowed by the CTA).
__global__ void __launch_bounds__(128) sse_plan_kernel(const KParams P) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t g = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const uint32_t g0 = g * PLAN_GROUP;
    if (g0 >= P.n_segs) return;
    const uint32_t g1 = min(g0 + PLAN_GROUP, P.n_segs);
    uint32_t cur_first = g0, acc = 0, cnt = 0;
    auto emit = [&](uint32_t first, uint32_t n) {
        if (n == 0) return;
        if (lane == 0) {
            const uint32_t idx = atomicAdd(&P.ctr->n_tiles, 1u);
            if (idx < P.cap_tiles) P.tiles[idx] = make_uint2(first, n);
        }
    };
    for (uint32_t base = g0; base < g1; base += 32) {
        const uint32_t i = base + lane;
        uint32_t size = 0;
        if (i < g1) {
            const sse_seg sd = P.segs[i];
            const ConnState cs = P.conns[sd.conn];
            if (!(cs.flags & (CONN_FINISHED | CONN_DEAD))) size = ((cs.carry_len + 15u) & ~15u) + ((sd.in_len + 15u) & ~15u);
        }
        uint32_t incl = size;
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t x = __shfl_up_sync(FULL, incl, d); if ((int)lane >= d) incl += x; }
        uint32_t done = 0;                         // lanes [0, done) of this batch are placed
        const uint32_t nvalid = min(32u, g1 - base);
        while (done < nvalid) {
            const uint32_t before = done ? __shfl_sync(FULL, incl, (int)done - 1) : 0u;
            const bool fits = lane >= done && lane < nvalid && (acc + incl - before <= TILE) && (cnt + (lane - done) + 1u <= (uint32_t)MAX_TSEGS);
            const unsigned fm = __ballot_sync(FULL, fits);
            // lanes from `done` upward that fit form a prefix (sizes are non-negative)
            const unsigned want = (nvalid == 32u ? 0xFFFFFFFFu : ((1u << nvalid) - 1u)) & (0xFFFFFFFFu << done);
            const unsigned miss = want & ~fm;
            const uint32_t stop = miss ? (uint32_t)__ffs(miss) - 1u : nvalid;    // first lane that does not fit
            const uint32_t upto = stop ? __shfl_sync(FULL, incl, (int)stop - 1) : 0u;
            acc += (stop > done) ? upto - before : 0u; cnt += stop - done; done = stop;
            if (done < nvalid) {
                if (cnt == 0) {                   // a segment that is larger than a whole tile
                    emit(base + done, 1); done++; cur_first = base + done; acc = 0; cnt = 0;
                } else { emit(cur_first, cnt); cur_first = base + done; acc = 0; cnt = 0; }
            }
        }
    }
    emit(cur_first, cnt);
}

} // namespace

int sse_fused_prepare(const DfaTables &D, void *image) {
    FTables &T = *static_cast<FTables *>(image);
    memset(&T, 0, sizeof T);
    memcpy(T.clssym, D.clssym, sizeof T.clssym);
    memcpy(T.tr, D.tr, NST * NCLS);
    memcpy(T.field, D.field, sizeof T.field);
    // the struct-tag names only: build_tables gives them the first ids, and every one of them names a field
    int n_names = 0;
    for (int id = 0; id < NNAMES; id++)
        for (int node = 0; node < N_NODES; node++)
            if (D.field[node * NNAMES + id] & FIELD_VALID) n_names = id + 1;
    for (int i = 0; i < n_names; i++) { memcpy(T.name[i].w, D.nword[i], sizeof T.name[i].w); T.name[i].len = D.nlen[i]; }
    for (int id = 0; id < NNAMES; id++) {
        const uint32_t v = D.finmap[id];
        if (v == 0xFFu) continue;
        if (v < 1u || v > (uint32_t)N_FIN || D.nlen[id] > sizeof T.fin[0].w) return (int)cudaErrorInvalidValue;
        FFin &F = T.fin[v - 1];
        memcpy(F.w, D.nword[id], sizeof F.w); F.len = D.nlen[id]; F.val = (uint8_t)v;
    }
    // perfect hash: the first odd multiplier under which the names fall into distinct slots
    uint32_t mul = 0x9E3779B1u;
    for (int tries = 0; tries < 100000; tries++, mul += 0x632BE5ABu * 2u) {
        uint8_t used[1 << HASH_BITS];
        memset(used, 0xFF, sizeof used);
        bool ok = true;
        for (int i = 0; i < n_names && ok; i++) {
            const uint32_t h = ((T.name[i].w[0] | 0x20202020u) * mul + T.name[i].len * 0x9E3779B1u) >> (32 - HASH_BITS);
            if (used[h] != 0xFF) ok = false; else used[h] = (uint8_t)i;
        }
        if (ok) { memcpy(T.hash, used, sizeof used); T.hash_mul = mul; break; }
    }
    if (!T.hash_mul) return (int)cudaErrorInvalidValue;
    return (int)cudaFuncSetAttribute(sse_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FSmem));
}

uint32_t sse_fused_max_line(void) { return TILE - 32u; }
uint32_t sse_fused_tables_bytes(void) { return sizeof(FTables); }
uint32_t sse_fused_tcache_words(void) { return 8192u; }   // (both engines' layouts fit)

int sse_launch_fused(const KParams &p, void *stream, LaunchState &ls) {
    const uint32_t groups = (p.n_segs + PLAN_GROUP - 1) / PLAN_GROUP;
    sse_plan_kernel<<<(groups + 3) / 4, 128, 0, (cudaStream_t)stream>>>(p);
    ls.launches++;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return (int)e;
    // persistent: the resident CTAs pull tiles by ticket
    sse_fused_kernel<<<ls.sm_count * F_CTAS_PER_SM, F_THREADS, sizeof(FSmem), (cudaStream_t)stream>>>(p, static_cast<const FTables *>(ls.tables));
    ls.launches++;
    return (int)cudaGetLastError();
}
