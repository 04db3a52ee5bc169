// sse_common.cuh -- device helpers shared by the stream kernels: schema of the decoded document, strings.TrimSpace,
// encoding/json pieces (number checks, unquote, key folding, the lane's unquote queue), run bookkeeping, the long-line
// path and the line pool. Included by every kernel source.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "sse_device.cuh"

namespace {

#ifndef SSE_V1_WARPS
#define SSE_V1_WARPS 12
#endif
constexpr int WARPS_PER_CTA = SSE_V1_WARPS;
constexpr int BUF = 8192;          // line window per warp (bytes, multiple of 16)
constexpr int LT_MAX = 64;         // lines per round
constexpr int DONE_MAX = 16;
constexpr unsigned FULL = 0xFFFFFFFFu;

// ---------------------------------------------------------------- schema of the decoded document
// providers/types/common_types.go:271-297 (tool-call chunk, function), :300-346 (choice, delta),
// :349-371 (logprobs), :384-393 (usage), :451-478 (stream response), :686-698 + :835-862 (extra_content)
enum : uint8_t { TY_SKIP, TY_STR, TY_PSTR, TY_INT, TY_F32, TY_STRUCT, TY_PSTRUCT, TY_SLICE, TY_PSLICE,
                 TY_GOOGLE, TY_ROOT, TY_TS };
enum : uint8_t { N_NONE = 0, N_ROOT, N_CHOICE, N_DELTA, N_TC, N_FUNC, N_EXTRA, N_USAGE, N_LOGPROBS, N_TOKLP,
                 N_TOPLP, N_GOOGLE, A_CHOICES, A_TOOLCALLS, A_TOKLP, A_TOPLP, A_INTS, N_COUNT };
enum : uint8_t { TG_NONE, TG_CHOICES, TG_USAGE, TG_PROMPT, TG_COMPLETION, TG_TOTAL, TG_FINISH, TG_CONTENT,
                 TG_TOOLCALLS, TG_TC_ID, TG_TC_TYPE, TG_TC_INDEX, TG_TC_FUNCTION, TG_NAME, TG_ARGS };

struct FieldDef { uint8_t len, ty, sub, tgt; char name[20]; };
constexpr int N_FIELDS = 39;
struct alignas(16) Schema { FieldDef f[N_FIELDS]; uint8_t first[N_COUNT]; uint8_t cnt[N_COUNT]; uint8_t pad[2]; };

// The one declaration of the schema: in constant memory for the slow key path (escaped, non-ASCII or case-folded keys:
// match_field), and constexpr, so that the host builds the decode tables from a compile-time copy of it (sse_build_tables).
#define FD(nm, ty, sub, tgt) { (uint8_t)(sizeof(nm) - 1), ty, sub, tgt, nm }
constexpr __constant__ Schema c_schema = {
    {
        /* N_ROOT (0..7) */
        FD("choices", TY_SLICE, A_CHOICES, TG_CHOICES), FD("created", TY_INT, 0, 0), FD("id", TY_STR, 0, 0),
        FD("model", TY_STR, 0, 0), FD("object", TY_STR, 0, 0), FD("reasoning_format", TY_PSTR, 0, 0),
        FD("system_fingerprint", TY_PSTR, 0, 0), FD("usage", TY_PSTRUCT, N_USAGE, TG_USAGE),
        /* N_CHOICE (8..11) */
        FD("delta", TY_STRUCT, N_DELTA, 0), FD("finish_reason", TY_STR, 0, TG_FINISH), FD("index", TY_INT, 0, 0),
        FD("logprobs", TY_PSTRUCT, N_LOGPROBS, 0),
        /* N_DELTA (12..17) */
        FD("content", TY_STR, 0, TG_CONTENT), FD("reasoning", TY_PSTR, 0, 0), FD("reasoning_content", TY_PSTR, 0, 0),
        FD("refusal", TY_PSTR, 0, 0), FD("role", TY_STR, 0, 0), FD("tool_calls", TY_PSLICE, A_TOOLCALLS, TG_TOOLCALLS),
        /* N_TC (18..22) */
        FD("extra_content", TY_PSTRUCT, N_EXTRA, 0), FD("function", TY_PSTRUCT, N_FUNC, TG_TC_FUNCTION),
        FD("id", TY_PSTR, 0, TG_TC_ID), FD("index", TY_INT, 0, TG_TC_INDEX), FD("type", TY_PSTR, 0, TG_TC_TYPE),
        /* N_FUNC (23..24) */
        FD("arguments", TY_STR, 0, TG_ARGS), FD("name", TY_STR, 0, TG_NAME),
        /* N_EXTRA (25) */
        FD("google", TY_GOOGLE, N_GOOGLE, 0),
        /* N_USAGE (26..28) */
        FD("completion_tokens", TY_INT, 0, TG_COMPLETION), FD("prompt_tokens", TY_INT, 0, TG_PROMPT),
        FD("total_tokens", TY_INT, 0, TG_TOTAL),
        /* N_LOGPROBS (29..30) */
        FD("content", TY_SLICE, A_TOKLP, 0), FD("refusal", TY_SLICE, A_TOKLP, 0),
        /* N_TOKLP (31..34) */
        FD("bytes", TY_SLICE, A_INTS, 0), FD("logprob", TY_F32, 0, 0), FD("token", TY_STR, 0, 0),
        FD("top_logprobs", TY_SLICE, A_TOPLP, 0),
        /* N_TOPLP (35..37) */
        FD("bytes", TY_SLICE, A_INTS, 0), FD("logprob", TY_F32, 0, 0), FD("token", TY_STR, 0, 0),
        /* N_GOOGLE (38): exact (case-sensitive) map key, common_types.go:842 */
        FD("thought_signature", TY_TS, 0, 0),
    },
    /* first */ { 0, 0, 8, 12, 18, 23, 25, 26, 29, 31, 35, 38, 0, 0, 0, 0, 0 },
    /* cnt   */ { 0, 8, 4, 6, 5, 2, 1, 3, 2, 4, 3, 1, 0, 0, 0, 0, 0 },
    { 0, 0 },
};
#undef FD

struct LineEnt {
    uint16_t nl;        // window position of the terminating '\n'
    uint16_t src_s;     // first source byte of the frame (mode P: line start; mode R: start of "data: ")
    uint16_t pay_s;     // payload handed to the decoder [pay_s, pay_e)
    uint16_t pay_e;
    uint16_t flen;      // emitted frame length (0: nothing emitted)
    uint8_t  kind;      // K_*
    uint16_t rel;       // index among this round's work items
    uint16_t zc;        // 1: the frame's bytes stand in the input arena as they are (no copy; offsets are input offsets)
    uint16_t clen;      // bytes this line occupies in the out arena (frame, or the payload of a swallowed line that is decoded)
};
enum : uint8_t { K_DROP = 0, K_EMIT = 1, K_DONE = 2, K_DONE_EXACT = 3 };

struct WarpSmem {
    alignas(16) uint8_t buf[BUF + 16];
    LineEnt lt[LT_MAX];
    uint16_t done_pos[DONE_MAX];
    uint32_t done_cnt;
    uint32_t pad[3];
};

struct CtaSmem {
    WarpSmem w[WARPS_PER_CTA];
};

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }
__device__ __forceinline__ void prefetch_l2(const uint8_t *p) { asm volatile("prefetch.global.L2 [%0];" :: "l"(p)); }

// 0x80 in every byte of x that is zero (exact)
__device__ __forceinline__ uint32_t zero_bytes(uint32_t x) { return ~((((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x)) & 0x80808080u; }
// bits 7, 15, 23, 31 -> bits 0..3
__device__ __forceinline__ uint32_t gather4(uint32_t z) { return (((z >> 7) * 0x00204081u) >> 21) & 0xFu; }
// 4-bit mask of the bytes of w equal to the byte replicated in pat
__device__ __forceinline__ uint32_t eqmask4(uint32_t w, uint32_t pat) { return gather4(zero_bytes(w ^ pat)); }
// 16-bit mask of the positions in v where '[' is followed by 'D' (position 15 cannot see its successor: any '[' there counts).
// A cheap superset of the places where "[DONE]" can start; 0 for almost every chunk of a JSON stream.
__device__ __forceinline__ uint32_t done_candidates16(const uint4 &v) {
    const uint32_t b0 = zero_bytes(v.x ^ 0x5B5B5B5Bu), b1 = zero_bytes(v.y ^ 0x5B5B5B5Bu), b2 = zero_bytes(v.z ^ 0x5B5B5B5Bu), b3 = zero_bytes(v.w ^ 0x5B5B5B5Bu);
    if ((b0 | b1 | b2 | b3) == 0) return 0;
    const uint32_t d0 = zero_bytes(v.x ^ 0x44444444u), d1 = zero_bytes(v.y ^ 0x44444444u), d2 = zero_bytes(v.z ^ 0x44444444u), d3 = zero_bytes(v.w ^ 0x44444444u);
    const uint32_t c0 = b0 & ((d0 >> 8) | (d1 << 24)), c1 = b1 & ((d1 >> 8) | (d2 << 24)), c2 = b2 & ((d2 >> 8) | (d3 << 24));
    const uint32_t c3 = b3 & ((d3 >> 8) | 0x80000000u);
    if ((c0 | c1 | c2 | c3) == 0) return 0;
    return gather4(c0) | (gather4(c1) << 4) | (gather4(c2) << 8) | (gather4(c3) << 12);
}
__device__ __forceinline__ uint32_t eqmask16(const uint4 &v, uint32_t pat) {
    return eqmask4(v.x, pat) | (eqmask4(v.y, pat) << 4) | (eqmask4(v.z, pat) << 8) | (eqmask4(v.w, pat) << 12);
}

// 0x80 in every byte of w that is '"', '\\', < 0x20 or >= 0x80 (exact for the lowest flagged byte only)
__device__ __forceinline__ uint32_t special_mask4(uint32_t w) {
    const uint32_t q = w ^ 0x22222222u, b = w ^ 0x5C5C5C5Cu;
    return (((q - 0x01010101u) & ~q) | ((b - 0x01010101u) & ~b) | ((w - 0x20202020u) & ~w) | w) & 0x80808080u;
}
// ---------------------------------------------------------------- strings.TrimSpace pieces
// unicode.IsSpace code points in UTF-8: ASCII \t\n\v\f\r ' ', U+0085, U+00A0, U+1680, U+2000-200A,
// U+2028, U+2029, U+202F, U+205F, U+3000 (Go strings.TrimSpace / utf8.DecodeRune semantics).
__device__ __forceinline__ int space_prefix(const uint8_t *s, int n) {
    if (n <= 0) return 0;
    uint32_t c = s[0];
    if (c == ' ' || (c >= 0x09 && c <= 0x0D)) return 1;
    if (c < 0x80) return 0;
    if (n >= 2 && c == 0xC2 && (s[1] == 0x85 || s[1] == 0xA0)) return 2;
    if (n >= 3) {
        uint32_t c1 = s[1], c2 = s[2];
        if (c == 0xE1 && c1 == 0x9A && c2 == 0x80) return 3;
        if (c == 0xE2 && c1 == 0x80 && ((c2 >= 0x80 && c2 <= 0x8A) || c2 == 0xA8 || c2 == 0xA9 || c2 == 0xAF)) return 3;
        if (c == 0xE2 && c1 == 0x81 && c2 == 0x9F) return 3;
        if (c == 0xE3 && c1 == 0x80 && c2 == 0x80) return 3;
    }
    return 0;
}
__device__ __forceinline__ int space_suffix(const uint8_t *s, int n) {
    if (n <= 0) return 0;
    uint32_t c = s[n - 1];
    if (c == ' ' || (c >= 0x09 && c <= 0x0D)) return 1;
    if (c < 0x80) return 0;
    if (n >= 2 && space_prefix(s + n - 2, 2) == 2) return 2;
    if (n >= 3 && space_prefix(s + n - 3, 3) == 3) return 3;
    return 0;
}
__device__ __forceinline__ void trim_space(const uint8_t *s, int &a, int &b) {
    int k;
    while (a < b && (k = space_prefix(s + a, b - a)) != 0) a += k;
    while (b > a && (k = space_suffix(s + a, b - a)) != 0) b -= k;
}
__device__ __forceinline__ bool is_data_prefix(const uint8_t *s, int n) {
    return n >= 6 && s[0] == 'd' && s[1] == 'a' && s[2] == 't' && s[3] == 'a' && s[4] == ':' && s[5] == ' ';
}
__device__ __forceinline__ bool is_done_at(const uint8_t *s) {   // "[DONE]"
    return s[0] == '[' && s[1] == 'D' && s[2] == 'O' && s[3] == 'N' && s[4] == 'E' && s[5] == ']';
}

// ---------------------------------------------------------------- encoding/json pieces
// utf8.DecodeRune acceptance: size of a valid sequence at s (n bytes available) or 0
__device__ __forceinline__ int utf8_valid_len(const uint8_t *s, int n) {
    uint32_t c = s[0];
    if (c < 0x80) return 1;
    if (c >= 0xC2 && c <= 0xDF) return (n >= 2 && (s[1] & 0xC0) == 0x80) ? 2 : 0;
    if (c >= 0xE0 && c <= 0xEF) {
        uint32_t lo = (c == 0xE0) ? 0xA0 : 0x80, hi = (c == 0xED) ? 0x9F : 0xBF;
        return (n >= 3 && s[1] >= lo && s[1] <= hi && (s[2] & 0xC0) == 0x80) ? 3 : 0;
    }
    if (c >= 0xF0 && c <= 0xF4) {
        uint32_t lo = (c == 0xF0) ? 0x90 : 0x80, hi = (c == 0xF4) ? 0x8F : 0xBF;
        return (n >= 4 && s[1] >= lo && s[1] <= hi && (s[2] & 0xC0) == 0x80 && (s[3] & 0xC0) == 0x80) ? 4 : 0;
    }
    return 0;
}
__device__ __forceinline__ int hexval(uint32_t c) {
    if (c >= '0' && c <= '9') return (int)c - '0';
    c |= 0x20;
    if (c >= 'a' && c <= 'f') return (int)c - 'a' + 10;
    return -1;
}
__device__ __forceinline__ int hex4(const uint8_t *s) {
    int a = hexval(s[0]), b = hexval(s[1]), c = hexval(s[2]), d = hexval(s[3]);
    if ((a | b | c | d) < 0) return -1;
    return (a << 12) | (b << 8) | (c << 4) | d;
}
// strconv.ParseInt(s, 10, 64) on an integer literal [s, e)
__device__ __noinline__ bool parse_i64(const uint8_t *sm, int s, int e, int64_t &out) {
    bool neg = false;
    if (sm[s] == '-') { neg = true; s++; }
    unsigned long long v = 0;
    for (; s < e; s++) {
        unsigned long long d = (unsigned long long)(sm[s] - '0');
        if (v > (0xFFFFFFFFFFFFFFFFull - d) / 10ull) return false;
        v = v * 10ull + d;
    }
    if (neg) { if (v > 0x8000000000000000ull) return false; out = (int64_t)(0ull - v); }
    else { if (v > 0x7FFFFFFFFFFFFFFFull) return false; out = (int64_t)v; }
    return true;
}
// strconv.ParseFloat(s, 32) range error: |x| >= 2^128 - 2^103 (exact decimal comparison)
__device__ __noinline__ bool f32_overflows(const uint8_t *sm, int s, int e) {
    const char *H = "340282356779733661637539395458142568448";   // 39 digits
    if (s < e && sm[s] == '-') s++;
    long long dexp = 0;
    bool seen = false;
    int cmp = 0, nd = 0;   // cmp: sign of (digits so far) vs H prefix
    auto feed = [&](uint32_t c) {
        if (nd < 39 && cmp == 0) { char h = H[nd]; cmp = ((char)c > h) - ((char)c < h); }
        nd++;
    };
    int i = s;
    for (; i < e && (uint32_t)(sm[i] - '0') <= 9u; i++) {
        if (sm[i] != '0' || seen) { seen = true; feed(sm[i]); dexp++; }
    }
    if (i < e && sm[i] == '.') {
        for (i++; i < e && (uint32_t)(sm[i] - '0') <= 9u; i++) {
            if (sm[i] != '0' || seen) { seen = true; feed(sm[i]); } else dexp--;
        }
    }
    if (!seen) return false;
    if (i < e && (sm[i] == 'e' || sm[i] == 'E')) {
        bool eneg = false; long long ex = 0;
        i++;
        if (i < e && (sm[i] == '+' || sm[i] == '-')) { eneg = sm[i] == '-'; i++; }
        for (; i < e; i++) if (ex < 100000000) ex = ex * 10 + (sm[i] - '0');
        dexp += eneg ? -ex : ex;
    }
    if (dexp > 39) return true;
    if (dexp < 39) return false;
    if (cmp != 0) return cmp > 0;
    // all compared digits equal: remaining H digits vs implicit zeros
    for (int k = nd; k < 39; k++) if (H[k] != '0') return false;
    return true;   // >= H
}
__device__ __forceinline__ uint32_t put_rune(uint8_t *dst, uint32_t n, uint32_t r) {
    if (r < 0x80) { if (dst) dst[n] = (uint8_t)r; return 1; }
    if (r < 0x800) { if (dst) { dst[n] = 0xC0 | (r >> 6); dst[n + 1] = 0x80 | (r & 0x3F); } return 2; }
    if (r < 0x10000) {
        if (dst) { dst[n] = 0xE0 | (r >> 12); dst[n + 1] = 0x80 | ((r >> 6) & 0x3F); dst[n + 2] = 0x80 | (r & 0x3F); }
        return 3;
    }
    if (dst) { dst[n] = 0xF0 | (r >> 18); dst[n + 1] = 0x80 | ((r >> 12) & 0x3F); dst[n + 2] = 0x80 | ((r >> 6) & 0x3F); dst[n + 3] = 0x80 | (r & 0x3F); }
    return 4;
}
// decode.go unquoteBytes over a validated string body [s, e). dst == nullptr: count only. cap: stop at cap bytes.
__device__ __noinline__ uint32_t json_unquote(const uint8_t *sm, int s, int e, uint8_t *dst, uint32_t cap) {
    uint32_t n = 0;
    int i = s;
    while (i < e && n + 4 <= cap) {
        uint32_t c = sm[i];
        if (c == '\\') {
            uint32_t esc = sm[i + 1];
            i += 2;
            uint32_t r;
            switch (esc) {
            case 'b': r = 8; break;
            case 'f': r = 12; break;
            case 'n': r = 10; break;
            case 'r': r = 13; break;
            case 't': r = 9; break;
            case 'u': {
                r = (uint32_t)hex4(sm + i);
                i += 4;
                if (r >= 0xD800 && r < 0xE000) {
                    int r1 = -1;
                    if (i + 6 <= e && sm[i] == '\\' && sm[i + 1] == 'u') r1 = hex4(sm + i + 2);
                    if (r < 0xDC00 && r1 >= 0xDC00 && r1 < 0xE000) { r = 0x10000 + ((r - 0xD800) << 10) + ((uint32_t)r1 - 0xDC00); i += 6; }
                    else r = 0xFFFD;
                }
                break;
            }
            default: r = esc; break;   // '"', '\\', '/'
            }
            n += put_rune(dst, n, r);
        } else if (c < 0x80) {
            if (dst) dst[n] = (uint8_t)c;
            n++; i++;
        } else {
            int k = utf8_valid_len(sm + i, e - i);
            if (k == 0) { n += put_rune(dst, n, 0xFFFD); i++; }
            else { if (dst) for (int q = 0; q < k; q++) dst[n + q] = sm[i + q]; n += k; i += k; }
        }
    }
    if (i < e) return cap + 1;   // did not fit
    return n;
}
// Single-pass unquote into a 4-byte aligned destination (text arena): same semantics as json_unquote, tight loop,
// bytes gathered into 32-bit stores. Returns the decoded length.
__device__ __noinline__ uint32_t json_unquote_write(const uint8_t *__restrict__ src, int s, int e, uint8_t *__restrict__ dst) {
    uint32_t n = 0, acc = 0;
    uint32_t *d32 = reinterpret_cast<uint32_t *>(dst);
    int i = s;
    auto put = [&](uint32_t c) {
        acc |= c << ((n & 3u) * 8u);
        if ((n & 3u) == 3u) { d32[n >> 2] = acc; acc = 0; }
        n++;
    };
    while (i < e) {
        uint32_t c = src[i];
        if (c != '\\' && c < 0x80) { put(c); i++; continue; }
        if (c == '\\') {
            uint32_t esc = src[i + 1];
            i += 2;
            uint32_t r;
            switch (esc) {
            case 'b': r = 8; break;
            case 'f': r = 12; break;
            case 'n': r = 10; break;
            case 'r': r = 13; break;
            case 't': r = 9; break;
            case 'u': {
                r = (uint32_t)hex4(src + i);
                i += 4;
                if (r >= 0xD800 && r < 0xE000) {
                    int r1 = -1;
                    if (i + 6 <= e && src[i] == '\\' && src[i + 1] == 'u') r1 = hex4(src + i + 2);
                    if (r < 0xDC00 && r1 >= 0xDC00 && r1 < 0xE000) { r = 0x10000 + ((r - 0xD800) << 10) + ((uint32_t)r1 - 0xDC00); i += 6; }
                    else r = 0xFFFD;
                }
                break;
            }
            default: r = esc; break;
            }
            if (r < 0x80) put(r);
            else if (r < 0x800) { put(0xC0 | (r >> 6)); put(0x80 | (r & 0x3F)); }
            else if (r < 0x10000) { put(0xE0 | (r >> 12)); put(0x80 | ((r >> 6) & 0x3F)); put(0x80 | (r & 0x3F)); }
            else { put(0xF0 | (r >> 18)); put(0x80 | ((r >> 12) & 0x3F)); put(0x80 | ((r >> 6) & 0x3F)); put(0x80 | (r & 0x3F)); }
        } else {
            int k = utf8_valid_len(src + i, e - i);
            if (k == 0) { put(0xEF); put(0xBF); put(0xBD); i++; }
            else { for (int q = 0; q < k; q++) put(src[i + q]); i += k; }
        }
    }
    if (n & 3u) d32[n >> 2] = acc;     // the allocation is padded to a multiple of 4
    return n;
}

// encoding/json foldName equality (Go >= 1.21): ASCII case-insensitive, U+212A == 'k', U+017F == 's'
__device__ __noinline__ bool key_eq(const uint8_t *k, int n, const char *name, int m, bool fold) {
    if (!fold) {
        if (n != m) return false;
        for (int i = 0; i < n; i++) if (k[i] != (uint8_t)name[i]) return false;
        return true;
    }
    int i = 0, q = 0;
    while (i < n) {
        uint32_t c = k[i];
        if (c < 0x80) { if (c >= 'A' && c <= 'Z') c += 32; i++; }
        else if (i + 1 < n && c == 0xC5 && k[i + 1] == 0xBF) { c = 's'; i += 2; }
        else if (i + 2 < n && c == 0xE2 && k[i + 1] == 0x84 && k[i + 2] == 0xAA) { c = 'k'; i += 3; }
        else return false;
        if (q >= m || c != (uint8_t)name[q]) return false;
        q++;
    }
    return q == m;
}
__device__ __noinline__ int match_field(const Schema &S, int node, const uint8_t *k, int n) {
    int first = S.first[node], cnt = S.cnt[node];
    bool fold = node != N_GOOGLE;
    for (int f = first; f < first + cnt; f++)
        if (key_eq(k, n, S.f[f].name, S.f[f].len, fold)) return f;
    return -1;
}
__device__ __noinline__ uint32_t classify_finish(const uint8_t *s, int n) {
    if (n == 0) return SSE_FIN_NONE;
    if (key_eq(s, n, "stop", 4, false)) return SSE_FIN_STOP;
    if (key_eq(s, n, "tool_calls", 10, false)) return SSE_FIN_TOOL_CALLS;
    if (key_eq(s, n, "length", 6, false)) return SSE_FIN_LENGTH;
    if (key_eq(s, n, "content_filter", 14, false)) return SSE_FIN_CONTENT_FILTER;
    if (key_eq(s, n, "function_call", 13, false)) return SSE_FIN_FUNCTION_CALL;
    return SSE_FIN_OTHER;
}

// ---------------------------------------------------------------- unquote queues
// Deferred unquote jobs of one lane: drained warp-cooperatively (warp_unquote) instead of byte-by-byte on one lane.
struct UnquoteJob { uint32_t s, e, dst, pad; uint32_t *patch; };
#ifndef SSE_MAX_JOBS
#define SSE_MAX_JOBS 1
#endif
constexpr int MAX_JOBS = SSE_MAX_JOBS;   // queue full: the lane unquotes the string itself (slow, exact)
struct LaneJobs { uint32_t n; uint32_t pad; UnquoteJob j[MAX_JOBS]; };
struct Span { uint32_t off, len; bool text; };

// Warp-cooperative unquote (same result as json_unquote_write): runs of plain bytes are copied 32 at a time, the byte that
// stops a run (escape or non-ASCII sequence) is handled by lane 0 with the exact decode.go rules.
__device__ __noinline__ void warp_unquote(const uint8_t *__restrict__ src, uint32_t s, uint32_t e, uint8_t *__restrict__ dst, uint32_t *patch) {
    const uint32_t lane = lane_id();
    uint32_t i = s, n = 0;
    while (i < e) {
        const uint32_t idx = i + lane;
        const uint32_t c = idx < e ? (uint32_t)src[idx] : 0x5Cu;
        const unsigned m = __ballot_sync(FULL, idx >= e || c == '\\' || c >= 0x80);
        const uint32_t run = m ? (uint32_t)(__ffs(m) - 1) : 32u;
        if (lane < run) dst[n + lane] = (uint8_t)c;
        n += run; i += run;
        if (i < e && run < 32u) {
            uint32_t ni = i, nn = n;
            if (lane == 0) {
                const uint32_t c0 = src[i];
                if (c0 == '\\') {
                    const uint32_t esc = src[i + 1];
                    ni = i + 2;
                    uint32_t r;
                    switch (esc) {
                    case 'b': r = 8; break;
                    case 'f': r = 12; break;
                    case 'n': r = 10; break;
                    case 'r': r = 13; break;
                    case 't': r = 9; break;
                    case 'u': {
                        r = (uint32_t)hex4(src + ni);
                        ni += 4;
                        if (r >= 0xD800 && r < 0xE000) {
                            int r1 = -1;
                            if (ni + 6 <= e && src[ni] == '\\' && src[ni + 1] == 'u') r1 = hex4(src + ni + 2);
                            if (r < 0xDC00 && r1 >= 0xDC00 && r1 < 0xE000) { r = 0x10000 + ((r - 0xD800) << 10) + ((uint32_t)r1 - 0xDC00); ni += 6; }
                            else r = 0xFFFD;
                        }
                        break;
                    }
                    default: r = esc; break;
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
    }
    if (lane == 0) *patch = n;
    __syncwarp();
}

// Warp-parallel unquote of a string body [s, e) the automaton accepted (escapes are well formed; the UTF-8 need not be): the
// same bytes as json_unquote_write, 32 source bytes per step, one per lane. What a byte is follows from facts local to it: a
// backslash starts an escape unless the run of backslashes before it has odd length (its parity is carried from step to step),
// and a byte is inside an earlier unit when an escape or a valid UTF-8 sequence that starts at most 11 bytes before it reaches
// over it (a max-scan of where the units end, carried from step to step). A byte nothing covers starts a unit: a plain byte, an
// escape (with its low surrogate when a high one is followed by one, else U+FFFD for a surrogate), a valid sequence (copied), or
// an invalid byte (U+FFFD). Output positions are a warp prefix sum of the units' lengths. The long-line kernel's (the decode kernel keeps
// warp_unquote above: its strings are short and mostly plain, and it is compiled as it was before the long-line stage).
__device__ __noinline__ void warp_unquote_parallel(const uint8_t *__restrict__ src, uint32_t s, uint32_t e, uint8_t *__restrict__ dst, uint32_t *patch) {
    const uint32_t lane = lane_id();
    uint32_t n = 0, cover = s, esc_in = 0;       // cover: no earlier unit reaches a byte at or after it; esc_in: a backslash escapes the step's first byte
    for (uint32_t b = s; b < e; b += 32u) {
        const uint32_t i = b + lane;
        const bool in = i < e;
        const uint32_t c = in ? (uint32_t)src[i] : 0u;
        const unsigned bsm = __ballot_sync(FULL, in && c == '\\');
        const unsigned him = __ballot_sync(FULL, in && c >= 0x80u);
        if (!(bsm | him | esc_in) && cover <= b) {       // plain ASCII: copied as it is
            if (in) dst[n + lane] = (uint8_t)c;
            n += min(32u, e - b);
            continue;
        }
        // backslashes right before this byte, and whether they leave it escaped
        const unsigned nz = ~bsm & ((1u << lane) - 1u);
        const bool escaped = nz ? (((lane - 1u - (31u - __clz(nz))) & 1u) != 0u) : (((lane + esc_in) & 1u) != 0u);
        const bool start_esc = in && c == '\\' && !escaped;
        uint32_t unit_end = 0, r = 0, k = 0;            // (candidate) unit [i, unit_end); r: rune of an escape; k: valid sequence length
        if (start_esc) {
            const uint32_t c1 = src[i + 1];
            unit_end = i + 2u;
            switch (c1) {
            case 'b': r = 8; break;
            case 'f': r = 12; break;
            case 'n': r = 10; break;
            case 'r': r = 13; break;
            case 't': r = 9; break;
            case 'u': {
                r = (uint32_t)hex4(src + i + 2u);
                unit_end = i + 6u;
                if (r >= 0xD800u && r < 0xE000u) {
                    int r1 = -1;
                    if (i + 12u <= e && src[i + 6u] == '\\' && src[i + 7u] == 'u') r1 = hex4(src + i + 8u);
                    if (r < 0xDC00u && r1 >= 0xDC00 && r1 < 0xE000) { r = 0x10000u + ((r - 0xD800u) << 10) + ((uint32_t)r1 - 0xDC00u); unit_end = i + 12u; }
                    else r = 0xFFFDu;
                }
                break;
            }
            default: r = c1; break;     // '"', '\\', '/'
            }
        } else if (in && c >= 0x80u) {
            k = (uint32_t)utf8_valid_len(src + i, (int)(e - i));
            if (k) unit_end = i + k;
        }
        uint32_t reach = unit_end;                       // inclusive max-scan: how far the units starting up to this lane reach
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t v = __shfl_up_sync(FULL, reach, d); if ((int)lane >= d) reach = max(reach, v); }
        uint32_t before = __shfl_up_sync(FULL, reach, 1);
        before = max(lane ? before : 0u, cover);
        const bool unit = in && before <= i;
        uint32_t len = 0;
        if (unit) len = start_esc ? (r < 0x80u ? 1u : r < 0x800u ? 2u : r < 0x10000u ? 3u : 4u) : c < 0x80u ? 1u : (k ? k : 3u);
        uint32_t incl = len;
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, d); if ((int)lane >= d) incl += v; }
        const uint32_t o = n + incl - len;
        if (unit) {
            if (start_esc) put_rune(dst, o, r);
            else if (c < 0x80u) dst[o] = (uint8_t)c;
            else if (k) { for (uint32_t q = 0; q < k; q++) dst[o + q] = src[i + q]; }
            else put_rune(dst, o, 0xFFFDu);
        }
        n += __shfl_sync(FULL, incl, 31);
        cover = max(cover, __shfl_sync(FULL, reach, 31));
        if (~bsm) esc_in = (uint32_t)__clz(~bsm) & 1u;      // the run of backslashes that ends the step (all 32: unchanged)
    }
    if (lane == 0) *patch = n;
    __syncwarp();
}

// ---------------------------------------------------------------- warp-cooperative helpers
// copy n bytes global -> shared so that they END at smem offset `end_off` (byte granularity)
__device__ void copy_g2s_bytes(uint8_t *sm_dst, const uint8_t *g_src, int n) {
    for (int i = lane_id(); i < n; i += 32) sm_dst[i] = g_src[i];
}
__device__ void copy_s2g_bytes(uint8_t *g_dst, const uint8_t *sm_src, int n) {
    for (int i = lane_id(); i < n; i += 32) g_dst[i] = sm_src[i];
}
__device__ void copy_g2g_bytes(uint8_t *g_dst, const uint8_t *g_src, int n) {
    for (int i = lane_id(); i < n; i += 32) g_dst[i] = g_src[i];
}

// Warp-cooperative copy of n bytes shared -> global with arbitrary alignment on both sides: the destination is written
// as aligned 16-byte vectors, the source is read as aligned words and funnel-shifted into place.
__device__ __forceinline__ void copy_s2g_vec(uint8_t *__restrict__ g_dst, const uint8_t *__restrict__ sm_src, int n) {
    const int lane = (int)lane_id();
    if (n < 48) { for (int i = lane; i < n; i += 32) g_dst[i] = sm_src[i]; return; }
    const int head = (int)((16u - ((uint32_t)(uintptr_t)g_dst & 15u)) & 15u);
    if (lane < head) g_dst[lane] = sm_src[lane];
    const int nch = (n - head) >> 4;
    const uint8_t *sb = sm_src + head;
    const uint32_t sh = ((uint32_t)(uintptr_t)sb & 3u) * 8u;
    const uint32_t *sw = reinterpret_cast<const uint32_t *>((uintptr_t)sb & ~(uintptr_t)3);
    uint4 *gd = reinterpret_cast<uint4 *>(g_dst + head);
    for (int c = lane; c < nch; c += 32) {
        const uint32_t *w = sw + c * 4;
        uint32_t a0 = w[0], a1 = w[1], a2 = w[2], a3 = w[3], a4 = w[4];
        uint4 v;
        v.x = __funnelshift_r(a0, a1, sh); v.y = __funnelshift_r(a1, a2, sh);
        v.z = __funnelshift_r(a2, a3, sh); v.w = __funnelshift_r(a3, a4, sh);
        gd[c] = v;
    }
    const int done = head + (nch << 4);
    if (lane < n - done) g_dst[done + lane] = sm_src[done + lane];
}

struct Resv { uint32_t ob, qb, fb, rb; };   // SSE_FLAG_DEFER: a long line's reservation (out offset, work item, frame, record)

struct RunChain {           // lane-uniform bookkeeping of a segment's result runs
    sse_run first;
    bool have_first;
    uint32_t last_idx;      // index in runs[] of the last appended run (SSE_NONE: the inline one)
    uint32_t pre;           // SSE_FLAG_DEFER: runs[] entry reserved for the next appended run (SSE_NONE: allocate it then)
    Resv rv;                // SSE_FLAG_DEFER: where the long line being completed puts its results (reserve_long)
};

__device__ __noinline__ void append_run(const KParams &P, RunChain &rc, uint32_t ff, uint32_t fc, uint32_t rf, uint32_t rcnt) {
    if (fc == 0 && rcnt == 0) return;
    if (!rc.have_first) {
        rc.first.frame_first = ff; rc.first.frame_count = fc; rc.first.rec_first = rf; rc.first.rec_count = rcnt;
        rc.first.next = SSE_NONE; rc.have_first = true; rc.last_idx = SSE_NONE;
        return;
    }
    uint32_t idx = rc.pre;
    rc.pre = SSE_NONE;
    if (idx == SSE_NONE) {
        if (lane_id() == 0) idx = atomicAdd(&P.ctr->n_runs, 1u);
        idx = __shfl_sync(FULL, idx, 0);
        if (idx >= P.cap_runs) { if (lane_id() == 0) sse_overflow(P.ctr, SSE_OVF_RUNS); return; }
    }
    if (lane_id() == 0) {
        sse_run r; r.frame_first = ff; r.frame_count = fc; r.rec_first = rf; r.rec_count = rcnt; r.next = SSE_NONE;
        P.runs[idx] = r;
        if (rc.last_idx != SSE_NONE) P.runs[rc.last_idx].next = idx;
    }
    if (rc.last_idx == SSE_NONE) rc.first.next = idx;
    rc.last_idx = idx;
}

// ---------------------------------------------------------------- SSE_FLAG_DEFER: results that do not fit wait for a later batch
// The produce stage allocates with plain atomicAdds (no compare-and-swap on the hot path), so a round or long line that does not
// fit may leave its counters past a capacity (sse_download clamps them) and holes below it. Out bytes, frames and records in a hole
// are never referenced by a run. Work items are read by the sort and decode stages whatever references them, so every work item a
// deferred allocation got below cap_items becomes an empty item that decodes into the sink record recs[cap_recs], which is
// allocated past the capacity and never returned.

__device__ __noinline__ void empty_items(const KParams &P, uint32_t qb, uint32_t n) {
    const uint32_t e = min(qb + n, P.cap_items);
    for (uint32_t i = qb + lane_id(); i < e; i += 32) P.items[i] = make_uint4(0u, 0u, P.cap_recs, 0u);
}

// SSE_FLAG_DEFER: a round's allocation did not fit (!fits), or the round needs a runs[] entry, which is reserved before the round
// writes anything. Returns true when the round may write its results; false: its allocation becomes a hole and the segment stops
// before the round.
__device__ __noinline__ bool admit_round(const KParams &P, RunChain &rc, bool fits, uint32_t qb, uint32_t nq, bool need_run) {
    const uint32_t lane = lane_id();
    uint32_t bits = SSE_OVF_OUT;
    if (fits && need_run) {
        uint32_t idx = 0;
        if (lane == 0) idx = atomicAdd(&P.ctr->n_runs, 1u);
        idx = __shfl_sync(FULL, idx, 0);
        if (idx < P.cap_runs) { rc.pre = idx; return true; }
        bits = SSE_OVF_RUNS;
    }
    empty_items(P, qb, nq);
    if (lane == 0) atomicOr(&P.ctr->overflow, bits);     // reported, but the batch stays good (status untouched)
    return false;
}

// SSE_FLAG_DEFER: everything a held line of L bytes ('\n' included) can need when it completes, or nothing: out bytes for the
// line and the second '\n' of a mode R frame (a pooled line is gathered there and emitted in place), one frame, one record, one
// work item and, after the segment's first run, one runs[] entry.
__device__ __noinline__ bool reserve_long(const KParams &P, RunChain &rc, uint32_t L) {
    const uint32_t lane = lane_id(), bytes = (L + 2u + 15u) & ~15u;
    const bool need_run = rc.have_first;
    uint32_t ob = 0, qb = 0, fb = 0, rb = 0, ri = 0;
    if (lane == 0) {
        const unsigned long long r0 = atomicAdd(reinterpret_cast<unsigned long long *>(&P.ctr->out_bytes), (unsigned long long)bytes | (1ull << 32));
        const unsigned long long r1 = atomicAdd(reinterpret_cast<unsigned long long *>(&P.ctr->n_frames), 1ull | (1ull << 32));
        ob = (uint32_t)r0; qb = (uint32_t)(r0 >> 32); fb = (uint32_t)r1; rb = (uint32_t)(r1 >> 32);
        if (need_run) ri = atomicAdd(&P.ctr->n_runs, 1u);
    }
    ob = __shfl_sync(FULL, ob, 0); qb = __shfl_sync(FULL, qb, 0); fb = __shfl_sync(FULL, fb, 0); rb = __shfl_sync(FULL, rb, 0);
    ri = __shfl_sync(FULL, ri, 0);
    const bool run_ok = !need_run || ri < P.cap_runs;
    const bool rest_ok = ob + bytes + 16u <= P.cap_out && qb < P.cap_items && fb < P.cap_frames && rb < P.cap_recs;
    if (!run_ok || !rest_ok) {
        empty_items(P, qb, 1u);
        if (lane == 0) atomicOr(&P.ctr->overflow, (run_ok ? 0u : SSE_OVF_RUNS) | (rest_ok ? 0u : SSE_OVF_OUT));
        return false;
    }
    // the work item stays empty unless the line turns out to have a payload to decode (process_long_line overwrites it)
    if (lane == 0) P.items[qb] = make_uint4(0u, 0u, P.cap_recs, 0u);
    rc.rv.ob = ob; rc.rv.qb = qb; rc.rv.fb = fb; rc.rv.rb = rb;
    rc.pre = need_run ? ri : SSE_NONE;
    return true;
}

// A line that never fit the window, assembled in the connection's carry slot (HBM): classified and emitted straight from
// global memory. Its payload becomes a work item of segment seg like any other line's -- the decode kernel reads payloads
// from the arenas, so a line of any length up to carry_slot_bytes is decoded. at != SSE_NONE: the line already stands in the
// out arena at offset `at` (a pooled line gathered there, one spare byte after it) and is emitted in place: frame, payload
// and the swallowed line's materialised payload are spans of it, nothing is copied. resv (SSE_FLAG_DEFER): the line's results
// go where reserve_long put them (rc.rv), and what the line does not use of that reservation is left as a hole.
template <bool RESV>
__device__ __noinline__ bool process_long_line(const KParams &P, RunChain &rc, const uint8_t *line, int L, uint32_t mode, uint32_t seg,
                                               uint32_t at = SSE_NONE) {
    const uint32_t lane = lane_id();
    int a = 0, b = L;           // frame source [a, b) ; R: trimmed
    bool emit = true, done = false, parse = false, pref = false;
    int flen = L;
    if (mode & SSE_MODE_R) {
        trim_space(line, a, b);   // every lane, from global (ends only)
        bool found = false;
        for (int i = a + (int)lane; i + 6 <= b; i += 32) if (is_done_at(line + i)) found = true;
        done = __any_sync(FULL, found);
        pref = is_data_prefix(line + a, b - a);
        emit = !done && pref && (b - a) > 6;
        flen = emit ? (b - a) + 2 : 0;
        parse = emit || (done);
    } else {
        pref = is_data_prefix(line, L);
        parse = (mode & SSE_MODE_PARSE) && pref;
    }
    // payload handed to the decoder: [ps, pe) of the line
    const int ps = (mode & SSE_MODE_R) ? (pref ? a + 6 : a) : 6, pe = (mode & SSE_MODE_R) ? b : L - 1;
    // `data: [DONE]` once its white space is trimmed: nothing to decode, the record is final and there is no work item
    const bool exact = done && pref && pe - ps == 6;
    const bool item = parse && !exact;
    const uint32_t extra = (parse && !emit) ? (uint32_t)(pe - ps) : 0u;   // a swallowed line's payload is materialised for the decoder
    uint32_t nf = emit ? 1u : 0u, nr = parse ? 1u : 0u;
    const bool in_place = at != SSE_NONE;
    uint32_t ob = 0, fb = 0, rb = 0, qb = 0;
    if (RESV) {
        ob = rc.rv.ob; fb = rc.rv.fb; rb = rc.rv.rb; qb = rc.rv.qb;
    } else {
        if (lane == 0) {
            if ((nf || extra) && !in_place) ob = atomicAdd(&P.ctr->out_bytes, ((uint32_t)flen + extra + 15u) & ~15u);
            if (nf) fb = atomicAdd(&P.ctr->n_frames, 1u);
            if (nr) rb = atomicAdd(&P.ctr->n_recs, 1u);
            if (item) qb = atomicAdd(&P.ctr->n_items, 1u);
        }
        ob = __shfl_sync(FULL, ob, 0); fb = __shfl_sync(FULL, fb, 0); rb = __shfl_sync(FULL, rb, 0); qb = __shfl_sync(FULL, qb, 0);
        bool ovf = (!in_place && (nf || extra) && (ob + (uint32_t)flen + extra + 16u > P.cap_out)) || (nf && fb >= P.cap_frames) ||
                   (nr && rb >= P.cap_recs) || (item && qb >= P.cap_items);
        if (ovf) { if (lane == 0) sse_overflow(P.ctr, SSE_OVF_OUT); return false; }
    }
    // frame and payload offsets in the out arena
    const uint32_t fo = in_place ? at + (uint32_t)((mode & SSE_MODE_R) ? a : 0) : ob;
    const uint32_t po = in_place ? at + (uint32_t)ps : (emit ? ob + (uint32_t)(ps - ((mode & SSE_MODE_R) ? a : 0)) : ob);
    if (emit) {
        if (mode & SSE_MODE_R) {
            if (!in_place) copy_g2g_bytes(P.out + fo, line + a, b - a);
            __syncwarp();   // in place: every lane has read the line's trimmed end before it is overwritten
            if (lane < 2) P.out[fo + (uint32_t)(b - a) + lane] = '\n';
        } else if (!in_place) copy_g2g_bytes(P.out + fo, line, L);
        if (lane == 0) { sse_frame f; f.off = fo; f.len = (uint32_t)flen; P.frames[fb] = f; }
    } else if (extra && !in_place) copy_g2g_bytes(P.out + ob, line + ps, pe - ps);
    if (parse && lane == 0) {
        sse_rec r;
        r.frame = emit ? fb : SSE_NONE;
        r.flags = exact ? (SSE_F_DONE_LINE | SSE_F_DONE_EXACT) : 0u;
        r.content_off = r.content_len = 0; r.tc_first = SSE_NONE; r.tc_count = 0; r.n_choices = 0; r.usage = SSE_NONE;
        r.payload_len = (uint32_t)(pe - ps);
        P.recs[rb] = r;
        if (item) {
            uint4 it;
            it.x = po;
            it.y = (uint32_t)(pe - ps) | (done ? 0x40000000u : ((mode & SSE_MODE_R) ? 0x80000000u : 0u));
            it.z = rb; it.w = seg;
            P.items[qb] = it;
        }
    }
    append_run(P, rc, fb, nf, rb, nr);
    if (RESV) rc.pre = SSE_NONE;      // a reserved runs[] entry this line did not use stays a hole
    return true;
}

// ---------------------------------------------------------------- line pool (lines longer than the carry slot)
// One lane at a time moves pages, under a spin lock: a page moves once per page_bytes of a long line, so the lock is cold. Pool
// metadata is read and written volatile (L2), because the lanes that move pages run on every SM.
__device__ __forceinline__ void pool_lock(PoolHdr *h) {
    uint32_t ns = 32;      // exponential back-off: hundreds of long lines may want a page at once
    while (atomicCAS(&h->lock, 0u, 1u) != 0u) { __nanosleep(ns); if (ns < 2048u) ns <<= 1; }
    __threadfence();
}
__device__ __forceinline__ void pool_unlock(PoolHdr *h) {
    __threadfence();
    atomicExch(&h->lock, 0u);
}
__device__ __forceinline__ uint32_t pool_next_page(const KParams &P, uint32_t pg) { return ((volatile uint32_t *)P.pool_next)[pg]; }

// Every page of conn's chain back on the free stack (caller holds the lock).
__device__ __noinline__ void pool_release_locked(const KParams &P, uint32_t conn) {
    volatile PoolHdr *h = P.pool_hdr;
    volatile PoolChain *c = P.pool_chain + conn;
    volatile uint32_t *stk = P.pool_stack;
    uint32_t n = h->n_free, pg = c->first;
    const uint32_t k = c->n_pages;
    for (uint32_t i = 0; i < k; i++) { stk[n++] = pg; pg = pool_next_page(P, pg); }
    h->n_free = n;
    c->first = c->last = SSE_NONE; c->n_pages = 0;
}

// conn's chain grows from `have` to `want` > have pages, all or none (caller holds the lock). Returns the page the next bytes
// go to (the old last page when it has room: from_last), SSE_NONE when too few pages are free.
__device__ __noinline__ uint32_t pool_grow_locked(const KParams &P, uint32_t conn, uint32_t have, uint32_t want, bool from_last) {
    volatile PoolHdr *h = P.pool_hdr;
    volatile PoolChain *c = P.pool_chain + conn;
    volatile uint32_t *stk = P.pool_stack, *nxt = P.pool_next;
    uint32_t n = h->n_free;
    if (want - have > n) return SSE_NONE;
    uint32_t first = have ? c->first : SSE_NONE, last = have ? c->last : SSE_NONE;
    uint32_t start = from_last ? last : SSE_NONE;
    for (uint32_t k = have; k < want; k++) {
        const uint32_t p = stk[--n];
        if (last == SSE_NONE) first = p; else nxt[last] = p;
        if (start == SSE_NONE) start = p;
        last = p;
    }
    h->n_free = n;
    if (P.pool_pages - n > h->high_water) h->high_water = P.pool_pages - n;
    c->first = first; c->last = last; c->n_pages = want;
    return start;
}

// Cold path of a line that outgrows the carry slot. The held-back line (clen bytes: in the slot while clen <= carry_slot,
// else all of them in pool pages) grows by `take` bytes of the warp's window at src. Takes the pages the longer line needs,
// moves the slot bytes to the first page when the line leaves the slot, appends. Fails, and returns the connection's pages,
// when the line would exceed max_line or too few pages are free (a pool of zero pages never has a free page).
__device__ __noinline__ bool pool_append(const KParams &P, uint32_t conn, const uint8_t *slot, int clen, const uint8_t *src, int take) {
    if (take == 0) return true;     // nothing to hold (an empty segment): the line and its chain stay as they are
    const uint32_t lane = lane_id(), PB = P.page_bytes;
    const bool leave_slot = clen <= (int)P.carry_slot;
    const uint32_t old_len = leave_slot ? 0u : (uint32_t)clen, new_len = (uint32_t)clen + (uint32_t)take;
    uint32_t pg = SSE_NONE;
    if (lane == 0) {
        const bool fits = new_len <= P.max_line;        // (max_line == carry_slot without a pool)
        const uint32_t have = (old_len + PB - 1) / PB, want = (new_len + PB - 1) / PB;
        if (fits && have == want) {
            // the bytes fit the last page (take > 0 and no new page: the line is pooled and its last page has room). Only
            // this warp changes the connection's chain during the launch, so it is read without the lock
            pg = ((volatile PoolChain *)P.pool_chain)[conn].last;
        } else if (fits || !leave_slot) {
            pool_lock(P.pool_hdr);
            if (fits) pg = pool_grow_locked(P, conn, have, want, (old_len % PB) != 0);
            if (pg == SSE_NONE) pool_release_locked(P, conn);
            pool_unlock(P.pool_hdr);
        }
    }
    pg = __shfl_sync(FULL, pg, 0);
    __syncwarp();
    if (pg == SSE_NONE) return false;
    uint32_t off = old_len % PB;
    if (leave_slot) {        // slot -> pages: both 16-byte aligned, whole vectors (the slot is a multiple of 16 bytes long)
        for (uint32_t d = 0; d < (uint32_t)clen;) {
            if (off == PB) { pg = pool_next_page(P, pg); off = 0; }
            const uint32_t n = min(PB - off, (uint32_t)clen - d);
            const uint4 *s = reinterpret_cast<const uint4 *>(slot + d);
            uint4 *o = reinterpret_cast<uint4 *>(P.pool + (size_t)pg * PB);
            for (uint32_t i = lane; i < (n + 15u) >> 4; i += 32) o[i] = s[i];
            d += n; off += n;
        }
        __syncwarp();        // the vector tail past clen is overwritten below
    }
    for (uint32_t d = 0; d < (uint32_t)take;) {
        if (off == PB) { pg = pool_next_page(P, pg); off = 0; }
        const uint32_t n = min(PB - off, (uint32_t)take - d);
        copy_s2g_vec(P.pool + (size_t)pg * PB + off, src + d, (int)n);
        d += n; off += n;
    }
    __syncwarp();
    return true;
}

// A pooled line is complete (its last byte, the '\n', was appended): gathered from its pages into the out arena with 16-byte
// copies, classified and emitted in place by process_long_line, then its pages are returned to the pool.
template <bool RESV>
__device__ __noinline__ bool pool_long_line(const KParams &P, RunChain &rc, uint32_t conn, int L, uint32_t mode, uint32_t seg) {
    const uint32_t lane = lane_id(), PB = P.page_bytes;
    const uint32_t bytes = ((uint32_t)L + 1u + 15u) & ~15u;    // + 1: mode R's frame ends in a second '\n'
    uint32_t ob = 0, pg = 0;
    if (lane == 0) { if (!RESV) ob = atomicAdd(&P.ctr->out_bytes, bytes); pg = ((volatile PoolChain *)P.pool_chain)[conn].first; }
    ob = RESV ? rc.rv.ob : __shfl_sync(FULL, ob, 0); pg = __shfl_sync(FULL, pg, 0);
    // on overflow the batch is discarded and the chain stays with the connection: its state still describes the line
    if (!RESV && ob + bytes + 16u > P.cap_out) { if (lane == 0) sse_overflow(P.ctr, SSE_OVF_OUT); return false; }
    for (uint32_t d = 0; d < (uint32_t)L; d += PB) {
        if (d) pg = pool_next_page(P, pg);
        const uint32_t nv = (min(PB, (uint32_t)L - d) + 15u) >> 4;
        const uint4 *s = reinterpret_cast<const uint4 *>(P.pool + (size_t)pg * PB);
        uint4 *o = reinterpret_cast<uint4 *>(P.out + ob + d);
        for (uint32_t i = lane; i < nv; i += 32) o[i] = __ldcg(s + i);
    }
    __syncwarp();
    const bool ok = process_long_line<RESV>(P, rc, P.out + ob, L, mode, seg, ob);
    __syncwarp();
    if (lane == 0) { pool_lock(P.pool_hdr); pool_release_locked(P, conn); pool_unlock(P.pool_hdr); }
    __syncwarp();
    return ok;
}

// Holds `take` bytes of the window back as the continuation of the connection's unterminated line: in the carry slot while
// the line fits it, else in line-pool pages. false: the line cannot be held (longer than max_line, or no free page).
__device__ __forceinline__ bool hold_back(const KParams &P, uint32_t conn, uint8_t *slot, int clen, const uint8_t *src, int take) {
    if (clen + take > (int)P.carry_slot) return pool_append(P, conn, slot, clen, src, take);
    copy_s2g_bytes(slot + clen, src, take);
    return true;
}

// SSE_FLAG_DEFER: the held line of clen bytes gives back its last byte, the '\n' just appended, so that the connection's state
// describes the line without it. Only the pool can have changed: the '\n' may have taken a new last page, or moved the line
// out of the carry slot. In the second case the slot holds only the bytes it had before this window (pool_append leaves them
// there, but writes the window's bytes to the pages alone), so the line's keep bytes are copied back from the pages into the
// slot before the pages go back.
__device__ __noinline__ void drop_newline(const KParams &P, uint32_t conn, uint8_t *slot, int clen) {
    const uint32_t keep = (uint32_t)clen - 1u, PB = P.page_bytes;
    if (clen <= (int)P.carry_slot || (keep > P.carry_slot && keep % PB != 0)) return;
    if (keep <= P.carry_slot) {
        uint32_t pg = 0;
        if (lane_id() == 0) pg = ((volatile PoolChain *)P.pool_chain)[conn].first;
        pg = __shfl_sync(FULL, pg, 0);
        for (uint32_t d = 0; d < keep; d += PB) {     // this warp wrote the pages (pool_append ends in __syncwarp)
            if (d) pg = pool_next_page(P, pg);
            const uint32_t n = min(PB, keep - d);
            copy_g2g_bytes(slot + d, P.pool + (size_t)pg * PB, (int)n);
        }
        __syncwarp();
    }
    if (lane_id() == 0) {
        pool_lock(P.pool_hdr);
        if (keep <= P.carry_slot) pool_release_locked(P, conn);
        else {
            volatile PoolHdr *h = P.pool_hdr;
            volatile PoolChain *c = P.pool_chain + conn;
            const uint32_t k = c->n_pages;
            uint32_t pg = c->first;
            for (uint32_t i = 0; i + 2u < k; i++) pg = pool_next_page(P, pg);
            const uint32_t n = h->n_free;
            ((volatile uint32_t *)P.pool_stack)[n] = c->last;
            h->n_free = n + 1u;
            c->last = pg; c->n_pages = k - 1u;
        }
        pool_unlock(P.pool_hdr);
    }
    __syncwarp();
}

// A line assembled outside the window is complete (clen bytes, '\n' included): in the carry slot, or in the pool. false: its
// results do not fit; without SSE_FLAG_DEFER the batch has failed. With SSE_FLAG_DEFER everything the line's results can need
// is reserved before anything is written, and when that does not fit the line gives its '\n' back: the connection keeps the
// line's other bytes (clen - 1) and the '\n' is the first byte the caller resubmits.
template <bool DEFER>
__device__ __noinline__ bool complete_long_line(const KParams &P, RunChain &rc, uint32_t conn, uint8_t *slot, int clen, uint32_t mode, uint32_t seg) {
    if (DEFER && !reserve_long(P, rc, (uint32_t)clen)) { drop_newline(P, conn, slot, clen); return false; }
    return clen > (int)P.carry_slot ? pool_long_line<DEFER>(P, rc, conn, clen, mode, seg)
                                    : process_long_line<DEFER>(P, rc, slot, clen, mode, seg);
}

} // namespace
