/*
 * sse_oracle.c -- CPU restatement of the reference's streaming-response path.
 * TEST INFRASTRUCTURE ONLY (see sse_oracle.h for scope, pinning status and citations).
 *
 * Structure mirrors the reference deliberately: encoding/json is restated as the two phases Go
 * runs (checkValid over the whole document, then a typed recursive-descent decode into the
 * struct graph of providers/types/common_types.go), and each consumer loop is restated as its
 * own function.  The product (inference_gateway_b200/csrc) is a single-pass iterative machine,
 * so the two implementations share no structure.
 */
#include "sse_oracle.h"
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------ buffers */
static void *xgrow(void *p, size_t *cap, size_t need, size_t esz) {
    if (need <= *cap) return p;
    size_t nc = *cap ? *cap * 2 : 64;
    while (nc < need) nc *= 2;
    p = realloc(p, nc * esz);
    if (!p) abort();
    *cap = nc;
    return p;
}
typedef struct { uint8_t *p; size_t n, cap; } buf;
static void buf_put(buf *b, const void *s, size_t n) {
    b->p = (uint8_t *)xgrow(b->p, &b->cap, b->n + n + 1, 1);
    if (n) memcpy(b->p + b->n, s, n);
    b->n += n;
}
static _Thread_local buf g_builder; /* responseBodyBuilder of the last orc_reframe_stream (per thread) */

orc_result *orc_result_new(void) { return (orc_result *)calloc(1, sizeof(orc_result)); }
void orc_result_clear(orc_result *r) {
    r->out_len = r->text_len = r->n_lines = r->n_chunks = r->n_tcs = 0;
    r->acc_content.off = r->acc_content.len = 0;
    r->has_tool_calls = r->terminated = r->term_finish = 0;
    r->tail_len = 0;
}
void orc_result_free(orc_result *r) {
    if (!r) return;
    free(r->out); free(r->text); free(r->lines); free(r->chunks); free(r->tcs); free(r);
}
static uint32_t out_put(orc_result *r, const void *s, size_t n) {
    r->out = (uint8_t *)xgrow(r->out, &r->out_cap, r->out_len + n + 1, 1);
    uint32_t off = (uint32_t)r->out_len;
    if (n) memcpy(r->out + r->out_len, s, n);
    r->out_len += n;
    return off;
}
static uint32_t text_put(orc_result *r, const void *s, size_t n) {
    r->text = (uint8_t *)xgrow(r->text, &r->text_cap, r->text_len + n + 1, 1);
    uint32_t off = (uint32_t)r->text_len;
    if (n) memcpy(r->text + r->text_len, s, n);
    r->text_len += n;
    return off;
}
static orc_line *line_new(orc_result *r) {
    r->lines = (orc_line *)xgrow(r->lines, &r->cap_lines, r->n_lines + 1, sizeof(orc_line));
    orc_line *l = &r->lines[r->n_lines++];
    memset(l, 0, sizeof *l);
    l->chunk = 0xFFFFFFFFu;
    return l;
}

/* ------------------------------------------------------------------ strings.TrimSpace
 * Go: ASCII fast path; on a byte >= 0x80 falls back to TrimFunc(unicode.IsSpace), which decodes
 * runes (utf8.DecodeRune / DecodeLastRune). White_Space code points and their UTF-8 forms: */
static size_t space_prefix(const uint8_t *s, size_t n) {
    if (n == 0) return 0;
    uint8_t c = s[0];
    if (c == ' ' || (c >= 0x09 && c <= 0x0D)) return 1;
    if (c < 0x80) return 0;
    if (n >= 2 && c == 0xC2 && (s[1] == 0x85 || s[1] == 0xA0)) return 2;
    if (n >= 3) {
        if (c == 0xE1 && s[1] == 0x9A && s[2] == 0x80) return 3;             /* U+1680 */
        if (c == 0xE2 && s[1] == 0x80 &&
            ((s[2] >= 0x80 && s[2] <= 0x8A) || s[2] == 0xA8 || s[2] == 0xA9 || s[2] == 0xAF)) return 3;
        if (c == 0xE2 && s[1] == 0x81 && s[2] == 0x9F) return 3;             /* U+205F */
        if (c == 0xE3 && s[1] == 0x80 && s[2] == 0x80) return 3;             /* U+3000 */
    }
    return 0;
}
static size_t space_suffix(const uint8_t *s, size_t n) {
    if (n == 0) return 0;
    uint8_t c = s[n - 1];
    if (c == ' ' || (c >= 0x09 && c <= 0x0D)) return 1;
    if (c < 0x80) return 0;
    if (n >= 2 && space_prefix(s + n - 2, 2) == 2) return 2;
    if (n >= 3 && space_prefix(s + n - 3, 3) == 3) return 3;
    return 0;
}
void orc_trim_space(const uint8_t *s, size_t n, size_t *a, size_t *b) {
    size_t i = 0, j = n, k;
    while (i < j && (k = space_prefix(s + i, j - i)) != 0) i += k;
    while (j > i && (k = space_suffix(s + i, j - i)) != 0) j -= k;
    *a = i; *b = j;
}
static int contains(const uint8_t *s, size_t n, const char *needle) {
    size_t m = strlen(needle);
    if (m > n) return 0;
    for (size_t i = 0; i + m <= n; i++) if (memcmp(s + i, needle, m) == 0) return 1;
    return 0;
}
static int has_prefix(const uint8_t *s, size_t n, const char *p) {
    size_t m = strlen(p);
    return n >= m && memcmp(s, p, m) == 0;
}

/* ------------------------------------------------------------------ encoding/json: checkValid
 * Go's scanner (encoding/json/scanner.go): RFC 8259 grammar, whitespace = SP HT CR LF,
 * raw bytes < 0x20 illegal in strings, bytes >= 0x80 unchecked, nesting limit 10000. */
#define ORC_MAX_DEPTH 10000
typedef struct { const uint8_t *s; size_t n, p; int max_depth, depth_hit; } jscan;
static void js_ws(jscan *j) {
    while (j->p < j->n) {
        uint8_t c = j->s[j->p];
        if (c == ' ' || c == '\t' || c == '\r' || c == '\n') j->p++; else break;
    }
}
static int is_hex(uint8_t c) { return (c >= '0' && c <= '9') || (c >= 'a' && c <= 'f') || (c >= 'A' && c <= 'F'); }
static int js_string(jscan *j) { /* at opening quote */
    j->p++;
    while (j->p < j->n) {
        uint8_t c = j->s[j->p++];
        if (c == '"') return 1;
        if (c < 0x20) return 0;
        if (c == '\\') {
            if (j->p >= j->n) return 0;
            uint8_t e = j->s[j->p++];
            switch (e) {
            case '"': case '\\': case '/': case 'b': case 'f': case 'n': case 'r': case 't': break;
            case 'u':
                if (j->p + 4 > j->n) return 0;
                for (int k = 0; k < 4; k++) if (!is_hex(j->s[j->p + k])) return 0;
                j->p += 4; break;
            default: return 0;
            }
        }
    }
    return 0;
}
static int js_number(jscan *j) {
    const uint8_t *s = j->s; size_t n = j->n, p = j->p;
    if (p < n && s[p] == '-') p++;
    if (p >= n) return 0;
    if (s[p] == '0') p++;
    else if (s[p] >= '1' && s[p] <= '9') { while (p < n && s[p] >= '0' && s[p] <= '9') p++; }
    else return 0;
    if (p < n && s[p] == '.') {
        p++;
        if (p >= n || s[p] < '0' || s[p] > '9') return 0;
        while (p < n && s[p] >= '0' && s[p] <= '9') p++;
    }
    if (p < n && (s[p] == 'e' || s[p] == 'E')) {
        p++;
        if (p < n && (s[p] == '+' || s[p] == '-')) p++;
        if (p >= n || s[p] < '0' || s[p] > '9') return 0;
        while (p < n && s[p] >= '0' && s[p] <= '9') p++;
    }
    j->p = p;
    return 1;
}
static int js_lit(jscan *j, const char *w) {
    size_t m = strlen(w);
    if (j->p + m > j->n || memcmp(j->s + j->p, w, m) != 0) return 0;
    j->p += m;
    return 1;
}
static int js_value(jscan *j, int depth) {
    js_ws(j);
    if (j->p >= j->n) return 0;
    uint8_t c = j->s[j->p];
    if (c == '{') {
        if (depth + 1 > j->max_depth) { j->depth_hit = 1; return 0; }
        j->p++; js_ws(j);
        if (j->p < j->n && j->s[j->p] == '}') { j->p++; return 1; }
        for (;;) {
            js_ws(j);
            if (j->p >= j->n || j->s[j->p] != '"') return 0;
            if (!js_string(j)) return 0;
            js_ws(j);
            if (j->p >= j->n || j->s[j->p] != ':') return 0;
            j->p++;
            if (!js_value(j, depth + 1)) return 0;
            js_ws(j);
            if (j->p >= j->n) return 0;
            if (j->s[j->p] == ',') { j->p++; continue; }
            if (j->s[j->p] == '}') { j->p++; return 1; }
            return 0;
        }
    }
    if (c == '[') {
        if (depth + 1 > j->max_depth) { j->depth_hit = 1; return 0; }
        j->p++; js_ws(j);
        if (j->p < j->n && j->s[j->p] == ']') { j->p++; return 1; }
        for (;;) {
            if (!js_value(j, depth + 1)) return 0;
            js_ws(j);
            if (j->p >= j->n) return 0;
            if (j->s[j->p] == ',') { j->p++; continue; }
            if (j->s[j->p] == ']') { j->p++; return 1; }
            return 0;
        }
    }
    if (c == '"') return js_string(j);
    if (c == '-' || (c >= '0' && c <= '9')) return js_number(j);
    if (c == 't') return js_lit(j, "true");
    if (c == 'f') return js_lit(j, "false");
    if (c == 'n') return js_lit(j, "null");
    return 0;
}
int orc_json_scan(const uint8_t *s, size_t n, int max_depth) {
    jscan j = { s, n, 0, max_depth, 0 };
    if (!js_value(&j, 0)) return j.depth_hit ? ORC_JSON_DEPTH : ORC_JSON_SYNTAX;
    js_ws(&j);
    return j.p == n ? ORC_JSON_OK : ORC_JSON_SYNTAX;
}
int orc_json_valid(const uint8_t *s, size_t n) { return orc_json_scan(s, n, ORC_MAX_DEPTH) == ORC_JSON_OK; }

/* ------------------------------------------------------------------ encoding/json: unquote
 * decode.go unquoteBytes: escapes, surrogate pairs, lone surrogate -> U+FFFD, invalid UTF-8 ->
 * U+FFFD per offending byte (utf8.DecodeRune acceptance ranges). Input is the string body
 * (between the quotes) of an already validated literal. */
static int hex4(const uint8_t *s) {
    int v = 0;
    for (int k = 0; k < 4; k++) {
        uint8_t c = s[k]; int d;
        if (c >= '0' && c <= '9') d = c - '0';
        else if (c >= 'a' && c <= 'f') d = c - 'a' + 10;
        else if (c >= 'A' && c <= 'F') d = c - 'A' + 10;
        else return -1;
        v = v * 16 + d;
    }
    return v;
}
static size_t utf8_valid_len(const uint8_t *s, size_t n) { /* utf8.DecodeRune: size if valid else 0 */
    uint8_t c = s[0];
    if (c < 0x80) return 1;
    if (c >= 0xC2 && c <= 0xDF) return (n >= 2 && (s[1] & 0xC0) == 0x80) ? 2 : 0;
    if (c >= 0xE0 && c <= 0xEF) {
        uint8_t lo = 0x80, hi = 0xBF;
        if (c == 0xE0) lo = 0xA0;
        if (c == 0xED) hi = 0x9F;
        return (n >= 3 && s[1] >= lo && s[1] <= hi && (s[2] & 0xC0) == 0x80) ? 3 : 0;
    }
    if (c >= 0xF0 && c <= 0xF4) {
        uint8_t lo = 0x80, hi = 0xBF;
        if (c == 0xF0) lo = 0x90;
        if (c == 0xF4) hi = 0x8F;
        return (n >= 4 && s[1] >= lo && s[1] <= hi && (s[2] & 0xC0) == 0x80 && (s[3] & 0xC0) == 0x80) ? 4 : 0;
    }
    return 0;
}
static void put_rune(buf *b, uint32_t r) {
    uint8_t t[4]; size_t k;
    if (r < 0x80) { t[0] = (uint8_t)r; k = 1; }
    else if (r < 0x800) { t[0] = 0xC0 | (r >> 6); t[1] = 0x80 | (r & 0x3F); k = 2; }
    else if (r < 0x10000) { t[0] = 0xE0 | (r >> 12); t[1] = 0x80 | ((r >> 6) & 0x3F); t[2] = 0x80 | (r & 0x3F); k = 3; }
    else { t[0] = 0xF0 | (r >> 18); t[1] = 0x80 | ((r >> 12) & 0x3F); t[2] = 0x80 | ((r >> 6) & 0x3F); t[3] = 0x80 | (r & 0x3F); k = 4; }
    buf_put(b, t, k);
}
static void unquote(const uint8_t *s, size_t n, buf *b) {
    b->n = 0;
    size_t i = 0;
    while (i < n) {
        uint8_t c = s[i];
        if (c == '\\') {
            uint8_t e = s[i + 1];
            i += 2;
            switch (e) {
            case '"': case '\\': case '/': { uint8_t t = e; buf_put(b, &t, 1); break; }
            case 'b': { uint8_t t = '\b'; buf_put(b, &t, 1); break; }
            case 'f': { uint8_t t = '\f'; buf_put(b, &t, 1); break; }
            case 'n': { uint8_t t = '\n'; buf_put(b, &t, 1); break; }
            case 'r': { uint8_t t = '\r'; buf_put(b, &t, 1); break; }
            case 't': { uint8_t t = '\t'; buf_put(b, &t, 1); break; }
            case 'u': {
                uint32_t rr = (uint32_t)hex4(s + i);
                i += 4;
                if (rr >= 0xD800 && rr < 0xE000) {
                    int rr1 = -1;
                    if (i + 6 <= n && s[i] == '\\' && s[i + 1] == 'u') rr1 = hex4(s + i + 2);
                    if (rr < 0xDC00 && rr1 >= 0xDC00 && rr1 < 0xE000) {
                        rr = 0x10000 + ((rr - 0xD800) << 10) + ((uint32_t)rr1 - 0xDC00);
                        i += 6;
                    } else rr = 0xFFFD;
                }
                put_rune(b, rr);
                break;
            }
            }
        } else if (c < 0x80) {
            buf_put(b, &c, 1); i++;
        } else {
            size_t k = utf8_valid_len(s + i, n - i);
            if (k == 0) { put_rune(b, 0xFFFD); i++; }
            else { buf_put(b, s + i, k); i += k; }
        }
    }
}

/* ------------------------------------------------------------------ encoding/json: typed decode */
enum { TY_SKIP, TY_STR, TY_PSTR, TY_INT, TY_F32, TY_STRUCT, TY_PSTRUCT, TY_SLICE, TY_PSLICE, TY_GOOGLE };
enum { S_NONE, S_ROOT, S_CHOICE, S_DELTA, S_TC, S_FUNC, S_EXTRA, S_USAGE, S_LOGPROBS, S_TOKLP, S_TOPLP };
enum { TG_NONE, TG_CHOICES, TG_USAGE, TG_PROMPT, TG_COMPLETION, TG_TOTAL, TG_FINISH, TG_CONTENT,
       TG_TOOLCALLS, TG_TC_ID, TG_TC_TYPE, TG_TC_INDEX, TG_TC_FUNCTION, TG_NAME, TG_ARGS };
typedef struct { const char *name; int ty, sub, ety, esub, tgt; } field;

/* struct tags of providers/types/common_types.go */
static const field F_ROOT[] = {               /* :451-478 */
    { "choices", TY_SLICE, 0, TY_STRUCT, S_CHOICE, TG_CHOICES },
    { "created", TY_INT, 0, 0, 0, 0 }, { "id", TY_STR, 0, 0, 0, 0 }, { "model", TY_STR, 0, 0, 0, 0 },
    { "object", TY_STR, 0, 0, 0, 0 }, { "reasoning_format", TY_PSTR, 0, 0, 0, 0 },
    { "system_fingerprint", TY_PSTR, 0, 0, 0, 0 }, { "usage", TY_PSTRUCT, S_USAGE, 0, 0, TG_USAGE }, { 0 } };
static const field F_CHOICE[] = {             /* :300-321 */
    { "delta", TY_STRUCT, S_DELTA, 0, 0, 0 }, { "finish_reason", TY_STR, 0, 0, 0, TG_FINISH },
    { "index", TY_INT, 0, 0, 0, 0 }, { "logprobs", TY_PSTRUCT, S_LOGPROBS, 0, 0, 0 }, { 0 } };
static const field F_DELTA[] = {              /* :330-346 */
    { "content", TY_STR, 0, 0, 0, TG_CONTENT }, { "reasoning", TY_PSTR, 0, 0, 0, 0 },
    { "reasoning_content", TY_PSTR, 0, 0, 0, 0 }, { "refusal", TY_PSTR, 0, 0, 0, 0 },
    { "role", TY_STR, 0, 0, 0, 0 }, { "tool_calls", TY_PSLICE, 0, TY_STRUCT, S_TC, TG_TOOLCALLS }, { 0 } };
static const field F_TC[] = {                 /* :271-288 */
    { "extra_content", TY_PSTRUCT, S_EXTRA, 0, 0, 0 }, { "function", TY_PSTRUCT, S_FUNC, 0, 0, TG_TC_FUNCTION },
    { "id", TY_PSTR, 0, 0, 0, TG_TC_ID }, { "index", TY_INT, 0, 0, 0, TG_TC_INDEX },
    { "type", TY_PSTR, 0, 0, 0, TG_TC_TYPE }, { 0 } };
static const field F_FUNC[] = {               /* :291-297 */
    { "arguments", TY_STR, 0, 0, 0, TG_ARGS }, { "name", TY_STR, 0, 0, 0, TG_NAME }, { 0 } };
static const field F_EXTRA[] = { { "google", TY_GOOGLE, 0, 0, 0, 0 }, { 0 } };   /* :686-689 */
static const field F_USAGE[] = {              /* :384-393 */
    { "completion_tokens", TY_INT, 0, 0, 0, TG_COMPLETION }, { "prompt_tokens", TY_INT, 0, 0, 0, TG_PROMPT },
    { "total_tokens", TY_INT, 0, 0, 0, TG_TOTAL }, { 0 } };
static const field F_LOGPROBS[] = {           /* :314-320 */
    { "content", TY_SLICE, 0, TY_STRUCT, S_TOKLP, 0 }, { "refusal", TY_SLICE, 0, TY_STRUCT, S_TOKLP, 0 }, { 0 } };
static const field F_TOKLP[] = {              /* :349-371 */
    { "bytes", TY_SLICE, 0, TY_INT, 0, 0 }, { "logprob", TY_F32, 0, 0, 0, 0 }, { "token", TY_STR, 0, 0, 0, 0 },
    { "top_logprobs", TY_SLICE, 0, TY_STRUCT, S_TOPLP, 0 }, { 0 } };
static const field F_TOPLP[] = {
    { "bytes", TY_SLICE, 0, TY_INT, 0, 0 }, { "logprob", TY_F32, 0, 0, 0, 0 }, { "token", TY_STR, 0, 0, 0, 0 }, { 0 } };
static const field *fields_of(int s) {
    switch (s) {
    case S_ROOT: return F_ROOT; case S_CHOICE: return F_CHOICE; case S_DELTA: return F_DELTA;
    case S_TC: return F_TC; case S_FUNC: return F_FUNC; case S_EXTRA: return F_EXTRA;
    case S_USAGE: return F_USAGE; case S_LOGPROBS: return F_LOGPROBS; case S_TOKLP: return F_TOKLP;
    case S_TOPLP: return F_TOPLP;
    }
    return 0;
}

typedef struct {
    const uint8_t *s; size_t n, p;
    int type_err;
    orc_result *r;
    /* decoded state of the response */
    uint32_t n_choices, finish, has_usage, tc_nonnil;
    int64_t prompt, completion, total;
    buf content;
    /* tool calls of choices[0] (strings kept in per-entry bufs until commit) */
    struct tcent { int64_t index; int has_id, has_type, has_function; buf id, type, name, args; } *tc;
    size_t n_tc, cap_tc;
    buf scratch;
} dec;

static void d_ws(dec *d) {
    while (d->p < d->n) { uint8_t c = d->s[d->p]; if (c == ' ' || c == '\t' || c == '\r' || c == '\n') d->p++; else break; }
}
static void d_skip(dec *d) { jscan j = { d->s, d->n, d->p, ORC_MAX_DEPTH, 0 }; js_value(&j, 0); d->p = j.p; }
/* reads a string literal at d->p, returns body span */
static void d_strbody(dec *d, size_t *a, size_t *b) {
    jscan j = { d->s, d->n, d->p, ORC_MAX_DEPTH, 0 }; js_string(&j);
    *a = d->p + 1; *b = j.p - 1; d->p = j.p;
}
/* foldName (encoding/json/fold.go, Go >= 1.21): ASCII upper-cases; U+212A -> 'K', U+017F -> 'S' */
static int key_matches(const uint8_t *k, size_t n, const char *name, int exact) {
    size_t m = strlen(name), i = 0, q = 0;
    if (exact) return n == m && memcmp(k, name, m) == 0;
    while (i < n) {
        uint32_t c = k[i];
        if (c < 0x80) { if (c >= 'a' && c <= 'z') c -= 32; i++; }
        else if (i + 1 < n && k[i] == 0xC5 && k[i + 1] == 0xBF) { c = 'S'; i += 2; }
        else if (i + 2 < n && k[i] == 0xE2 && k[i + 1] == 0x84 && k[i + 2] == 0xAA) { c = 'K'; i += 3; }
        else return 0;
        if (q >= m) return 0;
        uint32_t f = (uint8_t)name[q++];
        if (f >= 'a' && f <= 'z') f -= 32;
        if (c != f) return 0;
    }
    return q == m;
}
static const field *find_field(const field *fs, const uint8_t *k, size_t n) {
    for (const field *f = fs; f->name; f++) if (key_matches(k, n, f->name, 1)) return f;
    for (const field *f = fs; f->name; f++) if (key_matches(k, n, f->name, 0)) return f;
    return 0;
}

/* strconv.ParseInt(s, 10, 64) over a JSON number literal: 1 ok */
static int parse_int64(const uint8_t *s, size_t n, int64_t *out) {
    size_t i = 0; int neg = 0;
    if (i < n && s[i] == '-') { neg = 1; i++; }
    if (i >= n) return 0;
    uint64_t v = 0;
    for (; i < n; i++) {
        if (s[i] < '0' || s[i] > '9') return 0;      /* '.', 'e', 'E' -> syntax error in ParseInt */
        uint64_t dgt = (uint64_t)(s[i] - '0');
        if (v > (UINT64_MAX - dgt) / 10) return 0;
        v = v * 10 + dgt;
    }
    if (neg) { if (v > (uint64_t)INT64_MAX + 1) return 0; *out = (int64_t)(0 - v); }
    else { if (v > (uint64_t)INT64_MAX) return 0; *out = (int64_t)v; }
    return 1;
}
/* strconv.ParseFloat(s, 32) range error: |x| >= 2^128 - 2^103 rounds to +-Inf. Exact decimal compare. */
static int f32_overflows(const uint8_t *s, size_t n) {
    static const char H[] = "340282356779733661637539395458142568448"; /* 39 digits */
    size_t i = 0;
    if (i < n && s[i] == '-') i++;
    char dig[64]; size_t nd = 0; int64_t dexp = 0; int seen_nz = 0, sticky = 0;
    for (; i < n && s[i] >= '0' && s[i] <= '9'; i++) {
        if (s[i] != '0' || seen_nz) { seen_nz = 1; if (nd < 48) dig[nd++] = (char)s[i]; else if (s[i] != '0') sticky = 1; dexp++; }
    }
    if (i < n && s[i] == '.') {
        for (i++; i < n && s[i] >= '0' && s[i] <= '9'; i++) {
            if (s[i] != '0' || seen_nz) { seen_nz = 1; if (nd < 48) dig[nd++] = (char)s[i]; else if (s[i] != '0') sticky = 1; }
            else dexp--;
        }
    }
    if (!seen_nz) return 0;
    if (i < n && (s[i] == 'e' || s[i] == 'E')) {
        int eneg = 0; int64_t e = 0;
        i++;
        if (i < n && (s[i] == '+' || s[i] == '-')) { eneg = s[i] == '-'; i++; }
        for (; i < n && s[i] >= '0' && s[i] <= '9'; i++) if (e < 100000000) e = e * 10 + (s[i] - '0');
        dexp += eneg ? -e : e;
    }
    /* value = 0.dig x 10^dexp ; H = 0.3402... x 10^39 */
    if (dexp > 39) return 1;
    if (dexp < 39) return 0;
    for (size_t k = 0; k < 39; k++) {
        char c = k < nd ? dig[k] : '0';
        if (c > H[k]) return 1;
        if (c < H[k]) return 0;
    }
    (void)sticky;
    return 1; /* >= H */
}
static uint32_t classify_finish(const uint8_t *s, size_t n) {
    if (n == 0) return ORC_FIN_NONE;
    if (n == 4 && !memcmp(s, "stop", 4)) return ORC_FIN_STOP;
    if (n == 10 && !memcmp(s, "tool_calls", 10)) return ORC_FIN_TOOL_CALLS;
    if (n == 6 && !memcmp(s, "length", 6)) return ORC_FIN_LENGTH;
    if (n == 14 && !memcmp(s, "content_filter", 14)) return ORC_FIN_CONTENT_FILTER;
    if (n == 13 && !memcmp(s, "function_call", 13)) return ORC_FIN_FUNCTION_CALL;
    return ORC_FIN_OTHER;
}
static void reset_choice0(dec *d) {
    d->finish = ORC_FIN_NONE; d->content.n = 0; d->tc_nonnil = 0; d->n_tc = 0;
}
static struct tcent *tc_push(dec *d) {
    if (d->n_tc == d->cap_tc) {
        size_t oc = d->cap_tc;
        d->tc = (struct tcent *)xgrow(d->tc, &d->cap_tc, d->n_tc + 1, sizeof *d->tc);
        memset(d->tc + oc, 0, (d->cap_tc - oc) * sizeof *d->tc);
    }
    struct tcent *t = &d->tc[d->n_tc++];
    t->index = 0; t->has_id = t->has_type = t->has_function = 0;
    t->id.n = t->type.n = t->name.n = t->args.n = 0;
    return t;
}

static void d_value(dec *d, int ty, int sub, int ety, int esub, int tgt, int live, int depth);

static void d_google(dec *d) {
    /* ToolCallExtraContent_Google.UnmarshalJSON (common_types.go:835-862): map[string]RawMessage, then
     * the LAST "thought_signature" entry (exact key after unquote) must decode into *string. */
    int bad = 0;
    d->p++; d_ws(d);
    if (d->s[d->p] == '}') { d->p++; return; }
    for (;;) {
        d_ws(d);
        size_t a, b; d_strbody(d, &a, &b);
        unquote(d->s + a, b - a, &d->scratch);
        int is_ts = d->scratch.n == 17 && !memcmp(d->scratch.p, "thought_signature", 17);
        d_ws(d); d->p++; d_ws(d);
        uint8_t c = d->s[d->p];
        if (is_ts) bad = !(c == '"' || c == 'n');
        d_skip(d);
        d_ws(d);
        if (d->s[d->p] == ',') { d->p++; continue; }
        d->p++; break;
    }
    if (bad) d->type_err = 1;
}
static void d_object(dec *d, int sub, int live, int depth) {
    const field *fs = fields_of(sub);
    d->p++; d_ws(d);
    if (d->s[d->p] == '}') { d->p++; return; }
    for (;;) {
        d_ws(d);
        size_t a, b; d_strbody(d, &a, &b);
        unquote(d->s + a, b - a, &d->scratch);
        const field *f = find_field(fs, d->scratch.p, d->scratch.n);
        d_ws(d); d->p++; /* ':' */
        if (f) d_value(d, f->ty, f->sub, f->ety, f->esub, f->tgt, live, depth + 1);
        else d_value(d, TY_SKIP, 0, 0, 0, 0, 0, depth + 1);
        d_ws(d);
        if (d->s[d->p] == ',') { d->p++; continue; }
        d->p++; break;
    }
}
static void d_array(dec *d, int ety, int esub, int tgt, int live, int depth) {
    size_t count = 0;
    d->p++; d_ws(d);
    if (d->s[d->p] == ']') { d->p++; }
    else for (;;) {
        int elive = 0, etgt = 0;
        if (tgt == TG_CHOICES) elive = (count == 0);
        else if (tgt == TG_TOOLCALLS) { elive = live; if (live) { tc_push(d); etgt = 0; } }
        else elive = 0;
        d_value(d, ety, esub, 0, 0, etgt, elive, depth + 1);
        count++;
        d_ws(d);
        if (d->s[d->p] == ',') { d->p++; continue; }
        d->p++; break;
    }
    if (tgt == TG_CHOICES) {
        d->n_choices = (uint32_t)count;
        /* decode.go array(): an empty array sets a fresh slice of capacity 0, so a later "choices" array grows new, zeroed storage */
        if (count == 0) reset_choice0(d);
    }
}
static void d_value(dec *d, int ty, int sub, int ety, int esub, int tgt, int live, int depth) {
    (void)depth;
    d_ws(d);
    uint8_t c = d->s[d->p];
    struct tcent *cur = (d->n_tc > 0) ? &d->tc[d->n_tc - 1] : 0;
    if (c == '{') {
        if (ty == TY_STRUCT || ty == TY_PSTRUCT) {
            if (tgt == TG_USAGE) d->has_usage = 1;
            if (tgt == TG_TC_FUNCTION && live && cur) cur->has_function = 1;
            d_object(d, sub, live, depth);
        } else if (ty == TY_GOOGLE) d_google(d);
        else { if (ty != TY_SKIP) d->type_err = 1; d_skip(d); }
        return;
    }
    if (c == '[') {
        if (ty == TY_SLICE || ty == TY_PSLICE) {
            if (tgt == TG_TOOLCALLS && live) { d->tc_nonnil = 1; d->n_tc = 0; }
            d_array(d, ety, esub, tgt, live, depth);
        } else { if (ty != TY_SKIP) d->type_err = 1; d_skip(d); }
        return;
    }
    if (c == '"') {
        size_t a, b; d_strbody(d, &a, &b);
        if (ty == TY_STR || ty == TY_PSTR) {
            if (live && tgt) {
                unquote(d->s + a, b - a, &d->scratch);
                buf *dst = 0;
                switch (tgt) {
                case TG_CONTENT: dst = &d->content; break;
                case TG_FINISH: d->finish = classify_finish(d->scratch.p, d->scratch.n); break;
                case TG_TC_ID: if (cur) { cur->has_id = 1; dst = &cur->id; } break;
                case TG_TC_TYPE: if (cur) { cur->has_type = 1; dst = &cur->type; } break;
                case TG_NAME: if (cur) dst = &cur->name; break;
                case TG_ARGS: if (cur) dst = &cur->args; break;
                }
                if (dst) { dst->n = 0; buf_put(dst, d->scratch.p, d->scratch.n); }
            }
        } else if (ty != TY_SKIP) d->type_err = 1;
        return;
    }
    if (c == '-' || (c >= '0' && c <= '9')) {
        jscan j = { d->s, d->n, d->p, ORC_MAX_DEPTH, 0 }; js_number(&j);
        const uint8_t *num = d->s + d->p; size_t nn = j.p - d->p;
        d->p = j.p;
        if (ty == TY_INT) {
            int64_t v;
            if (!parse_int64(num, nn, &v)) { d->type_err = 1; return; }
            if (tgt == TG_PROMPT) d->prompt = v;
            else if (tgt == TG_COMPLETION) d->completion = v;
            else if (tgt == TG_TOTAL) d->total = v;
            else if (tgt == TG_TC_INDEX && live && cur) cur->index = v;
        } else if (ty == TY_F32) {
            if (f32_overflows(num, nn)) d->type_err = 1;
        } else if (ty != TY_SKIP) d->type_err = 1;
        return;
    }
    if (c == 't' || c == 'f') {
        d->p += (c == 't') ? 4 : 5;
        if (ty != TY_SKIP) d->type_err = 1;   /* no bool field anywhere in the schema */
        return;
    }
    /* null: literalStore sets pointers/slices/maps to nil, otherwise no-op */
    d->p += 4;
    switch (tgt) {
    case TG_CHOICES: d->n_choices = 0; reset_choice0(d); break;
    case TG_USAGE: d->has_usage = 0; d->prompt = d->completion = d->total = 0; break;
    case TG_TOOLCALLS: if (live) { d->tc_nonnil = 0; d->n_tc = 0; } break;
    case TG_TC_ID: if (live && cur) { cur->has_id = 0; cur->id.n = 0; } break;
    case TG_TC_TYPE: if (live && cur) { cur->has_type = 0; cur->type.n = 0; } break;
    case TG_TC_FUNCTION: if (live && cur) { cur->has_function = 0; cur->name.n = 0; cur->args.n = 0; } break;
    default: break;
    }
}

static _Thread_local dec g_dec; /* reused buffers (per thread) */

uint32_t orc_unmarshal_chunk(orc_result *r, const uint8_t *data, size_t n) {
    r->chunks = (orc_chunk *)xgrow(r->chunks, &r->cap_chunks, r->n_chunks + 1, sizeof(orc_chunk));
    uint32_t idx = (uint32_t)r->n_chunks++;
    orc_chunk *ck = &r->chunks[idx];
    memset(ck, 0, sizeof *ck);
    if (!orc_json_valid(data, n)) return idx;
    dec *d = &g_dec;
    d->s = data; d->n = n; d->p = 0; d->type_err = 0; d->r = r;
    d->n_choices = 0; d->has_usage = 0; d->prompt = d->completion = d->total = 0;
    reset_choice0(d);
    d_ws(d);
    uint8_t c = data[d->p];
    if (c == '{') d_object(d, S_ROOT, 0, 0);
    else if (c == 'n') { /* null into struct: no-op */ }
    else d->type_err = 1;
    if (d->type_err) return idx;
    ck = &r->chunks[idx];
    ck->json_ok = 1;
    ck->n_choices = d->n_choices;
    ck->has_usage = d->has_usage;
    ck->prompt = d->prompt; ck->completion = d->completion; ck->total = d->total;
    if (d->n_choices > 0) {
        ck->finish = d->finish;
        ck->content.off = text_put(r, d->content.p, d->content.n);
        ck->content.len = (uint32_t)d->content.n;
        ck->tool_calls_nonnil = d->tc_nonnil;
        ck->tc_first = (uint32_t)r->n_tcs;
        ck->tc_count = (uint32_t)d->n_tc;
        for (size_t i = 0; i < d->n_tc; i++) {
            struct tcent *t = &d->tc[i];
            r->tcs = (orc_tc *)xgrow(r->tcs, &r->cap_tcs, r->n_tcs + 1, sizeof(orc_tc));
            orc_tc *o = &r->tcs[r->n_tcs++];
            memset(o, 0, sizeof *o);
            o->index = t->index; o->has_id = t->has_id; o->has_type = t->has_type; o->has_function = t->has_function;
            o->id.off = text_put(r, t->id.p, t->id.n); o->id.len = (uint32_t)t->id.n;
            o->type.off = text_put(r, t->type.p, t->type.n); o->type.len = (uint32_t)t->type.n;
            o->name.off = text_put(r, t->name.p, t->name.n); o->name.len = (uint32_t)t->name.n;
            o->args.off = text_put(r, t->args.p, t->args.n); o->args.len = (uint32_t)t->args.n;
            if (t->has_id || (t->has_function && (t->name.n || t->args.n))) ck->has_valid_tool_call = 1;
        }
    }
    return idx;
}

/* ------------------------------------------------------------------ A1: provider.go:308-341 */
typedef void (*line_cb)(void *u, const uint8_t *line, size_t n, size_t off);
static size_t split_lines(const uint8_t *in, size_t n, line_cb cb, void *u) {
    size_t start = 0;
    for (;;) {
        const uint8_t *nl = (const uint8_t *)memchr(in + start, '\n', n - start);
        if (!nl) break;                       /* ReadBytes error (EOF): partial tail discarded */
        size_t end = (size_t)(nl - in) + 1;
        cb(u, in + start, end - start, start);
        start = end;
    }
    return n - start;
}

/* ------------------------------------------------------------------ mode P */
typedef struct { orc_result *r; int parse; } pctx;
static void p_line(void *u, const uint8_t *line, size_t n, size_t off) {
    pctx *c = (pctx *)u;
    orc_line *l = line_new(c->r);
    l->line_off = (uint32_t)off; l->line_len = (uint32_t)n;
    l->kind = ORC_L_EMITTED;
    l->out_off = out_put(c->r, line, n);      /* routes.go:613 w.Write(line) */
    l->out_len = (uint32_t)n;
    if (c->parse && has_prefix(line, n, "data: ")) {
        l->pay_off = (uint32_t)off + 6; l->pay_len = (uint32_t)n - 7;
        uint32_t ci = orc_unmarshal_chunk(c->r, line + 6, n - 7);
        c->r->lines[c->r->n_lines - 1].chunk = ci;
    }
}
void orc_passthrough(orc_result *r, const uint8_t *in, size_t n, int parse) {
    pctx c = { r, parse };
    r->tail_len = split_lines(in, n, p_line, &c);
}

/* ------------------------------------------------------------------ mode R: agent.go:169-248 */
typedef struct { orc_result *r; buf acc; } rctx;
static void r_line(void *u, const uint8_t *line, size_t n, size_t off) {
    rctx *c = (rctx *)u; orc_result *r = c->r;
    orc_line *l = line_new(r);
    l->line_off = (uint32_t)off; l->line_len = (uint32_t)n;
    if (r->terminated) { l->kind = ORC_L_UNREAD; return; }   /* loop exited, :169 */
    size_t a, b;
    orc_trim_space(line, n, &a, &b);                          /* :178-179 */
    const uint8_t *t = line + a; size_t tn = b - a;
    if (contains(t, tn, "[DONE]")) {                          /* :181-184 */
        buf_put(&g_builder, line, n);
        l->kind = ORC_L_DONE;
        /* what parseStreamingToolCalls (:377-402) will see for this builder line */
        const uint8_t *dd = t; size_t dn = tn; int pref = 0;
        if (has_prefix(t, tn, "data: ")) { dd = t + 6; dn = tn - 6; pref = 1; }
        l->pay_off = (uint32_t)(off + (size_t)(dd - line)); l->pay_len = (uint32_t)dn;
        /* A6 breaks only on `data: [DONE]` (:385-396: data == "[DONE]" after the "data: " case); a bare `[DONE]` line
         * takes the switch's default branch (line == "[DONE]" fails case 2) and is skipped, like any unparsable line */
        if (pref && dn == 6 && !memcmp(dd, "[DONE]", 6)) l->kind = ORC_L_DONE_EXACT; /* exact: A6 breaks here */
        else { uint32_t ci = orc_unmarshal_chunk(r, dd, dn); r->lines[r->n_lines - 1].chunk = ci; }
        return;
    }
    if (!has_prefix(t, tn, "data: ")) { l->kind = ORC_L_DROPPED; return; }     /* :186-188 */
    const uint8_t *pay = t + 6; size_t pn = tn - 6;                               /* :190 */
    if (pn == 0) { l->kind = ORC_L_DROPPED; return; }                             /* :191-193 */
    l->kind = ORC_L_EMITTED;                                                      /* :195-197 */
    l->pay_off = (uint32_t)(off + (size_t)(pay - line)); l->pay_len = (uint32_t)pn;
    l->out_off = out_put(r, "data: ", 6); out_put(r, pay, pn); out_put(r, "\n\n", 2);
    l->out_len = (uint32_t)(pn + 8);
    buf_put(&g_builder, r->out + l->out_off, l->out_len);
    uint32_t ci = orc_unmarshal_chunk(r, pay, pn);                                /* :199-203 */
    l = &r->lines[r->n_lines - 1];
    l->chunk = ci;
    orc_chunk *ck = &r->chunks[ci];
    if (!ck->json_ok) return;
    if (ck->n_choices == 0) return;                                               /* :205-207 */
    if (ck->content.len) buf_put(&c->acc, r->text + ck->content.off, ck->content.len); /* :211-222 */
    if (ck->has_valid_tool_call) r->has_tool_calls = 1;                           /* :224-233 */
    if (ck->finish == ORC_FIN_TOOL_CALLS || ck->finish == ORC_FIN_STOP) {         /* :235-242 */
        r->terminated = 1; r->term_finish = ck->finish;
    }
}
void orc_reframe_stream(orc_result *r, const uint8_t *in, size_t n, int append_done) {
    rctx c; memset(&c, 0, sizeof c); c.r = r;
    g_builder.n = 0;
    r->tail_len = split_lines(in, n, r_line, &c);
    r->acc_content.off = text_put(r, c.acc.p, c.acc.n);
    r->acc_content.len = (uint32_t)c.acc.n;
    free(c.acc.p);
    if (append_done) out_put(r, "data: [DONE]\n\n", 14);                          /* :140-143 */
}
const uint8_t *orc_last_builder(const orc_result *r, size_t *n) { (void)r; *n = g_builder.n; return g_builder.p; }

/* ------------------------------------------------------------------ tool-call accumulation */
typedef struct { int64_t index; buf id, type, name, args; } acc_call;
typedef struct { acc_call *v; size_t n, cap; } acc_map;
static acc_call *acc_get(acc_map *m, int64_t index, int create) {
    for (size_t i = 0; i < m->n; i++) if (m->v[i].index == index) return &m->v[i];
    if (!create) return 0;
    size_t oc = m->cap;
    m->v = (acc_call *)xgrow(m->v, &m->cap, m->n + 1, sizeof *m->v);
    memset(m->v + oc, 0, (m->cap - oc) * sizeof *m->v);
    acc_call *c = &m->v[m->n++];
    c->index = index; c->id.n = c->name.n = c->args.n = 0; c->type.n = 0;
    buf_put(&c->type, "function", 8);           /* Type: types.Function */
    return c;
}
static size_t acc_emit(orc_result *r, acc_map *m, orc_call *calls, size_t cap, int require_name) {
    size_t out = 0;
    for (size_t i = 0; i < m->n; i++) {        /* for i := 0; i < len(map); i++ { if map[i] exists */
        acc_call *c = acc_get(m, (int64_t)i, 0);
        if (!c) continue;
        if (require_name && c->name.n == 0) continue;
        if (out < cap) {
            calls[out].id.off = text_put(r, c->id.p, c->id.n); calls[out].id.len = (uint32_t)c->id.n;
            calls[out].type.off = text_put(r, c->type.p, c->type.n); calls[out].type.len = (uint32_t)c->type.n;
            calls[out].name.off = text_put(r, c->name.p, c->name.n); calls[out].name.len = (uint32_t)c->name.n;
            calls[out].args.off = text_put(r, c->args.p, c->args.n); calls[out].args.len = (uint32_t)c->args.n;
        }
        out++;
    }
    for (size_t i = 0; i < m->cap; i++) { free(m->v[i].id.p); free(m->v[i].type.p); free(m->v[i].name.p); free(m->v[i].args.p); }
    free(m->v);
    return out;
}
static void set_buf(buf *b, orc_result *r, orc_span s) { b->n = 0; buf_put(b, r->text + s.off, s.len); }

/* agent.go:377-481 */
size_t orc_parse_tool_calls(orc_result *r, const uint8_t *body, size_t n, orc_call *calls, size_t cap) {
    acc_map m; memset(&m, 0, sizeof m);
    size_t start = 0;
    for (;;) {                                       /* strings.Split(body, "\n") */
        const uint8_t *nl = start <= n ? (const uint8_t *)memchr(body + start, '\n', n - start) : 0;
        size_t end = nl ? (size_t)(nl - body) : n;
        size_t a, b; orc_trim_space(body + start, end - start, &a, &b);     /* :382 */
        const uint8_t *line = body + start + a; size_t ln = b - a;
        const uint8_t *data = 0; size_t dn = 0; int skip = 0;
        if (has_prefix(line, ln, "data: ")) { data = line + 6; dn = ln - 6; }                 /* :386-387 */
        else if (ln != 0 && !(ln == 6 && !memcmp(line, "[DONE]", 6))) { data = line; dn = ln; } /* :388-389 */
        else skip = 1;                                                                        /* :390-392 */
        if (!skip) {
            if ((dn == 6 && !memcmp(data, "[DONE]", 6)) || dn == 0) break;                    /* :394-396 */
            uint32_t ci = orc_unmarshal_chunk(r, data, dn);                                   /* :398-402 */
            orc_chunk *ck = &r->chunks[ci];
            if (ck->json_ok && ck->n_choices > 0 && ck->tool_calls_nonnil) {                  /* :404-406 */
                for (uint32_t i = 0; i < ck->tc_count; i++) {
                    orc_tc *t = &r->tcs[ck->tc_first + i];
                    acc_call *c = acc_get(&m, t->index, 1);                                   /* :409-421 */
                    if (t->has_id) set_buf(&c->id, r, t->id);                                 /* :424-426 */
                    if (t->has_type) set_buf(&c->type, r, t->type);                           /* :428-430 */
                    if (t->has_function) {                                                    /* :432-466 */
                        for (uint32_t k = 0; k < ck->tc_count; k++) {   /* tempResp loop over ALL entries */
                            orc_tc *t2 = &r->tcs[ck->tc_first + k];
                            if (t2->index != t->index) continue;
                            if (t2->name.len) set_buf(&c->name, r, t2->name);
                            if (t2->args.len) buf_put(&c->args, r->text + t2->args.off, t2->args.len);
                        }
                    }
                }
            }
        }
        if (!nl) break;
        start = end + 1;
    }
    return acc_emit(r, &m, calls, cap, 0);
}

/* telemetry.go:190-277 */
size_t orc_telemetry(orc_result *r, const uint8_t *body, size_t n, orc_usage *u, orc_call *calls, size_t cap) {
    /* strings.Split(body, "\n\n"): non-overlapping, left to right */
    size_t *st = 0, *en = 0, np = 0, capp = 0, cape = 0;
    size_t start = 0, i = 0;
    while (i + 1 < n + 0 && n >= 2) {
        if (body[i] == '\n' && body[i + 1] == '\n') {
            st = (size_t *)xgrow(st, &capp, np + 1, sizeof *st); en = (size_t *)xgrow(en, &cape, np + 1, sizeof *en);
            st[np] = start; en[np] = i; np++;
            i += 2; start = i;
        } else i++;
    }
    st = (size_t *)xgrow(st, &capp, np + 1, sizeof *st); en = (size_t *)xgrow(en, &cape, np + 1, sizeof *en);
    st[np] = start; en[np] = n; np++;
    u->prompt = u->completion = u->total = 0;
    size_t first = np > 4 ? np - 4 : 0;                                   /* :195-198 */
    for (size_t k = first; k < np; k++) {                                 /* :200-224 */
        const uint8_t *c = body + st[k]; size_t cn = en[k] - st[k];
        if (cn == 0 || !has_prefix(c, cn, "data: ")) continue;
        c += 6; cn -= 6;
        if (cn == 6 && !memcmp(c, "[DONE]", 6)) continue;
        uint32_t ci = orc_unmarshal_chunk(r, c, cn);
        orc_chunk *ck = &r->chunks[ci];
        if (!ck->json_ok) continue;
        if (ck->has_usage) { u->prompt = ck->prompt; u->completion = ck->completion; u->total = ck->total; }
    }
    acc_map m; memset(&m, 0, sizeof m);
    for (size_t k = 0; k < np; k++) {                                     /* :226-266 */
        const uint8_t *c = body + st[k]; size_t cn = en[k] - st[k];
        if (!has_prefix(c, cn, "data: ")) continue;
        c += 6; cn -= 6;
        if ((cn == 6 && !memcmp(c, "[DONE]", 6)) || cn == 0) continue;
        uint32_t ci = orc_unmarshal_chunk(r, c, cn);
        orc_chunk *ck = &r->chunks[ci];
        if (!ck->json_ok || ck->n_choices == 0 || !ck->tool_calls_nonnil) continue;
        for (uint32_t t_i = 0; t_i < ck->tc_count; t_i++) {
            orc_tc *t = &r->tcs[ck->tc_first + t_i];
            acc_call *a = acc_get(&m, t->index, 1);
            if (t->has_id) set_buf(&a->id, r, t->id);
            if (t->has_function) {
                if (t->name.len) set_buf(&a->name, r, t->name);
                if (t->args.len) buf_put(&a->args, r->text + t->args.off, t->args.len);
            }
        }
    }
    free(st); free(en);
    return acc_emit(r, &m, calls, cap, 1);                                /* :268-274 name != "" */
}
