// sse_tables.h -- lookup tables of the v2 decoder: a byte-class table, the JSON pushdown automaton's transition
// table (scanner.go grammar + utf8.DecodeRune validity), a perfect hash over every struct-tag name of
// providers/types/common_types.go (:271-297,:300-346,:349-371,:384-393,:451-478,:686-698) plus the finish_reason
// values (:33-39), and the (struct, name) -> field table. Built on the host at sse_init, copied to shared memory
// by each CTA. This is the "table-driven field map" of the design: all 11 providers use the identity table
// because the reference forwards OpenAI-compatible chunks unchanged (SURVEY.md section 0).
#pragma once
#include <stdint.h>
#include <string.h>

namespace ssetab {

// ---- automaton states
enum : uint8_t {
    S_VAL = 0, S_ARR0, S_OBJ0, S_KEY, S_COLON, S_AFTO, S_AFTA, S_END,
    S_T1, S_T2, S_T3, S_F1, S_F2, S_F3, S_F4, S_N1, S_N2, S_N3,
    // states >= S_NMINUS are inside a token (number or string); states >= S_KSTR are inside a string
    S_NMINUS, S_NZERO, S_NINT, S_NDOT, S_NFRAC, S_NE, S_NESIGN, S_NEXP,
    S_KSTR, S_KESC, S_KU1, S_KU2, S_KU3, S_KU4,
    S_VSTR, S_VESC, S_VU1, S_VU2, S_VU3, S_VU4,
    S_V8_1, S_V8_2, S_V8_E0, S_V8_ED, S_V8_3, S_V8_F0, S_V8_F4,
    NST
};
// ---- transition outcomes >= A_FIRST are actions
enum : uint8_t {
    A_FIRST = 64,
    A_OPEN_OBJ = 64, A_OPEN_ARR, A_CLOSE_OBJ, A_CLOSE_ARR, A_KEY_END, A_VSTR_END, A_BAD_STAY, A_BAD_REDO,
    A_NUM_END, A_LIT_TRUE, A_LIT_FALSE, A_LIT_NULL, A_ELEM_REDO, A_COMMA_ARR,
    A_ERR = 255
};
// ---- byte classes
enum : uint8_t {
    C_OTHER = 0, C_SPACE, C_WSCTL, C_CTL, C_LBRACE, C_RBRACE, C_LBRACK, C_RBRACK, C_COLON, C_COMMA, C_QUOTE, C_BSLASH,
    C_SLASH, C_MINUS, C_PLUS, C_DOT, C_ZERO, C_DIGIT, C_e, C_E, C_a, C_b, C_f, C_l, C_n, C_r, C_s, C_t, C_u, C_HEXO,
    C_H80, C_H90, C_HA0, C_HC2, C_HE0, C_HE1, C_HED, C_HF0, C_HF1, C_HF4, C_HINV,
    NCLS
};
constexpr uint16_t CLS_ESC = 0x2000, CLS_HI = 0x4000;   // clssym flags: backslash, byte >= 0x80 (>> 13 gives the per-string flag bits)
constexpr int NAME_WORDS = 5, NAME_LEN_MAX = 4 * NAME_WORDS;   // longest name: 20 bytes
constexpr int NHASH_BITS = 7;
constexpr int N_NODES = 17;                // the schema's node count (N_COUNT, sse_common.cuh)
constexpr int NNAMES = 40;
constexpr uint16_t FIELD_VALID = 0x8000;   // field entry: ty | sub << 4 | tgt << 9 | FIELD_VALID

struct DfaTables {
    uint32_t nword[NNAMES][NAME_WORDS];  // name bytes, zero padded
    uint32_t nhash_mul;                  // name_hash multiplier
    uint16_t clssym[256];                // class | CLS_ESC | CLS_HI
    uint8_t  tr[NST * NCLS + 3];         // next state or action
    uint16_t field[N_NODES * NNAMES];    // (node, name) -> packed field
    uint8_t  nhash[1 << NHASH_BITS];     // name_hash slot -> name id (0xFF: empty)
    uint8_t  nlen[NNAMES];               // name length
    uint8_t  finmap[NNAMES];             // name id -> SSE_FIN_* (0xFF: not a finish_reason value)
};

#ifdef __CUDACC__
#define SSETAB_HD __host__ __device__ __forceinline__
#else
#define SSETAB_HD inline
#endif
// Names are looked up by a perfect hash of (first four bytes with ASCII letters lower-cased, length), then compared word by
// word with the folded bytes of the key or finish_reason value.
SSETAB_HD uint32_t name_hash(uint32_t mul, uint32_t w0, uint32_t len) { return (w0 * mul + len * 0x9E3779B1u) >> (32 - NHASH_BITS); }
// w with 'A'..'Z' lower-cased; up collects 0x80 in each byte that was upper-case. Bytes >= 0x80 are left alone.
SSETAB_HD uint32_t fold_ascii4(uint32_t w, uint32_t &up) {
    const uint32_t x = w & 0x7F7F7F7Fu;
    const uint32_t u = (x + 0x3F3F3F3Fu) & ~(x + 0x25252525u) & ~w & 0x80808080u;
    up |= u;
    return w | (u >> 2);
}
// Name id of an n-byte string body with its ASCII letters case-folded (0xFF: none); upper: the body has an ASCII upper-case
// letter. load4(i) gives body bytes i..i+3 as a little-endian word (what lies past the body does not matter). The body has no
// escapes. Names are [a-z_] only, so a match without upper-case letters is an exact match.
template <class Load4>
SSETAB_HD uint32_t name_lookup(const DfaTables &T, uint32_t n, Load4 load4, bool &upper) {
    if (n == 0 || n > (uint32_t)NAME_LEN_MAX) return 0xFFu;
    uint32_t up = 0, w = load4(0u);
    if (n < 4u) w &= (1u << (n * 8u)) - 1u;
    const uint32_t k = fold_ascii4(w, up);
    const uint32_t id = T.nhash[name_hash(T.nhash_mul, k, n)];
    if (id == 0xFFu || T.nlen[id] != n) return 0xFFu;
    uint32_t diff = k ^ T.nword[id][0];
#ifdef __CUDA_ARCH__
    #pragma unroll 1
#endif
    for (uint32_t i = 4; i < n; i += 4u) {
        w = load4(i);
        if (n - i < 4u) w &= (1u << ((n - i) * 8u)) - 1u;
        diff |= fold_ascii4(w, up) ^ T.nword[id][i >> 2];
    }
    upper = up != 0;
    return diff ? 0xFFu : id;
}

struct FieldSrc { uint8_t node; const char *name; uint8_t ty, sub, tgt; };

// Returns 0 on success. `fields` is the schema (node, name, ty, sub, tgt); `fin` maps finish values. Every name is [a-z_]
// and at most NAME_LEN_MAX bytes long.
inline int build_tables(DfaTables &T, const FieldSrc *fields, int n_fields, const char *const *fin_names,
                        const uint8_t *fin_vals, int n_fin) {
    memset(&T, 0, sizeof T);
    // ---------------- byte classes
    for (int c = 0; c < 256; c++) {
        uint8_t k = C_OTHER;
        if (c == ' ') k = C_SPACE;
        else if (c == '\t' || c == '\n' || c == '\r') k = C_WSCTL;
        else if (c < 0x20) k = C_CTL;
        else if (c == '{') k = C_LBRACE; else if (c == '}') k = C_RBRACE;
        else if (c == '[') k = C_LBRACK; else if (c == ']') k = C_RBRACK;
        else if (c == ':') k = C_COLON; else if (c == ',') k = C_COMMA;
        else if (c == '"') k = C_QUOTE; else if (c == '\\') k = C_BSLASH; else if (c == '/') k = C_SLASH;
        else if (c == '-') k = C_MINUS; else if (c == '+') k = C_PLUS; else if (c == '.') k = C_DOT;
        else if (c == '0') k = C_ZERO; else if (c >= '1' && c <= '9') k = C_DIGIT;
        else if (c == 'e') k = C_e; else if (c == 'E') k = C_E; else if (c == 'a') k = C_a; else if (c == 'b') k = C_b;
        else if (c == 'f') k = C_f; else if (c == 'l') k = C_l; else if (c == 'n') k = C_n; else if (c == 'r') k = C_r;
        else if (c == 's') k = C_s; else if (c == 't') k = C_t; else if (c == 'u') k = C_u;
        else if ((c >= 'A' && c <= 'F') || c == 'c' || c == 'd') k = C_HEXO;
        else if (c >= 0x80 && c <= 0x8F) k = C_H80; else if (c >= 0x90 && c <= 0x9F) k = C_H90;
        else if (c >= 0xA0 && c <= 0xBF) k = C_HA0; else if (c >= 0xC2 && c <= 0xDF) k = C_HC2;
        else if (c == 0xE0) k = C_HE0; else if (c == 0xED) k = C_HED; else if (c >= 0xE1 && c <= 0xEF) k = C_HE1;
        else if (c == 0xF0) k = C_HF0; else if (c >= 0xF1 && c <= 0xF3) k = C_HF1; else if (c == 0xF4) k = C_HF4;
        else if (c >= 0x80) k = C_HINV;
        T.clssym[c] = (uint16_t)(k | (k == C_BSLASH ? CLS_ESC : 0) | (k >= C_H80 ? CLS_HI : 0));
    }
    // ---------------- automaton
    auto set = [&](int s, int c, uint8_t v) { T.tr[s * NCLS + c] = v; };
    for (int i = 0; i < NST * NCLS; i++) T.tr[i] = A_ERR;
    const int ws[] = { C_SPACE, C_WSCTL };
    for (int s : { (int)S_VAL, (int)S_ARR0, (int)S_OBJ0, (int)S_KEY, (int)S_COLON, (int)S_AFTO, (int)S_AFTA, (int)S_END })
        for (int c : ws) set(s, c, (uint8_t)s);
    auto value_start = [&](int s, bool redo) {
        auto tgt = [&](int t) { return redo ? (int)A_ELEM_REDO : t; };   // states and actions share one byte of the table
        set(s, C_LBRACE, tgt(A_OPEN_OBJ)); set(s, C_LBRACK, tgt(A_OPEN_ARR));
        set(s, C_QUOTE, tgt(S_VSTR)); set(s, C_MINUS, tgt(S_NMINUS));
        set(s, C_ZERO, tgt(S_NZERO)); set(s, C_DIGIT, tgt(S_NINT));
        set(s, C_t, tgt(S_T1)); set(s, C_f, tgt(S_F1)); set(s, C_n, tgt(S_N1));
    };
    value_start(S_VAL, false);
    value_start(S_ARR0, true);
    set(S_ARR0, C_RBRACK, A_CLOSE_ARR);
    set(S_OBJ0, C_RBRACE, A_CLOSE_OBJ); set(S_OBJ0, C_QUOTE, S_KSTR);
    set(S_KEY, C_QUOTE, S_KSTR);
    set(S_COLON, C_COLON, S_VAL);
    set(S_AFTO, C_COMMA, S_KEY); set(S_AFTO, C_RBRACE, A_CLOSE_OBJ);
    set(S_AFTA, C_COMMA, A_COMMA_ARR); set(S_AFTA, C_RBRACK, A_CLOSE_ARR);
    // strings
    for (int base : { (int)S_KSTR, (int)S_VSTR }) {
        const int STR = base, ESC = base + 1, U1 = base + 2;
        for (int c = 0; c < NCLS; c++) set(STR, c, (uint8_t)STR);
        set(STR, C_WSCTL, A_ERR); set(STR, C_CTL, A_ERR);
        set(STR, C_QUOTE, base == S_KSTR ? A_KEY_END : A_VSTR_END);
        set(STR, C_BSLASH, (uint8_t)ESC);
        for (int c : { (int)C_QUOTE, (int)C_BSLASH, (int)C_SLASH, (int)C_b, (int)C_f, (int)C_n, (int)C_r, (int)C_t }) set(ESC, c, (uint8_t)STR);
        set(ESC, C_u, (uint8_t)U1);
        const int hex[] = { C_ZERO, C_DIGIT, C_e, C_E, C_a, C_b, C_f, C_HEXO };
        for (int k = 0; k < 4; k++) for (int c : hex) set(U1 + k, c, (uint8_t)(k == 3 ? STR : U1 + k + 1));
    }
    // UTF-8 validity inside value strings (utf8.DecodeRune ranges); keys with high bytes take the slow path
    set(S_VSTR, C_HC2, S_V8_1); set(S_VSTR, C_HE0, S_V8_E0); set(S_VSTR, C_HE1, S_V8_2); set(S_VSTR, C_HED, S_V8_ED);
    set(S_VSTR, C_HF0, S_V8_F0); set(S_VSTR, C_HF1, S_V8_3); set(S_VSTR, C_HF4, S_V8_F4);
    for (int c : { (int)C_H80, (int)C_H90, (int)C_HA0, (int)C_HINV }) set(S_VSTR, c, A_BAD_STAY);
    for (int s = S_V8_1; s <= S_V8_F4; s++) for (int c = 0; c < NCLS; c++) set(s, c, A_BAD_REDO);
    for (int c : { (int)C_H80, (int)C_H90, (int)C_HA0 }) { set(S_V8_1, c, S_VSTR); set(S_V8_2, c, S_V8_1); set(S_V8_3, c, S_V8_2); }
    set(S_V8_E0, C_HA0, S_V8_1);
    set(S_V8_ED, C_H80, S_V8_1); set(S_V8_ED, C_H90, S_V8_1);
    set(S_V8_F0, C_H90, S_V8_2); set(S_V8_F0, C_HA0, S_V8_2);
    set(S_V8_F4, C_H80, S_V8_2);
    // numbers
    const int delim[] = { C_SPACE, C_WSCTL, C_COMMA, C_RBRACE, C_RBRACK };
    set(S_NMINUS, C_ZERO, S_NZERO); set(S_NMINUS, C_DIGIT, S_NINT);
    set(S_NZERO, C_DOT, S_NDOT); set(S_NZERO, C_e, S_NE); set(S_NZERO, C_E, S_NE);
    set(S_NINT, C_ZERO, S_NINT); set(S_NINT, C_DIGIT, S_NINT); set(S_NINT, C_DOT, S_NDOT); set(S_NINT, C_e, S_NE); set(S_NINT, C_E, S_NE);
    set(S_NDOT, C_ZERO, S_NFRAC); set(S_NDOT, C_DIGIT, S_NFRAC);
    set(S_NFRAC, C_ZERO, S_NFRAC); set(S_NFRAC, C_DIGIT, S_NFRAC); set(S_NFRAC, C_e, S_NE); set(S_NFRAC, C_E, S_NE);
    set(S_NE, C_PLUS, S_NESIGN); set(S_NE, C_MINUS, S_NESIGN); set(S_NE, C_ZERO, S_NEXP); set(S_NE, C_DIGIT, S_NEXP);
    set(S_NESIGN, C_ZERO, S_NEXP); set(S_NESIGN, C_DIGIT, S_NEXP);
    set(S_NEXP, C_ZERO, S_NEXP); set(S_NEXP, C_DIGIT, S_NEXP);
    for (int s : { (int)S_NZERO, (int)S_NINT, (int)S_NFRAC, (int)S_NEXP }) for (int c : delim) set(s, c, A_NUM_END);
    // literals
    set(S_T1, C_r, S_T2); set(S_T2, C_u, S_T3); set(S_T3, C_e, A_LIT_TRUE);
    set(S_F1, C_a, S_F2); set(S_F2, C_l, S_F3); set(S_F3, C_s, S_F4); set(S_F4, C_e, A_LIT_FALSE);
    set(S_N1, C_u, S_N2); set(S_N2, C_l, S_N3); set(S_N3, C_l, A_LIT_NULL);
    // ---------------- names: hash + field table
    const char *names[NNAMES]; int n_names = 0;
    auto name_id = [&](const char *s) {
        for (int i = 0; i < n_names; i++) if (!strcmp(names[i], s)) return i;
        const size_t n = strlen(s);
        if (n_names >= NNAMES || n == 0 || n > (size_t)NAME_LEN_MAX) return -1;
        for (const char *p = s; *p; p++) if (!((*p >= 'a' && *p <= 'z') || *p == '_')) return -1;
        names[n_names] = s;
        memcpy(T.nword[n_names], s, n);        // little-endian words, as the device loads them
        T.nlen[n_names] = (uint8_t)n;
        return n_names++;
    };
    memset(T.finmap, 0xFF, sizeof T.finmap);
    for (int i = 0; i < n_fields; i++) {
        int id = name_id(fields[i].name);
        if (id < 0) return -1;
        T.field[fields[i].node * NNAMES + id] =
            (uint16_t)(fields[i].ty | (fields[i].sub << 4) | (fields[i].tgt << 9) | FIELD_VALID);
    }
    for (int i = 0; i < n_fin; i++) {
        int id = name_id(fin_names[i]);
        if (id < 0) return -1;
        T.finmap[id] = fin_vals[i];
    }
    // perfect hash: the first odd multiplier under which the names fall into distinct slots
    uint32_t mul = 0x9E3779B1u;
    for (int tries = 0; tries < 100000 && !T.nhash_mul; tries++, mul += 0x632BE5ABu * 2u) {
        memset(T.nhash, 0xFF, sizeof T.nhash);
        bool ok = true;
        for (int i = 0; i < n_names && ok; i++) {
            const uint32_t h = name_hash(mul, T.nword[i][0], T.nlen[i]);
            if (T.nhash[h] != 0xFF) ok = false; else T.nhash[h] = (uint8_t)i;
        }
        if (ok) T.nhash_mul = mul;
    }
    return T.nhash_mul ? 0 : -1;
}

} // namespace ssetab
