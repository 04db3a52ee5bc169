/*
 * sse_oracle.h -- CPU restatement of inference-gateway v0.24.0's streaming-response path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product: only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load it.
 *
 * PARITY STATUS: "parity unpinned" at byte level.  The reference is pure Go and no Go
 * toolchain exists in this image (SURVEY.md section 8c), so the reference cannot be executed
 * here.  This restatement follows the reference source line by line (citations below, all
 * relative to /root/reference) plus the published behaviour of the Go 1.26 stdlib calls it
 * makes (bufio.ReadBytes, strings.TrimSpace/Contains/HasPrefix/TrimPrefix/Split,
 * fmt.Sprintf, encoding/json.Unmarshal v1).  It is pinned by:
 *   - the reference's own SSE fixtures and the semantic assertions its tests make on them
 *     (tests/golden/ref_fixtures.json, produced by tools/make_golden.py, which also audits that every
 *     string literal holding SSE bytes in the reference's *_test.go files is one of the fixtures),
 *   - SURVEY.md Appendix B hand-derived vectors,
 *   - a cross-check of the JSON validator/decoder against CPython's json module and an
 *     independent Python model of the typed decode (tests/go_model.py, tests/test_oracle_json.py),
 *   - an independent Python model of everything above the decoder -- TrimSpace, the agent
 *     iteration, parseStreamingToolCalls, telemetry (tests/go_stream_model.py,
 *     tests/test_oracle_stream_model.py).
 * None of these is a run of the Go code: tools/check_go_dump.py + baseline/go/ is the byte-level
 * check for a machine that has Go.
 *
 * Functions and the reference code they restate:
 *   orc_split_lines       providers/core/provider.go:308-341 (ReadBytes('\n'), tail dropped)
 *   orc_passthrough       provider.go:308-341 -> api/routes.go:600-625 / :178-231 (mode P)
 *   orc_unmarshal_chunk   encoding/json.Unmarshal into types.CreateChatCompletionStreamResponse
 *                         (providers/types/common_types.go:271-297,:300-346,:384-393,:451-478,
 *                          :686-698,:835-862)
 *   orc_reframe_stream    mcp/agent.go:169-248 (+ :140-143 final [DONE]) (mode R)
 *   orc_parse_tool_calls  mcp/agent.go:377-481
 *   orc_telemetry         api/middlewares/telemetry.go:190-277
 */
#ifndef SSE_ORACLE_H
#define SSE_ORACLE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* finish_reason classes (types.FinishReason, common_types.go:33-39) */
enum { ORC_FIN_NONE = 0, ORC_FIN_STOP = 1, ORC_FIN_TOOL_CALLS = 2, ORC_FIN_LENGTH = 3,
       ORC_FIN_CONTENT_FILTER = 4, ORC_FIN_FUNCTION_CALL = 5, ORC_FIN_OTHER = 7 };

/* A decoded string lives in the result's text blob. */
typedef struct { uint32_t off, len; } orc_span;

typedef struct {
    int64_t  index;          /* ChatCompletionMessageToolCallChunk.Index */
    uint32_t has_id;         /* ID != nil */
    uint32_t has_type;       /* Type != nil */
    uint32_t has_function;   /* Function != nil */
    uint32_t pad;
    orc_span id, type, name, args;
} orc_tc;

typedef struct {
    uint32_t json_ok;        /* json.Unmarshal returned nil */
    uint32_t n_choices;      /* len(resp.Choices) */
    uint32_t finish;         /* ORC_FIN_* of choices[0].finish_reason */
    uint32_t has_usage;      /* resp.Usage != nil */
    int64_t  prompt, completion, total;
    orc_span content;        /* choices[0].delta.content, decoded */
    uint32_t tool_calls_nonnil; /* choices[0].delta.tool_calls != nil */
    uint32_t tc_first, tc_count; /* into result tcs[] */
    uint32_t has_valid_tool_call; /* agent.go:224-233 predicate */
} orc_chunk;

/* One event per input line for the line-oriented consumers. */
typedef struct {
    uint32_t line_off, line_len;   /* input line incl. '\n' */
    uint32_t out_off, out_len;     /* emitted bytes in out[] (0 len: nothing emitted) */
    uint32_t kind;                 /* ORC_L_* */
    uint32_t chunk;                /* index into chunks[] or 0xFFFFFFFF */
    uint32_t pay_off, pay_len;     /* input bytes handed to orc_unmarshal_chunk (when chunk != 0xFFFFFFFF, and for a
                                      DONE_EXACT line the "[DONE]" it did not decode) */
} orc_line;

enum { ORC_L_DROPPED = 0,     /* R: not "data: "-prefixed / empty payload */
       ORC_L_EMITTED = 1,     /* P: every line; R: frame emitted */
       ORC_L_DONE = 2,        /* R: swallowed, Contains "[DONE]" (agent.go:181-184) */
       ORC_L_UNREAD = 3,      /* R: after the terminating chunk (agent.go:235-242) */
       ORC_L_DONE_EXACT = 4 };/* R: swallowed, and the payload is exactly "[DONE]" (agent.go:394-396 breaks on it) */

typedef struct {
    uint8_t  *out;     size_t out_len,  out_cap;
    uint8_t  *text;    size_t text_len, text_cap;
    orc_line *lines;   size_t n_lines,  cap_lines;
    orc_chunk*chunks;  size_t n_chunks, cap_chunks;
    orc_tc   *tcs;     size_t n_tcs,    cap_tcs;
    /* stream-level results */
    orc_span acc_content;       /* agent.go:211-222 accumulated content */
    uint32_t has_tool_calls;    /* agent.go:224-233 */
    uint32_t terminated;        /* finish_reason stop/tool_calls seen */
    uint32_t term_finish;
    size_t   tail_len;          /* unterminated tail dropped by provider.go:323-330 */
} orc_result;

orc_result *orc_result_new(void);
void orc_result_free(orc_result *r);
void orc_result_clear(orc_result *r);

/* strings.TrimSpace: returns [*a,*b) */
void orc_trim_space(const uint8_t *s, size_t n, size_t *a, size_t *b);
/* encoding/json checkValid: 1 valid, 0 invalid */
int orc_json_valid(const uint8_t *s, size_t n);
/* checkValid with a nesting limit, and why it stopped: ORC_JSON_DEPTH when the scan opens a container while max_depth are
 * open, before the document's first syntax error. max_depth 128 restates the product's documented limit (DESIGN.md §5,
 * deviation 2: such a line is reported not JSON_OK and flagged SSE_F_DEPTH_LIMIT); Go's own limit is 10000. */
enum { ORC_JSON_OK = 0, ORC_JSON_SYNTAX = 1, ORC_JSON_DEPTH = 2 };
#define ORC_DEPTH_LIMIT 128
int orc_json_scan(const uint8_t *s, size_t n, int max_depth);

/* json.Unmarshal(data, &CreateChatCompletionStreamResponse); appends one orc_chunk. */
uint32_t orc_unmarshal_chunk(orc_result *r, const uint8_t *data, size_t n);

/* Mode P: provider.go:308-341 + routes.go:600-625. parse!=0 additionally decodes each line that
 * starts with "data: " (payload = line[6:len-1]) so the telemetry fold can be checked per line. */
void orc_passthrough(orc_result *r, const uint8_t *in, size_t n, int parse);

/* Mode R: provider.go:308-341 + agent.go:169-248 for ONE agent iteration (one upstream stream).
 * append_done!=0 appends the final "data: [DONE]\n\n" of agent.go:140-143. */
void orc_reframe_stream(orc_result *r, const uint8_t *in, size_t n, int append_done);

/* agent.go:377-481 over the iteration's responseBodyBuilder text. Results -> r->tcs
 * (merged calls, ordered as the reference orders them). Returns count. */
typedef struct { orc_span id, type, name, args; } orc_call;
size_t orc_parse_tool_calls(orc_result *r, const uint8_t *body, size_t n, orc_call *calls, size_t cap);

/* telemetry.go:190-277 over a whole response body. */
typedef struct { int64_t prompt, completion, total; } orc_usage;
size_t orc_telemetry(orc_result *r, const uint8_t *body, size_t n, orc_usage *u, orc_call *calls, size_t cap);

/* responseBodyBuilder text of the last orc_reframe_stream call (agent.go:156,:182,:197). */
const uint8_t *orc_last_builder(const orc_result *r, size_t *n);

#ifdef __cplusplus
}
#endif
#endif
