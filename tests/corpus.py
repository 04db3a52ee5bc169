"""JSON documents that exercise every decode rule, and a byte-level mutator (shared by CPU and GPU tests)."""
import functools

import numpy as np

from tests.name_table import hash_mul, name_hash, table_names

TRICKY = [
    b'{}', b'null', b' null ', b'[]', b'"x"', b'5', b'true', b'', b' ', b'{', b'}', b'{"a"}', b'{"a":}', b'{"a":1,}',
    b'[1,]', b'{"a":1}}', b'{"a":1} x', b'{"a":01}', b'{"a":-}', b'{"a":1.}', b'{"a":.5}', b'{"a":1e}', b'{"a":1e+}',
    b'{"a":+1}', b'{"a":tru}', b'{"a":nul}', b'{"a":"\\x"}', b'{"a":"\\u12"}', b'{"a":"\\u12g4"}', b'{"a":"\x01"}',
    b'{"a":"\t"}', b'{"a":"\x7f"}', b'{"a":"\xff\xfe"}', b'{"choices":null}', b'{"choices":[]}', b'{"choices":{}}',
    b'{"choices":"x"}', b'{"choices":[null]}', b'{"choices":[1]}', b'{"choices":[{}]}', b'{"choices":[{"delta":null}]}',
    b'{"choices":[{"delta":[]}]}', b'{"choices":[{"delta":{"content":null}}]}', b'{"choices":[{"delta":{"content":5}}]}',
    b'{"choices":[{"delta":{"content":"a","content":"b"}}]}', b'{"choices":[{"delta":{"content":"a","content":null}}]}',
    b'{"Choices":[{"DELTA":{"CONTENT":"x"},"Finish_Reason":"stop"}]}',
    b'{"choice\xc5\xbf":[{"delta":{"content":"long s"}}]}', b'{"to\xe2\x84\xaaen":1,"choices":[{"delta":{"tool_calls":null}}]}',
    b'{"ch\\u006fices":[{"delta":{"c\\u006Fntent":"esc key"}}]}', b'{"choices":[{"delta":{"content":"\\ud83d\\ude00 \\ud83d x \\ude00 \\ud800\\u0041"}}]}',
    b'{"choices":[{"delta":{"content":"bad \xc0\xaf \xed\xa0\x80 \xf4\x90\x80\x80 \xe2\x82"}}]}',
    b'{"choices":[{"delta":{"content":"\\u0000\\b\\f\\n\\r\\t\\/\\\\\\""}}]}',
    b'{"choices":[{"finish_reason":"st\\u006fp"}]}', b'{"choices":[{"finish_reason":"tool_calls"}]}',
    b'{"choices":[{"finish_reason":"length"}]}', b'{"choices":[{"finish_reason":"weird_reason_that_is_long_and_unknown"}]}',
    b'{"choices":[{"finish_reason":""}]}', b'{"choices":[{"finish_reason":null}]}', b'{"choices":[{"finish_reason":7}]}',
    b'{"choices":[{"index":"0"}]}', b'{"choices":[{"index":1.0}]}', b'{"choices":[{"index":1e2}]}', b'{"choices":[{"index":-0}]}',
    b'{"choices":[{"index":9223372036854775807}]}', b'{"choices":[{"index":9223372036854775808}]}',
    b'{"choices":[{"index":-9223372036854775808}]}', b'{"choices":[{"index":-9223372036854775809}]}',
    b'{"created":12345678901234567890}', b'{"created":null}', b'{"created":true}', b'{"id":5}', b'{"id":null}', b'{"model":{}}',
    b'{"usage":null}', b'{"usage":{}}', b'{"usage":[]}', b'{"usage":{"prompt_tokens":1,"completion_tokens":2,"total_tokens":3}}',
    b'{"usage":{"prompt_tokens":"1"}}', b'{"usage":{"prompt_tokens":1},"usage":{"total_tokens":9}}',
    b'{"usage":{"prompt_tokens":1},"usage":null}', b'{"usage":{"PROMPT_TOKENS":7}}',
    b'{"choices":[{"delta":{"tool_calls":[]}}]}', b'{"choices":[{"delta":{"tool_calls":[null]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{}]}}]}', b'{"choices":[{"delta":{"tool_calls":[{"id":""}]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"id":null,"function":null}]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"function":{}}]}}]}', b'{"choices":[{"delta":{"tool_calls":[{"function":{"name":"n"}}]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"function":{"arguments":"{\\"a\\":1}"},"index":3,"type":"function","id":"c"}]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"index":0,"function":{"name":"a"}},{"index":0,"function":{"arguments":"x"}},{"index":-1}]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"index":0}],"tool_calls":[{"index":1},{"index":2}]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"index":0,"id":"a"}],"tool_calls":null}}]}',
    b'{"choices":[{"delta":{"tool_calls":{"index":0}}}]}', b'{"choices":[{"delta":{"tool_calls":[5]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"extra_content":{"google":{"thought_signature":"s","other":[1,{"a":2}]}}}]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"extra_content":{"google":{"thought_signature":5}}}]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"extra_content":{"google":{"thought_signature":5,"thought_signature":"ok"}}}]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"extra_content":{"google":{"Thought_Signature":5}}}]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"extra_content":{"google":[1]}}]}}]}', b'{"choices":[{"delta":{"tool_calls":[{"extra_content":{"google":null}}]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"extra_content":{"GOOGLE":"x"}}]}}]}',
    b'{"choices":[{"logprobs":{"content":[{"token":"a","logprob":-0.5,"bytes":[97],"top_logprobs":[{"token":"b","logprob":-9999.0,"bytes":null}]}],"refusal":null}}]}',
    b'{"choices":[{"logprobs":{"content":[{"logprob":3.4028235e38}]}}]}', b'{"choices":[{"logprobs":{"content":[{"logprob":3.4028236e38}]}}]}',
    b'{"choices":[{"logprobs":{"content":[{"logprob":340282356779733661637539395458142568447}]}}]}',
    b'{"choices":[{"logprobs":{"content":[{"logprob":340282356779733661637539395458142568448}]}}]}',
    b'{"choices":[{"logprobs":{"content":[{"logprob":-1e39}]}}]}', b'{"choices":[{"logprobs":{"content":[{"logprob":1e-400}]}}]}',
    b'{"choices":[{"logprobs":{"content":[{"logprob":0.00000e999}]}}]}', b'{"choices":[{"logprobs":{"content":[{"logprob":"x"}]}}]}',
    b'{"choices":[{"logprobs":{"content":[{"bytes":[1.5]}]}}]}', b'{"choices":[{"logprobs":{"content":{}}}]}',
    b'{"choices":[{"delta":{"content":"first"}},{"delta":{"content":"second","tool_calls":[{"id":"x"}]},"finish_reason":"stop"}]}',
    b'{"choices":[{"delta":{"content":"a"}}],"choices":[{"finish_reason":"stop"}]}',
    b'{"choices":[{"delta":{"content":"a"}}],"choices":null}', b'{"choices":[{"delta":{"content":"a"}}],"choices":[]}',
    # an empty "choices" array is a fresh slice of capacity 0 (decode.go array()): a later array's element 0 starts empty
    b'{"choices":[{"delta":{"content":"a"},"finish_reason":"stop"}],"choices":[],"choices":[{"delta":{}}]}',
    b'{"choices":[{"delta":{"content":"a"},"finish_reason":"stop"}],"choices":[],"choices":null}',
    b'{"choices":[{"delta":{"content":"a"},"finish_reason":"stop"}],"choices":[]}',
    b'{"choices":[{"delta":{"tool_calls":[{"index":0,"id":"c","function":{"name":"f","arguments":"x"}}]},"finish_reason":"tool_calls"}],'
    b'"choices":[ ],"choices":[{"delta":{"content":"b"}}]}',
    b'{"choices":[{"delta":{"content":"a"}}],"choices":[],"choices":[{"finish_reason":"stop"}],"choices":[{"delta":{"content":"c"}}]}',
    b'{"choices":[],"choices":[{"delta":{"content":"b"},"finish_reason":"stop"}]}',
    b'{"unknown":{"deep":[1,2,{"x":[true,false,null,"s",1.5e-3]}]},"choices":[{"delta":{"content":"ok"}}]}',
    b'\t\r\n {"choices" : [ { "delta" : { "content" : "ws" } , "finish_reason" : null } ] } \r',
    b"[" * 128 + b"]" * 128, b"[" * 129 + b"]" * 129, b'{"a":' * 100 + b"1" + b"}" * 100,
    b'{"choices":[{"delta":{"role":"assistant","content":null,"reasoning":5}}]}', b'{"system_fingerprint":false}',
    b'{"reasoning_format":"raw","choices":[{"delta":{"reasoning_content":"r","refusal":null,"content":"c"}}]}',
]


def mutate(rng, doc: bytes) -> bytes:
    b = bytearray(doc)
    if not b:
        return bytes(b)
    for _ in range(int(rng.integers(1, 4))):
        op = int(rng.integers(0, 6))
        i = int(rng.integers(0, len(b)))
        if op == 0:
            b[i] = int(rng.integers(0x20, 0x7F))
        elif op == 1:
            del b[i]
        elif op == 2:
            alphabet = b'{}[]:,"\\0123456789.eE-+ tfn'
            b.insert(i, alphabet[int(rng.integers(0, len(alphabet)))])
        elif op == 3 and len(b) > 2:
            j = int(rng.integers(0, len(b)))
            b[i], b[j] = b[j], b[i]
        elif op == 4:
            b[i] = int(rng.integers(0x80, 0x100))
        else:
            b[i:i] = b'\\u00' + b'%02x' % int(rng.integers(0, 256))
        if not b:
            break
    return bytes(b).replace(b"\n", b" ")


# ------------------------------------------------------------------ strings at every alignment
# One string per document, in each field the decoder captures. The decode stage skips plain string bytes 16 at a time, a
# lane at most 4 windows (64 bytes) per round, a whole warp 512 bytes per step, and unquotes in 32-byte steps; its item sort
# puts every payload of 4,064 bytes or more in one bucket.
STRING_FIELDS = {
    "content": b'{"choices":[{"index":0,"delta":{"content":"%s"},"finish_reason":null}]}',
    "id": b'{"choices":[{"index":0,"delta":{"tool_calls":[{"index":0,"id":"%s","type":"function","function":{"name":"f","arguments":""}}]}}]}',
    "name": b'{"choices":[{"index":0,"delta":{"tool_calls":[{"index":0,"id":"c","type":"function","function":{"name":"%s","arguments":""}}]}}]}',
    "arguments": b'{"choices":[{"index":0,"delta":{"tool_calls":[{"index":0,"function":{"arguments":"%s"}}]}}]}',
    "finish_reason": b'{"choices":[{"index":0,"delta":{},"finish_reason":"%s"}]}',
    "thought_signature": b'{"choices":[{"index":0,"delta":{"tool_calls":[{"index":0,"id":"c","extra_content":{"google":{"thought_signature":"%s"}}}]}}]}',
}
STRING_LENGTHS = (16, 32, 64, 512, 4096, 8192)
# what stands at offset k of the string: None = the closing quote, b"EOF" = the payload ends there, anything else is inserted
STRING_EVENTS = (
    None, b"EOF",
    b"\\\\", b'\\"', b"\\n", b"\\u00e9",
    b"\\ud83d\\ude00", b"\\ud83d", b"\\ude00",                        # a pair, a lone high and a lone low surrogate
    "é".encode(), "漢".encode(), "😀".encode(),                         # raw UTF-8 of 2, 3 and 4 bytes
    b"\xe6\xbc", b"\xc0\xaf", b"\xed\xa0\x80", b"\xf4\x90\x80\x80",   # truncated, overlong, surrogate-encoded, above U+10FFFF
    b"\x01", b"\x1f", b"\x7f",                                        # raw control bytes (invalid JSON), and DEL (valid)
)


def _plain(n: int) -> bytes:
    from inference_gateway_b200.synth import _WORDS
    words = b" ".join(w.encode() for w in _WORDS)
    return (words * (n // len(words) + 1))[:n]


def string_offsets(length: int) -> list:
    """Offsets k of the event in a string of about `length` bytes: 0-33, 480-544 and the last 33 bytes. The 480-544 band is
    left out at 8,192, where it repeats what 4,096 puts there."""
    ks = set(range(34)) | set(range(max(0, length - 33), length + 1))
    if length < 8192:
        ks |= set(range(480, 545))
    return sorted(k for k in ks if k <= length)


def string_alignment_docs() -> list:
    """Deterministic: every event of STRING_EVENTS at every offset of string_offsets(L), for each L of STRING_LENGTHS; the
    field cycles through STRING_FIELDS so that each of them sees every event and every length."""
    plain = _plain(max(STRING_LENGTHS) + 64)
    fields = list(STRING_FIELDS.values())
    docs = []
    for li, length in enumerate(STRING_LENGTHS):
        for ei, ev in enumerate(STRING_EVENTS):
            for k in string_offsets(length):
                tpl = fields[(li + ei + k) % len(fields)]
                if ev is None:
                    docs.append(tpl % plain[:k])
                elif ev == b"EOF":
                    docs.append(tpl[:tpl.index(b"%s")] + plain[:k])
                else:
                    docs.append(tpl % (plain[:k] + ev + plain[k:max(k, length - len(ev))]))
    return docs


# ------------------------------------------------------------------ skeleton-template near-misses
# A template is a learnt line with its string bodies and integers cut out (wildcards); a line replays it when everything else
# is byte for byte the same and every wildcard is again a well-formed string body or integer. The variants below differ from
# a canonical chunk in one place; whichever way the decoder takes them, the record must be the reference's.
STRING_VARIANTS = (b"a\\nb", "café".encode(), b"\xff", b"x\x01y", b"5", b"null", b"{}")        # unterminated: built apart
INT_VARIANTS = (b"01", b"-0", b"-", b"1.0", b"1e2", b"9223372036854775807", b"9223372036854775808",
                b"-9223372036854775808", b"-9223372036854775809", b"12345678901234567890", b'"1"')


def _wildcards(doc: bytes) -> list:
    """(start, end, kind) of every string value and integer of a JSON document outside strings; a string's span includes
    its quotes."""
    out, i, n = [], 0, len(doc)
    prev = b""                                  # last significant byte outside strings
    while i < n:
        c = doc[i:i + 1]
        if c == b'"':
            j = i + 1
            while doc[j:j + 1] != b'"':
                j += 2 if doc[j:j + 1] == b"\\" else 1
            if prev in (b":", b"["):
                out.append((i, j + 1, "str"))
            elif prev == b"," and _in_array(doc, i):
                out.append((i, j + 1, "str"))
            prev = b'"'
            i = j + 1
        elif c in b"-0123456789":
            j = i + 1
            while j < n and doc[j:j + 1] in b"0123456789.eE+-":
                j += 1
            if all(ch in b"-0123456789" for ch in doc[i:j]):
                out.append((i, j, "int"))
            prev = b"0"
            i = j
        else:
            if c not in b" \t\r\n":
                prev = c
            i += 1
    return out


def _in_array(doc: bytes, i: int) -> bool:
    depth = 0
    for j in range(i - 1, -1, -1):
        ch = doc[j:j + 1]
        if ch in b"]}":
            depth += 1
        elif ch in b"[{":
            if depth == 0:
                return ch == b"["
            depth -= 1
    return False


def canonical_chunks() -> list:
    """Deterministic: every data payload of one synth stream per flavour, with tool-call chunks and a usage chunk."""
    from inference_gateway_b200.synth import MODELS, StreamSpec, Synth
    g = Synth(0x7E3)
    out = []
    for fl in MODELS:
        for tool in (0, 5):
            body, _ = g.stream(StreamSpec(flavour=fl, n_content=4, tool_run=tool, usage_chunk=True, with_done=False))
            out += [ev[6:] for ev in body.split(b"\n\n") if ev.startswith(b"data: {")]
    return out


def template_near_misses() -> tuple:
    """Deterministic: (canonical chunks, near-misses). Per wildcard of every canonical chunk: string bodies with an escape,
    non-ASCII, invalid UTF-8, a control byte, left unterminated, or a number / null / object in their place; integers with a
    leading zero, -0, a lone '-', a fraction, an exponent, int64 max / max+1 / min / min-1, 20 digits or a string; the line cut
    just before and just after the wildcard. Per chunk: the first occurrence of a key name with another case or a Unicode
    folding (K = Kelvin sign, ſ = long s) -- that is the value in "finish_reason":"tool_calls", which must then compare
    exactly --, a duplicated key, extra whitespace, and a key changed in the middle so the line keeps its last two bytes."""
    canon = canonical_chunks()
    miss = []
    for doc in canon:
        for s, e, kind in _wildcards(doc):
            if kind == "str":
                miss += [doc[:s + 1] + v + doc[e - 1:] for v in STRING_VARIANTS[:4]]
                miss += [doc[:s] + v + doc[e:] for v in STRING_VARIANTS[4:]]
                miss.append(doc[:e - 1] + doc[e:])                       # the closing quote is gone
            else:
                miss += [doc[:s] + v + doc[e:] for v in INT_VARIANTS]
            miss += [doc[:s], doc[:e]]
        keys = [(m, m + len(k)) for k in (b'"index"', b'"content"', b'"choices"', b'"id"', b'"tool_calls"', b'"arguments"',
                                          b'"prompt_tokens"', b'"finish_reason"') for m in [doc.find(k)] if m >= 0]
        for s, e in keys:
            key = doc[s:e]
            miss.append(doc[:s] + key.upper() + doc[e:])
            if b"k" in key:
                miss.append(doc[:s] + key.replace(b"k", "K".encode(), 1) + doc[e:])
            if b"s" in key:
                miss.append(doc[:s] + key.replace(b"s", "ſ".encode(), 1) + doc[e:])
            # the key and its value once more, right behind it
            v = next(((a, b) for a, b, _ in _wildcards(doc) if a > e), None)
            if v is not None and doc[e:v[0]].strip() == b":":
                miss.append(doc[:v[1]] + b"," + doc[s:v[1]] + doc[v[1]:])
            miss.append(doc[:e] + b" " + doc[e:])
        miss.append(doc[:-1] + b" " + doc[-1:])
        # a letter of a key, the one nearest the middle, replaced
        wild = _wildcards(doc)
        letters = [i for i in range(len(doc)) if chr(doc[i]).isalpha() and not any(s <= i < e for s, e, _ in wild)]
        m = min(letters, key=lambda i: abs(i - len(doc) // 2))
        miss.append(doc[:m] + (b"y" if doc[m:m + 1] == b"x" else b"x") + doc[m + 1:])
    return canon, miss


# ------------------------------------------------------------------ nesting at the 128-level limit (DESIGN.md §5, deviation 2)
NEST_DEPTHS = (127, 128, 129, 130)
# (name, text before the nested value, text after it, containers open around it)
NEST_PLACES = [
    ("top", b"", b"", 0),
    ("unknown_key", b'{"choices":[{"delta":{"content":"x"}}],"unknown":', b"}", 1),
    ("content", b'{"choices":[{"delta":{"content":', b"}}]}", 4),
    ("arguments", b'{"choices":[{"delta":{"tool_calls":[{"index":0,"function":{"name":"f","arguments":', b"}}]}}]}", 7),
    ("usage", b'{"choices":[],"usage":{"prompt_tokens":1,"x":', b"}}", 2),
    ("finish_reason", b'{"choices":[{"delta":{},"finish_reason":', b"}]}", 3),
]


def nest_kinds(n: int, pattern: str) -> list:
    """Container kinds ('[' or '{') of n nested levels: all arrays, all objects, alternating, or seeded random."""
    if pattern == "arr":
        return ["["] * n
    if pattern == "obj":
        return ["{"] * n
    if pattern == "alt":
        return ["[{"[i & 1] for i in range(n)]
    rng = np.random.default_rng(n)
    return ["[{"[int(b)] for b in rng.integers(0, 2, size=n)]


def _open(k: str) -> bytes:
    return b"[" if k == "[" else b'{"k":'


def _close(k: str) -> bytes:
    return b"]" if k == "[" else b"}"


def nested(kinds, leaf: bytes = b"1") -> bytes:
    return b"".join(_open(k) for k in kinds) + leaf + b"".join(_close(k) for k in reversed(kinds))


def nesting_docs() -> list:
    """Payloads around the nesting limit: (name, payload, shallow twin). The twin has the payload's text with the nested value
    shallow, so a template engine has seen the line's shape when the deep one comes.
    - every depth of NEST_DEPTHS at top level, under an unknown key and inside each captured field, in four kinds of nesting;
      brackets inside a string at those depths (they do not count);
    - each depth with a syntax error just before and just after the 129th opener;
    - a mismatched closer at every depth 1-129, where the nesting opens to that depth, and where it opens to 128 and closes
      down to it, so both 64-bit words of the container-type stack and their boundary are read;
    - the same behind a 4,208-byte string, so the deep part starts after many 16-byte windows and a long-string skip."""
    out = []
    long_head = b'{"choices":[{"delta":{"content":"' + b"abcdefghijklmnop" * 263 + b'"}}],"x":'
    for d in NEST_DEPTHS:
        for name, pre, post, around in NEST_PLACES:
            for pat in ("arr", "obj", "alt", "rnd"):
                kinds = nest_kinds(d - around, pat)
                out.append((f"{name}-{pat}-d{d}", pre + nested(kinds) + post, pre + nested(kinds[:2]) + post))
        s = b'{"choices":[{"delta":{"content":"' + b"[{" * d + b'"}}]}'
        out.append((f"in_string-d{d}", s, b'{"choices":[{"delta":{"content":"[{"}}]}'))
        for where in ("before", "after"):
            kinds = nest_kinds(d, "alt")
            at = 128 if where == "before" else min(129, d)         # openers before the bad byte
            body = b"".join(_open(k) for k in kinds[:at]) + b"\x01" + b"".join(_open(k) for k in kinds[at:]) + b"1" + \
                b"".join(_close(k) for k in reversed(kinds))
            out.append((f"syntax_{where}-d{d}", body, nested(kinds[:2])))
            out.append((f"syntax_{where}-long-d{d}", long_head + body + b"}", long_head + nested(kinds[:2]) + b"}"))
    for k in range(1, 130):
        for pat in ("alt", "rnd"):
            kinds = nest_kinds(k, pat)
            wrong = b"}" if kinds[-1] == "[" else b"]"
            # opens to depth k and closes level k with the other closer
            inner = b"".join(_open(x) for x in kinds) + b"1" + wrong + b"".join(_close(x) for x in reversed(kinds[:-1]))
            # opens to 128, closes down to level k + 1, then level k with the other closer
            full = nest_kinds(128, pat)[:k - 1] + kinds[-1:] + nest_kinds(128 - k, "obj") if k <= 128 else None
            docs = [("open", inner)]
            if full is not None:
                wrong = b"}" if full[k - 1] == "[" else b"]"
                docs.append(("deep", b"".join(_open(x) for x in full) + b"1" + b"".join(_close(x) for x in reversed(full[k:])) +
                             wrong + b"".join(_close(x) for x in reversed(full[:k - 1]))))
            for how, body in docs:
                out.append((f"mismatch_{how}-{pat}-k{k}", body, nested(kinds[:1])))
                out.append((f"mismatch_{how}-long-{pat}-k{k}", long_head + body + b"}", long_head + nested(kinds[:1]) + b"}"))
    return out


# ------------------------------------------------------------------ whole streams of mutated documents
def adversarial_bodies(rng, n):
    out = []
    for k in range(n):
        docs = [TRICKY[int(rng.integers(0, len(TRICKY)))] for _ in range(int(rng.integers(4, 40)))]
        docs = [mutate(rng, d) if rng.random() < 0.4 else d for d in docs]
        sep = [b"\n\n", b"\n", b"\r\n\r\n", b"\n: ping\n\n"][k % 4]
        out.append(b"".join(b"data: " + d + sep for d in docs) + (b"data: [DONE]\n\n" if k % 3 else b"data: {\"tail"))
    return out


# ------------------------------------------------------------------ member keys, values and digit runs (test_gpu_whole_tokens)
# a document with KEY: VALUE inside each struct of the schema
CONTEXTS = [
    b'{"%s":%s,"choices":[{"index":0,"delta":{"content":"x"}}]}',
    b'{"choices":[{"%s":%s,"delta":{"content":"x"}}]}',
    b'{"choices":[{"delta":{"%s":%s}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"%s":%s}]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"index":0,"function":{"%s":%s}}]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"extra_content":{"%s":%s}}]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"extra_content":{"google":{"%s":%s}}}]}}]}',
    b'{"usage":{"%s":%s},"choices":[]}',
    b'{"choices":[{"logprobs":{"%s":%s}}]}',
    b'{"choices":[{"logprobs":{"content":[{"%s":%s}]}}]}',
    b'{"choices":[{"logprobs":{"content":[{"top_logprobs":[{"%s":%s}]}]}}]}',
]
VALUES = [b'"v"', b'7', b'null', b'{"content":"c"}', b'[{"index":1}]', b'-2.5e3', b'"stop"', b'true']


def cases(name: str):
    return {name, name.upper(), name.title(), "".join(c.upper() if i % 2 else c for i, c in enumerate(name)),
            "".join(c.upper() if i % 2 == 0 else c for i, c in enumerate(name))}


def colliding_keys(names, per_name=2):
    """[a-z_] keys of a known name's length that hash to its slot and are not a name."""
    mul, rng, known, out = hash_mul(names), np.random.default_rng(5), set(names), []
    slot = {name_hash(mul, n.encode()): n for n in names}
    for n in names:
        want, got = name_hash(mul, n.encode()), 0
        for _ in range(200000):
            k = "".join(rng.choice(list("abcdefghijklmnopqrstuvwxyz_"), len(n)))
            if k not in known and name_hash(mul, k.encode()) == want:
                out.append(k); got += 1
                if got == per_name:
                    break
    assert len(out) >= len(names) and all(name_hash(mul, k.encode()) in slot for k in out)
    return out


def numbers():
    digits = "1234567890" * 4
    out = []
    for n in range(1, 41):
        d = digits[:n]
        out += [d, "-" + d, "0" + d, d + ".5", d + "." + d, d + "e" + d[:3], d + "E-7", "-" + d + ".25e+12", "0." + d]
    return out + ["0", "-0", "00", "-", "1.", "1e", "1e+"]


@functools.lru_cache(None)
def documents():
    names = table_names()
    docs = []
    keys = {k for n in names for k in cases(n)}
    for n in names:                                                       # near misses of every name
        keys |= {n[:-1], n + "s", n + "_", "x" + n, n[1:], n[:-1] + n[-1].upper() + "x"}
    keys |= {"", "conten", "contents", "finish_reason_", "a" * 17, "b" * 40, "finish_reason" * 6, "thought_signature_x" * 4}
    keys |= set(colliding_keys(names))
    for k in sorted(keys):
        for i, ctx in enumerate(CONTEXTS):
            docs.append(ctx % (k.encode(), VALUES[(len(k) + i) % len(VALUES)]))
    for pad in range(16):                                                 # keys crossing a window at every alignment
        for k in ("choices", "finish_reason", "system_fingerprint", "Reasoning_Content", "a" * 33, "unknown_key_name"):
            docs.append(b'{"id":"%s","%s":1,"choices":[{"delta":{"content":"y"},"finish_reason":"stop"}]}' % (b"x" * pad, k.encode()))
            docs.append(b'%s{"%s":{},"choices":[{"delta":{"content":"%s"}}]}' % (b" " * pad, k.encode(), b"z" * pad))
    for k in (b"\\u0063ontent", b"cont\\u0065nt", b"CONT\\u0045NT", b"con\\ttent", b"\\u0063", b"choice\\u017f", b"choice\xc5\xbf",
              b"to\xe2\x84\xaaen", b"to\\u212aen", b"\\u212A", b"finish_reason\\u0000", b"Finish_Reason\xc2\xa0", b"fin\\/ish"):
        for ctx in CONTEXTS:
            docs.append(ctx % (k, b'"v"'))
    for k in (b"thought_signature", b"Thought_signature", b"THOUGHT_SIGNATURE", b"thought_signaturE", b"thought\\u005fsignature"):
        for v in (b'"sig"', b'5', b'null'):
            docs.append(b'{"choices":[{"delta":{"tool_calls":[{"extra_content":{"google":{"%s":%s}}}]}}]}' % (k, v))
    fins = set()
    for f in ("stop", "tool_calls", "length", "content_filter", "function_call"):
        fins |= cases(f) | {f[:-1], f + "s", f + " "}
    fins |= {"", "st\\u006fp", "\\u0073top", "STO\\u0050", "stop\\n", "tool_c\\u0061lls", "st\xc3\xb6p", "x" * 40, "choices"}
    for f in sorted(fins):
        for pad in range(4):
            docs.append(b'{"choices":[{"index":0,"delta":{"content":"%s"},"finish_reason":"%s"}]}' % (b"p" * pad, f.encode()))
    for i, num in enumerate(numbers()):                                   # digit runs at every alignment, every ending
        num, pad = num.encode(), b" " * (i % 16)
        docs += [b'{"created":%s%s}' % (pad, num), b'{"created":%s%s,"choices":[]}' % (pad, num), pad + num,
                 b'{"usage":{"prompt_tokens":%s%s},"choices":[]}' % (pad, num),
                 b'{"choices":[{"index":%s,"logprobs":{"content":[{"logprob":%s%s,"bytes":[%s,%s]}]}}]}' % (num, pad, num, num, num),
                 b'{"x_unknown":[%s%s],"choices":[{"delta":{"tool_calls":[{"index":%s}]}}]}' % (pad, num, num)]
    return docs
