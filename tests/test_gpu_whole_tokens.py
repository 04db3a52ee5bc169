"""GPU: member keys, string values and digit runs that the decode automaton takes a window at a time, against the oracle.

The decode kernel skips the plain bytes of key and value strings and of digit runs, and resolves a key (and a finish_reason
value) at its end from its bytes through the name table (csrc/sse_tables.h). These documents put those tokens at every window
alignment and every case the name match distinguishes: schema keys in mixed case and in the wrong struct, near misses, long keys,
keys that hash to a known name's slot, escaped and Unicode-folded keys, the case-sensitive google map, finish_reason values, and
numbers of 1-40 digits. Every engine decodes them alone (field-by-field parity, per connection) and among filler lines that put
the launch in each of the 8-, 16- and 32-item decode shapes (digest parity)."""
import functools

import numpy as np
import pytest
import torch

from inference_gateway_b200 import SseEngine, _abi as A
from tests.name_table import hash_mul, name_hash, table_names
from tests.test_gpu_occupancy import ENGINES, TARGET, dealt, filler_payload, parity, shape_check
from tests.util import check_stream, run_streams

pytestmark = pytest.mark.gpu
R, PP = A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE

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


def bodies_of(docs):
    return [b"data: " + d + b"\n\n" for d in docs], np.array([(R, PP)[i % 2] for i in range(len(docs))], dtype=np.uint8)


@pytest.mark.parametrize("engine_name", list(ENGINES))
def test_whole_tokens_field_by_field(engine_name):
    bodies, modes = bodies_of(documents())
    eng = SseEngine(device=0, max_conns=len(bodies) + 16, bytes_per_batch=8 << 20, flags=ENGINES[engine_name])
    try:
        for nb in (1, 3):
            outs = run_streams(eng, bodies, list(modes), n_batches=nb, seed=nb)
            for i, (b, o) in enumerate(zip(bodies, outs)):
                check_stream(b, int(modes[i]), o, label=f"{engine_name} x{nb} doc {i}")
    finally:
        eng.close()


@pytest.mark.parametrize("engine_name", list(ENGINES))
@pytest.mark.parametrize("shape", [8, 16, 32])
def test_whole_tokens_in_each_decode_shape(engine_name, shape):
    sm_count = torch.cuda.get_device_properties(0).multi_processor_count
    docs = documents()
    target = int(TARGET[shape] * sm_count * 32)
    rng = np.random.default_rng(shape)
    assert len(docs) < target
    fill = [filler_payload("strings" if i % 2 else "nostring", int(n)) for i, n in enumerate(rng.integers(40, 700, target - len(docs)))]
    per = docs + fill
    per = [per[i] for i in rng.permutation(len(per))]
    bodies, bounds, _ = dealt([per])
    eng = SseEngine(device=0, max_conns=len(bodies) + 16, bytes_per_batch=96 << 20, n_slots=1, flags=ENGINES[engine_name])
    try:
        log = []
        parity(eng, bodies, PP, bounds, on_batch=shape_check(eng, sm_count, shape, log), label=f"{engine_name} {shape}-item shape")
        assert len(log) == 1
    finally:
        eng.close()
