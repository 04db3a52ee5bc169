"""CPU: the C oracle (oracle/sse_oracle.c) against an independent Python model of the streaming path
(tests/go_stream_model.py + tests/go_model.py): line splitting, strings.TrimSpace, the agent iteration of mcp/agent.go:169-248,
parseStreamingToolCalls (:377-481) and telemetry.go:190-277 -- on the reference's fixtures, the synthetic workloads and
adversarial streams (unicode spaces, invalid UTF-8 around the trim, "[DONE]" anywhere, non-data lines, CRLF, duplicate
tool-call indices, data after the terminating chunk)."""
import json
import os

import numpy as np

from inference_gateway_b200 import synth
from oracle import orc
from tests import go_stream_model as sm
from tests.corpus import TRICKY

GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "ref_fixtures.json")))["fixtures"]

SPACES = [b"", b" ", b"\t", b"\r", b"\x0b\x0c"] + [c.encode() for c in (
    "", " ", " ", " ", " ", " ", " ", " ", " ", " ", "　",
    "​", "﻿", "᠎")] + [      # the last three are NOT spaces for Go
    b"\xc2", b"\xe2\x80", b"\xa0", b"\x85", b"\xe3\x80\x80\x80", b"\xff", b"\xed\xa0\x80", b"\xc0\xa0", b"\xe2\x80\xa8\xe2"]
PAYLOADS = [d for d in TRICKY if b"\n" not in d] + [
    b'{"choices":[{"delta":{"content":"a"}}]}', b'{"choices":[{"delta":{"content":"say [DONE]"}}]}', b"[DONE]", b" [DONE]", b"x[DONE]y",
    b'{"choices":[{"delta":{},"finish_reason":"stop"}]}', b'{"choices":[{"delta":{},"finish_reason":"tool_calls"}]}',
    b'{"choices":[{"delta":{},"finish_reason":"length"}]}', b'{"choices":[],"usage":{"prompt_tokens":3,"completion_tokens":4,"total_tokens":7}}',
    b'{"choices":[{"delta":{"tool_calls":[{"index":0,"id":"a","type":"function","function":{"name":"f","arguments":"{"}}]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"index":0,"function":{"arguments":"x"}},{"index":0,"function":{"name":"g","arguments":"y"}}]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"index":2,"id":"late","function":{"name":"gap"}}]}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"index":1,"function":null,"id":null}]}}]}', b'{"choices":[{"delta":{"tool_calls":null}}]}',
    b'{"choices":[{"delta":{"tool_calls":[{"index":-1,"id":"neg","function":{"name":"n"}}]}}]}', b"{oops", b"", b"{}", b"null",
]
PREFIX = [b"data: ", b"data: ", b"data: ", b"data:", b"data:  ", b"Data: ", b"event: x", b": ping", b"", b"id: 7"]
EOL = [b"\n", b"\n", b"\n\n", b"\n\n", b"\r\n", b"\r\n\r\n", b"\n\n\n"]


def _adversarial(rng, n_lines):
    out = bytearray()

    def pick(xs):
        return xs[int(rng.integers(len(xs)))]

    for _ in range(n_lines):
        out += pick(SPACES) + pick(PREFIX) + pick(PAYLOADS) + pick(SPACES) + pick(EOL)
    if rng.integers(3) == 0:
        out += b"data: {\"tail\":"          # unterminated tail
    return bytes(out)


def _bodies():
    bodies = []
    for fx in GOLD:
        for v in fx.values():
            if isinstance(v, list) and v and all(isinstance(x, str) for x in v):
                bodies.append("".join(x if x.endswith("\n") else x + "\n\n" for x in v).encode())
            elif isinstance(v, str) and "data: " in v:
                bodies.append(v.encode())
    for name in ("C2", "C3", "C4"):
        streams, _ = synth.make_config(name, n_streams=60)
        bodies += [b for b, _, _ in streams]
    rng = np.random.default_rng(1234)
    bodies += [_adversarial(rng, int(rng.integers(1, 14))) for _ in range(1500)]
    return bodies


BODIES = _bodies()


def test_trim_space_model_matches_oracle():
    rng = np.random.default_rng(5)
    for _ in range(4000):
        s = b"".join(SPACES[int(rng.integers(len(SPACES)))] for _ in range(int(rng.integers(0, 4)))) + \
            [b"", b"x", b"data: y", "é".encode()][int(rng.integers(4))] + \
            b"".join(SPACES[int(rng.integers(len(SPACES)))] for _ in range(int(rng.integers(0, 4))))
        assert orc.trim_space(s) == sm.trim_space(s), s


def test_agent_iteration_model_matches_oracle():
    assert len(BODIES) > 1600
    n_term = n_tc = 0
    for body in BODIES:
        v = orc.reframe(body)
        m = sm.run_with_stream(body)
        assert [ln.out for ln in v.lines if ln.kind == orc.L_EMITTED] == m["frames"], body[:120]
        assert v.builder == m["builder"] and v.acc_content == m["content"], body[:120]
        assert v.has_tool_calls == m["has_tool_calls"] and v.terminated == m["terminated"], body[:120]
        assert orc.parse_tool_calls(v.builder) == sm.parse_streaming_tool_calls(m["builder"]), body[:120]
        n_term += m["terminated"]
        n_tc += m["has_tool_calls"]
    assert n_term > 100 and n_tc > 50


def test_passthrough_and_telemetry_model_match_oracle():
    n_usage = 0
    for body in BODIES:
        v = orc.passthrough(body)
        assert [ln.out for ln in v.lines] == sm.lines(body) and v.out == b"".join(sm.lines(body))
        got = orc.telemetry(v.out)
        assert got == sm.telemetry(v.out), body[:120]
        n_usage += got[0] != (0, 0, 0)
    assert n_usage > 50


def test_decoded_payload_lengths_match_model():
    """orc_line's payload span: what each decoded line hands to json.Unmarshal (sse_rec.payload_len on the GPU side)."""
    n_done = n_exact = 0
    for body in BODIES:
        v = orc.reframe(body)
        got = [ln.payload for ln in v.lines if ln.kind in (orc.L_EMITTED, orc.L_DONE, orc.L_DONE_EXACT)]
        assert got == sm.decoded_payloads(body, True), body[:120]
        n_done += sum(ln.kind == orc.L_DONE for ln in v.lines)
        n_exact += sum(ln.kind == orc.L_DONE_EXACT for ln in v.lines)
        assert all(ln.payload_len == 6 for ln in v.lines if ln.kind == orc.L_DONE_EXACT)
        v = orc.passthrough(body, parse=True)
        assert [ln.payload for ln in v.lines if ln.chunk is not None] == sm.decoded_payloads(body, False), body[:120]
    assert n_done > 100 and n_exact > 0
