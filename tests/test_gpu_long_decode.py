"""GPU: the long-line decode stage. Work items of at least SSE_LONG_LINE payload bytes are decoded by a whole warp each (string
and digit-run jumps, warp-parallel unquote); every result must be the oracle's, bit for bit, wherever an escape, a UTF-8 sequence
or an error falls against the warp's 16-byte lanes and 512-byte steps, in every capture, and with counters, deferral and batches
in flight."""
import os
import re

import numpy as np
import pytest

from inference_gateway_b200 import SseEngine, _abi as A, synth
from inference_gateway_b200.gateway import Gateway
from oracle import orc
from tests.streams import USAGE, chunk, filler, long_line, stream_with
from tests.util import (ENGINES, check_agent, check_batch, check_folds, check_stream, check_streams, cut_bounds, digest_parity,
                        run_streams, text_spans)

pytestmark = pytest.mark.gpu
P, R, PP = A.MODE_P, A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE
MiB = 1 << 20
SLOT = 32768


def _threshold():
    src = open(os.path.join(os.path.dirname(os.path.dirname(__file__)), "inference_gateway_b200", "csrc", "sse_device.cuh")).read()
    return int(re.search(r"#define SSE_LONG_LINE (\d+)", src).group(1))


LONG = _threshold()
assert LONG > 0


def engine(flags=0, **kw):
    kw.setdefault("max_conns", 4096)
    kw.setdefault("bytes_per_batch", 96 * MiB)
    kw.setdefault("text_arena_bytes", 200 * MiB)
    return SseEngine(device=0, carry_slot_bytes=SLOT, flags=flags, line_pool=dict(pool_pages=4096), **kw)


@pytest.fixture(scope="module", params=["split", "templates", "copy"])
def eng(request):
    e = engine(ENGINES[request.param])
    yield e
    e.close()


HEAD = b'data: {"choices":[{"index":0,"delta":{"content":"'
TAIL = b'"},"finish_reason":null}]}'


def content_line(body, closed=True):
    """One data line (without its '\\n') whose payload is a content string with this body."""
    return HEAD + body + (TAIL if closed else b"")


def payload_len(line):
    return len(line) - 6


def sized(body_fn, n):
    """content_line whose payload is exactly n bytes: body_fn(k) gives a body of k bytes."""
    return content_line(body_fn(n - payload_len(content_line(b""))))


def streams_of(lines, tail=b""):
    return [chunk(b"a") + l + b"\n\n" + tail + chunk(b"z", '"stop"') + b"data: [DONE]\n\n" for l in lines]


def check_all(e, bodies, modes=(R, PP), nbs=(1, 3), label=""):
    for m in modes:
        for nb in nbs:
            digest_parity(e, bodies, m, cut_bounds(bodies, nb, seed=nb), f"{label} mode {m} x{nb}")


# ------------------------------------------------------------------ the seam
def test_seam(eng):
    rng = np.random.default_rng(1)
    lines = []
    for n in (LONG - 1, LONG, LONG + 1):
        lines.append(sized(lambda k: filler(rng, k), n))
        lines.append(sized(lambda k: b"x" * k, n))
        lines.append(sized(lambda k: ("中\U0001F600".encode() * k)[:k // 7 * 7] + b"y" * (k % 7), n))
        tc = long_line("toolcall", n + 7, rng)[:-1]
        assert payload_len(tc) == n
        lines.append(tc)
    assert sorted({payload_len(l) for l in lines}) == [LONG - 1, LONG, LONG + 1]
    check_all(eng, streams_of(lines), label="seam")


# ------------------------------------------------------------------ adversarial bodies at every offset
VALID = [b"\\" * k + b'"' for k in range(1, 34, 2)] + [b"\\" * k for k in range(2, 34, 2)] + [
    "😀".encode(), b"\\ud83d\\ude00", b"\\ud83d", b"\\ude00", b"\\ud83d\\ud83d\\ude00", b"\\ude00\\ud83d", b"\\u00e9\\n",
    "é".encode(), "€".encode(), "中".encode(), b"\xc0\x80", b"\xc1\xbf", b"\xe0\x80\x80", b"\xed\xa0\x80", b"\xf4\x90\x80\x80",
    b"\xe2\x82", b"\x80", b"\xbf\xbf", b"\xf5", b"\xff", b"\xf0\x9f\x98", b"\\/", b"\\b\\f\\r\\t"]
ERRORS = [b"\x01", b"\x1f", b"\t", b"\\x", b"\\u12g4", b"\\ug234", b"\\u1g34", b"\\u123g", b"\\'", b'\\\\"x',
          b'\\\\\\\\"x', b"\\\xc3\xa9"]
ENDS = [b"", b"\\", b"\\u", b"\\u12", b"\\ud83d\\u", b"\xe2\x82", b"\xf0\x9f\x98", b"\\\\\\"]


def test_valid_units_at_every_offset(eng):
    """Each kind of unit repeated with every gap of 0..63 plain bytes: it meets every lane and step border."""
    lines = []
    for u in VALID:
        body = b"".join(b"x" * g + u for g in range(64) for _ in range(1 + LONG // (64 * (32 + len(u)))))
        lines.append(content_line(body + b"x" * max(0, LONG + 64 - len(body))))
    rng = np.random.default_rng(2)
    mixed = b"".join(b"x" * int(rng.integers(0, 40)) + VALID[int(rng.integers(0, len(VALID)))] for _ in range(6000))
    lines.append(content_line(mixed))
    assert all(payload_len(l) >= LONG for l in lines)
    check_all(eng, streams_of(lines), label="valid units")


def test_errors_and_ends_at_every_offset(eng):
    lines = []
    for err in ERRORS:
        for off in range(48):
            lines.append(content_line(b"x" * (600 + off) + err + b"x" * LONG))
    for end in ENDS:
        for off in range(48):
            lines.append(content_line(b"x" * (LONG + off) + end, closed=False))
    check_all(eng, streams_of(lines), nbs=(1,), label="errors")


def test_errors_across_a_whole_step():
    """Every error and payload end at each of 528 consecutive body offsets: wherever the warp's 512-byte steps begin, each one
    meets a step border (where lane 31 reads its look-ahead from the next step) and every lane border."""
    e = engine(max_conns=2048, bytes_per_batch=80 * MiB)
    try:
        lines = [content_line(b"x" * (600 + off) + err + b"x" * LONG) for err in ERRORS for off in range(528)]
        lines += [content_line(b"x" * (LONG + off) + end, closed=False) for end in ENDS for off in range(528)]
        for k in range(0, len(lines), 2000):
            bodies = streams_of(lines[k:k + 2000])
            digest_parity(e, bodies, R, cut_bounds(bodies, 1, seed=k), f"errors across a step, lines {k}..")
    finally:
        e.close()


def test_folds_of_long_tool_calls():
    """The agent and telemetry folds of streams whose tool call is one long line (around the threshold and far above it)
    agree with the oracle."""
    e = engine(max_conns=64, bytes_per_batch=16 * MiB)
    try:
        rng = np.random.default_rng(14)
        bodies = [chunk(b"Writing.") + long_line("toolcall", n, rng) + b"\n" +
                  b'data: {"choices":[{"index":0,"delta":{},"finish_reason":"tool_calls"}]}\n\n' + USAGE
                  for n in (LONG + 6, LONG + 7, LONG + 8, 5 * LONG, 2 * MiB)]   # payloads LONG - 1, LONG, LONG + 1, ...
        for nb in (1, 4):
            outs = run_streams(e, bodies, [R] * len(bodies), n_batches=nb, seed=nb, with_folds=True)
            for i, (b, o) in enumerate(zip(bodies, outs)):
                v = check_stream(b, R, o, label=f"folds stream {i} x{nb}")
                _, has, term, fin, calls = check_folds(e.L, o, R, v, f"folds stream {i} x{nb}")
                assert has and term and fin == 2 and len(calls) == 1
                e.L.sse_agent_free(o.agent)
                e.L.sse_telemetry_free(o.tele)
    finally:
        e.close()


# ------------------------------------------------------------------ long strings in every capture
def esc(n, rng):
    return filler(rng, n)


def tc_elem(i, parts):
    return b'{"index":%d,%s}' % (i, b",".join(parts))


def test_every_capture(eng):
    rng = np.random.default_rng(3)
    big = LONG + 100
    tc = b'data: {"choices":[{"index":0,"delta":{"tool_calls":[%s]},"finish_reason":null}]}'
    lines = [
        tc % tc_elem(0, [b'"id":"%s"' % esc(big, rng), b'"type":"%s"' % esc(big, rng),
                         b'"function":{"name":"%s","arguments":"%s"}' % (esc(big, rng), esc(big, rng))]),
        tc % tc_elem(0, [b'"id":"c\\n1"', b'"function":{"name":"w","arguments":"%s"}' % esc(big, rng)]),
        tc % b",".join(tc_elem(i, [b'"id":"%s"' % esc(big // 4, rng), b'"function":{"arguments":"%s"}' % esc(big // 4, rng)])
                       for i in range(4)),
        b'data: {"choices":[{"index":0,"delta":{"content":"%s"},"finish_reason":"%s"}]}' % (esc(100, rng), b"q" * big),
        b'data: {"choices":[{"index":0,"delta":{"content":"%s"},"finish_reason":"stop"}],"usage":{"prompt_tokens":1,"completion_tokens":2,"total_tokens":3}}' % esc(big, rng),
        b'data: {"choices":[{"index":0,"delta":{"content":"a","%s":"%s"},"finish_reason":null}]}' % (b"k" * big, esc(big, rng)),
        b'data: {"x_unknown":"%s","choices":[{"index":0,"delta":{"content":"b"}}]}' % esc(big, rng),
        b'data: {"choices":[{"index":0,"delta":{"content":"%s[DONE]%s"}}]}' % (esc(big // 2, rng), esc(big // 2, rng)),
        b'data: {"choices":[{"index":0,"delta":{"tool_calls":[{"index":%s}]}}]}' % (b"9" * big),
        b'data: {"choices":[{"index":0,"delta":{"content":"c"},"logprobs":{"content":[{"token":"t","logprob":-0.%s,"bytes":[1]}]}}]}' % (b"1" * big),
        b'data: {"choices":[{"index":0,"delta":{"content":"d"},"logprobs":{"content":[{"token":"t","logprob":1.5e%s}]}}]}' % (b"0" * big + b"7"),
        b'data: {"choices":[{"index":0,"delta":{"content":"e"}}],"created":%s}' % (b"1" * big),
        b'data: {"choices":[{"index":0,"delta":{"tool_calls":[%s]},"finish_reason":null}]}' % b",".join(
            tc_elem(i, [b'"id":"c%d"' % i, b'"function":{"arguments":"{\\"i\\":%d}"}' % i]) for i in range(LONG // 40)),
    ]
    for depth in (127, 128, 129):
        lines.append(b'data: {"choices":[{"index":0,"delta":{"content":"f"}}],"x":' + b"[" * (depth - 1) + b'"%s"' % esc(big, rng)
                     + b"]" * (depth - 1) + b"}")
    assert all(payload_len(l) >= LONG for l in lines)
    bodies = streams_of(lines, USAGE)
    check_all(eng, bodies, label="captures")
    outs = run_streams(eng, bodies, [R] * len(bodies), n_batches=2, seed=4)
    check_streams(bodies, R, outs, "captures")


def test_terminating_long_chunk():
    e = engine(max_conns=64, bytes_per_batch=8 * MiB)
    try:
        rng = np.random.default_rng(5)
        bodies = [stream_with(long_line("terminal", n, rng), "terminal") for n in (LONG + 10, 3 * LONG, MiB)]
        check_all(e, bodies, label="terminal")
        outs = run_streams(e, bodies, [R] * len(bodies), n_batches=1)
        assert all(o.terminated for o in outs)
    finally:
        e.close()


# ------------------------------------------------------------------ counters, deferral, batches in flight
def test_counters_long_only_and_jobs_per_span():
    rng = np.random.default_rng(6)
    big = LONG + 10
    tc = b'data: {"choices":[{"index":0,"delta":{"tool_calls":[%s]},"finish_reason":null}]}'
    lines = [tc % tc_elem(0, [b'"id":"%s"' % esc(big, rng), b'"function":{"name":"n\\t","arguments":"%s"}' % esc(big, rng)]),
             tc % tc_elem(0, [b'"id":"%s"' % esc(big, rng), b'"type":"f\\n"', b'"function":{"name":"n\\t","arguments":"%s"}' % esc(big, rng)]),
             content_line(esc(big, rng)), long_line("toolcall", 2 * big, rng)[:-1]]
    e = SseEngine(device=0, max_conns=64, bytes_per_batch=8 * MiB, carry_slot_bytes=SLOT, n_slots=1, text_arena_bytes=32 * MiB,
                  flags=A.FLAG_COUNTERS, line_pool=dict(pool_pages=256))
    try:
        for only_long in (True, False):
            payloads = [l[6:] for l in lines] + ([] if only_long else [b'{"choices":[{"index":0,"delta":{"content":"s\\n"}}]}'] * 50)
            items = [(i, PP, b"data: " + pl + b"\n\n") for i, pl in enumerate(payloads)]
            slot, res = e.process(items)
            try:
                k = e.counters(slot)
                check_batch(k, res, b"".join(it[2] for it in items), one_job_per_span=False)
                spans, _, two = text_spans(res)
                assert two and k["d_unquote_jobs"] == spans, (k["d_unquote_jobs"], spans)
                assert k["d_coop_strings"] > 0 and k["d_coop_bytes"] > 4 * LONG
                if only_long:
                    assert k["d_pulls"] == k["d_items"] == len(lines)
            finally:
                e.release(slot)
    finally:
        e.close()


def test_deferred_redecode_runs_the_long_kernel():
    rng = np.random.default_rng(7)
    bodies = streams_of([content_line(esc(LONG + 500 * i, rng)) for i in range(24)])
    e = SseEngine(device=0, max_conns=64, bytes_per_batch=8 * MiB, carry_slot_bytes=SLOT, text_arena_bytes=8192,
                  flags=A.FLAG_DEFER | A.FLAG_COUNTERS, n_slots=1, line_pool=dict(pool_pages=256))
    try:
        passes = []

        def hook(b, res):
            k = e.counters(0)
            check_batch(k, res)
            passes.append(k["decode_passes"])
        digest_parity(e, bodies, R, cut_bounds(bodies, 1, seed=1), "deferred", on_batch=hook)
        assert max(passes) > 1, passes
    finally:
        e.close()


def test_batches_in_flight():
    rng = np.random.default_rng(8)
    bodies = [b for b, _, _ in synth.make_config("C4", n_streams=512)[0]]
    for i in range(0, len(bodies), 16):
        cut = bodies[i].find(b"\n\n") + 2
        bodies[i] = bodies[i][:cut] + long_line("toolcall", LONG + int(rng.integers(0, 4 * LONG)), rng) + b"\n" + bodies[i][cut:]
    e = engine(max_conns=len(bodies), bytes_per_batch=32 * MiB, n_slots=4)
    try:
        digest_parity(e, bodies, R, cut_bounds(bodies, 4, seed=9), "batches in flight", depth=4)
    finally:
        e.close()


def test_mixed_traffic_and_a_context_without_long_lines():
    """C4-sized traffic with 1 % long tool calls in 4 pieces, and the same context on traffic with no long line."""
    rng = np.random.default_rng(10)
    bodies = [b for b, _, _ in synth.make_config("C4", n_streams=16384)[0]]
    plain = list(bodies)
    for i in rng.choice(len(bodies), size=len(bodies) // 100, replace=False):
        cut = bodies[i].find(b"\n\n") + 2
        bodies[i] = bodies[i][:cut] + long_line("toolcall", 200_000, rng) + b"\n" + bodies[i][cut:]
    e = engine(max_conns=len(bodies), bytes_per_batch=sum(map(len, bodies)))
    try:
        digest_parity(e, bodies, R, cut_bounds(bodies, 4, seed=11), "mixed")
        digest_parity(e, plain, R, cut_bounds(plain, 4, seed=12), "no long line")
    finally:
        e.close()


def test_gateway_folds_a_long_tool_call():
    g = Gateway(device=0, max_conns=8, bytes_per_batch=1 << 20, line_pool=dict(pool_pages=64))
    try:
        rng = np.random.default_rng(13)
        line = long_line("toolcall", 3 * LONG, rng)
        body = chunk(b"Saving.") + line + b"\n" + b'data: {"choices":[{"index":0,"delta":{},"finish_reason":"tool_calls"}]}\n\n'
        sid = g.stream_chat_completions(R)
        for i in range(0, len(body), 20_000):
            assert g.upstream_write(sid, body[i:i + 20_000]) == len(body[i:i + 20_000])
            g.pump()
        g.upstream_close(sid)
        g.pump()
        state = g.agent_state(sid)
        check_agent(state, orc.reframe(body), "gateway")
        content, has, term, fin, calls = state
        assert has and term and fin == 2 and content == b"Saving."
        assert len(calls) == 1 and len(calls[0]["args"]) > 2 * LONG
        g.release(sid)
    finally:
        g.close()
