"""GPU: lines longer than the carry slot continue in the line pool (sse_init_ex) and come out bit-exact against the CPU
oracle, which has no line limit (bufio.Reader.ReadBytes grows for as long as a line goes on, provider.go:312-322)."""
import json

import numpy as np
import pytest

from inference_gateway_b200 import SseEngine, _abi as A, synth
from oracle import orc
from tests.streams import PAGE, SLOT, USAGE, chunk, long_line, stream_with
from tests.util import ENGINES, check_folds, check_stream, check_streams, run_pieces, run_streams

pytestmark = pytest.mark.gpu

P, R, PP = A.MODE_P, A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE
MODES = (P, R, PP)
MiB = 1 << 20


@pytest.fixture(scope="module", params=["split", "templates", "copy"])
def eng(request):
    """The default pipeline, with skeleton templates, and with SSE_FLAG_COPY_OUT, each with a 64 MiB line pool. Decoded text
    of a line may take 3 bytes per input byte (invalid UTF-8 -> U+FFFD), so the text arena is raised for 16 MiB lines."""
    e = SseEngine(device=0, max_conns=1024, bytes_per_batch=64 * MiB, carry_slot_bytes=SLOT, n_slots=2,
                  text_arena_bytes=128 * MiB, flags=ENGINES[request.param], line_pool=dict(pool_pages=1024, page_bytes=PAGE))
    yield e
    e.close()


LENGTHS = [64 * 1024 + 1, 100_000, MiB, 8 * MiB, A.MAX_LINE_BYTES]


def _kinds(n):
    if n <= MiB:
        return ["content", "toolcall", "done", "crlf", "terminal"]
    return ["content", "terminal"] if n <= 8 * MiB else ["toolcall"]


@pytest.mark.parametrize("n_batches", [1, 3, 17, 64])
@pytest.mark.parametrize("length", LENGTHS, ids=lambda n: f"L{n}")
def test_long_line_lengths(eng, length, n_batches):
    rng = np.random.default_rng(length ^ n_batches)
    bodies, modes = [], []
    for kind in _kinds(length):
        line = long_line(kind, length, rng)
        assert len(line) == length
        for m in MODES:
            bodies.append(stream_with(line, kind))
            modes.append(m)
    outs = run_streams(eng, bodies, modes, n_batches=n_batches, seed=length + n_batches, with_folds=True)
    check_streams(bodies, modes, outs, f"L={length} batches={n_batches}")
    assert not any(o.flags & (A.SEG_DEAD | A.SEG_LINE_TOO_LONG) for o in outs)
    assert eng.pool_stats()[0] == 0          # every line completed: every page is back


def test_one_mib_tool_call_folds(eng):
    """sse_agent_tool_calls and the telemetry fold see the whole 1 MiB arguments string of a single-chunk tool call."""
    rng = np.random.default_rng(5)
    line = long_line("toolcall", MiB, rng)
    body = chunk(b"Writing the file.") + line + b"\n" + b'data: {"choices":[{"index":0,"delta":{},"finish_reason":"tool_calls"}]}\n\n' + USAGE
    for nb in (1, 8):
        outs = run_streams(eng, [body, body], [R, PP], n_batches=nb, seed=nb, with_folds=True)
        views = check_streams([body, body], [R, PP], outs, f"folds batches={nb}")
        content, has, term, fin, calls = check_folds(eng.L, outs[0], R, views[0], f"folds batches={nb}")
        check_folds(eng.L, outs[1], PP, views[1], f"folds batches={nb} mode {PP}")
        assert has and term and fin == 2
        args = json.loads(line[6:])["choices"][0]["delta"]["tool_calls"][0]["function"]["arguments"].encode()
        assert len(calls) == 1 and calls[0]["args"] == args and len(args) > 900_000
        for o in outs:
            eng.L.sse_agent_free(o.agent)
            eng.L.sse_telemetry_free(o.tele)


def test_mixed_workload_with_rare_long_tool_calls(eng):
    """C4 at 512 streams, about 2 % of them with an extra 300 KB single-chunk tool call: every stream is bit-exact,
    including the ones without a long line."""
    streams, mode = synth.make_config("C4", n_streams=512)
    rng = np.random.default_rng(42)
    bodies, n_long = [], 0
    for i, (b, _, _) in enumerate(streams):
        if rng.random() < 0.02 or i == 7:
            cut = b.find(b"\n\n") + 2
            b = b[:cut] + long_line("toolcall", 300_000 + int(rng.integers(0, 50_000)), rng) + b"\n" + b[cut:]
            n_long += 1
        bodies.append(b)
    assert n_long >= 5
    outs = run_streams(eng, bodies, [mode] * len(bodies), n_batches=6, seed=3)
    check_streams(bodies, [mode] * len(bodies), outs, "mixed C4")
    assert not any(o.flags & A.SEG_DEAD for o in outs)
    eng.reset_all()
    assert eng.pool_stats()[0] == 0


def test_finished_connection_returns_pooled_tail():
    """A terminating chunk followed, in the same segment, by a long line: the produce stage pools the line before decode
    finds the termination; the connection ends FINISHED (not DEAD) and its pages go back. A reset in the middle of a pooled
    line returns its pages too."""
    e = SseEngine(device=0, max_conns=64, bytes_per_batch=4 * MiB, carry_slot_bytes=SLOT, line_pool=dict(pool_pages=64))
    try:
        rng = np.random.default_rng(9)
        term = b'data: {"choices":[{"index":0,"delta":{"content":"done"},"finish_reason":"stop"}]}\n\n'
        tail = long_line("content", 300_000, rng)[:-1]           # never terminated
        body = chunk(b"a") + term + tail
        outs = run_streams(e, [body], [R], n_batches=1)
        check_stream(body, R, outs[0], "finished")
        assert outs[0].terminated and not outs[0].flags & A.SEG_DEAD
        assert e.pool_stats()[0] == 0
        # mode P keeps the unterminated tail in the pool: carry_len reports all of it
        outs = run_streams(e, [body], [P], n_batches=3, seed=1)
        check_stream(body, P, outs[0], "pooled tail")
        assert outs[0].carry_len == len(tail)
        used, hw = e.pool_stats()
        assert used == (len(tail) + PAGE - 1) // PAGE and hw >= used
        e.reset_conn(0)
        assert e.pool_stats()[0] == 0
        # the connection starts over cleanly after the reset
        slot, res = e.process([(0, R, chunk(b"again"))])
        try:
            assert res.seg_frames(0) == [chunk(b"again")]
        finally:
            e.release(slot)
    finally:
        e.close()


def test_pool_exhaustion_fails_only_the_unlucky():
    """More simultaneous long lines than the pool holds: each connection completes bit-exact or ends LINE_TOO_LONG | DEAD,
    at least one completes, no batch overflows, and after the resets no page is held."""
    e = SseEngine(device=0, max_conns=64, bytes_per_batch=8 * MiB, carry_slot_bytes=SLOT, line_pool=dict(pool_pages=8))
    try:
        rng = np.random.default_rng(11)
        dead = 0
        for nb in (1, 4):
            bodies = [stream_with(long_line("toolcall", 200_000 + 1000 * i, rng), "toolcall") for i in range(12)]
            modes = [MODES[i % 3] for i in range(12)]
            outs = run_streams(e, bodies, modes, n_batches=nb, seed=nb)     # an overflow would raise in sse_collect
            ok = 0
            for i, (b, m, o) in enumerate(zip(bodies, modes, outs)):
                if o.flags & A.SEG_DEAD:
                    assert o.flags & A.SEG_LINE_TOO_LONG
                    dead += 1
                else:
                    check_stream(b, m, o, f"exhaustion stream {i}")
                    ok += 1
            assert ok >= 1
            for c in range(12):
                e.reset_conn(c)
            used, hw = e.pool_stats()
            assert used == 0 and hw <= 8
        assert dead > 0                           # the pool did run dry
    finally:
        e.close()


def test_line_over_max_line_bytes_fails_only_its_connection():
    e = SseEngine(device=0, max_conns=64, bytes_per_batch=4 * MiB, carry_slot_bytes=SLOT,
                  line_pool=dict(pool_pages=64, max_line_bytes=128 * 1024))
    try:
        rng = np.random.default_rng(13)
        bodies = [stream_with(long_line("content", 200_000, rng), "content"),
                  stream_with(long_line("content", 100_000, rng), "content"),
                  chunk(b"short") + b"data: [DONE]\n\n"]
        for nb in (1, 5):
            outs = run_streams(e, bodies, [R, R, R], n_batches=nb, seed=nb)
            assert outs[0].flags & A.SEG_LINE_TOO_LONG and outs[0].flags & A.SEG_DEAD
            check_stream(bodies[1], R, outs[1], "under the cap")
            check_stream(bodies[2], R, outs[2], "short")
            assert e.pool_stats()[0] == 0
    finally:
        e.close()


def test_gateway_agent_iteration_with_a_2mib_tool_call():
    """One agent iteration through the gateway mirror whose upstream sends a 2 MiB single-chunk tool call, written in 37 KB
    pieces: the agent state holds the exact arguments and the MCP writer gets the oracle's frames plus one [DONE]."""
    from inference_gateway_b200.gateway import Gateway
    g = Gateway(device=0, max_conns=8, bytes_per_batch=1 << 20, line_pool=dict(pool_pages=64))
    try:
        rng = np.random.default_rng(17)
        line = long_line("toolcall", 2 * MiB, rng)
        body = chunk(b"Saving.") + line + b"\n" + b'data: {"choices":[{"index":0,"delta":{},"finish_reason":"tool_calls"}]}\n\n'
        sid = g.stream_chat_completions(R)
        written = b""
        for i in range(0, len(body), 37_000):
            piece = body[i:i + 37_000]
            assert g.upstream_write(sid, piece) == len(piece)
            g.pump()
            out, _, ended = g.mcp_write_loop(sid)
            written += out
        g.upstream_close(sid)
        g.pump()
        out, status_503, ended = g.mcp_write_loop(sid)
        written += out
        content, has, term, fin, calls = g.agent_state(sid)
        args = json.loads(line[6:])["choices"][0]["delta"]["tool_calls"][0]["function"]["arguments"].encode()
        assert has and term and fin == 2 and content == b"Saving."
        assert len(calls) == 1 and calls[0]["args"] == args and calls[0]["name"] == b"write_file"
        v = orc.reframe(body)
        assert ended and not status_503
        assert written == b"".join(l.out for l in v.lines if l.kind == orc.L_EMITTED) + b"data: [DONE]\n\n"
        g.release(sid)
    finally:
        g.close()


# ------------------------------------------------------------------ page arithmetic: pages smaller than the slot, odd sizes
SMALL_PAGE = 4096 + 16       # not a power of two; the 32 KiB slot spans 8 of them when a line leaves it


@pytest.fixture(scope="module")
def small_pages():
    e = SseEngine(device=0, max_conns=64, bytes_per_batch=20 * MiB, carry_slot_bytes=SLOT, n_slots=2, text_arena_bytes=64 * MiB,
                  line_pool=dict(pool_pages=4096, page_bytes=SMALL_PAGE))
    yield e
    e.close()


@pytest.mark.parametrize("n_batches", [1, 3, 17, 64])
@pytest.mark.parametrize("length", LENGTHS[:3], ids=lambda n: f"L{n}")
def test_long_lines_with_small_odd_pages(small_pages, length, n_batches):
    test_long_line_lengths(small_pages, length, n_batches)


@pytest.mark.parametrize("page", [SMALL_PAGE, PAGE], ids=["page4112", "page65536"])
def test_empty_segments_while_a_line_is_held(page):
    """An empty segment for a connection whose held-back line fills its slot or its pages exactly (a whole number of pages,
    the slot to the byte) or not, changes nothing: the line later completes bit-exact and every page comes back."""
    e = SseEngine(device=0, max_conns=64, bytes_per_batch=4 * MiB, carry_slot_bytes=SLOT, line_pool=dict(pool_pages=512, page_bytes=page))
    try:
        rng = np.random.default_rng(21)
        line = long_line("toolcall", 600_000, rng)
        body = chunk(b"a") + line + b"\n" + chunk(b"b", '"stop"') + b"data: [DONE]\n\n"
        start = len(chunk(b"a"))
        for held in (SLOT - 1, SLOT, SLOT + 1, 3 * page, 3 * page + 1, 8 * page, 8 * page - 1):
            cut = start + held
            pieces = [body[:cut], b"", body[cut:cut + 5000], b"", b"", body[cut + 5000:]]
            if held % page == 0 and held > SLOT:       # the pooled prefix is a whole number of pages when the empty segment comes
                pieces = [body[:cut], b"", b"", body[cut:]]
            outs = run_pieces(e, [pieces] * 3, list(MODES))
            check_streams([body] * 3, list(MODES), outs, f"held={held} page={page}")
            assert not any(o.flags & (A.SEG_DEAD | A.SEG_LINE_TOO_LONG) for o in outs), held
            assert e.pool_stats()[0] == 0
        # a pooled line of exactly k pages, then only empty segments: still held, its pages still owned
        outs = run_pieces(e, [[body[:start + 8 * page], b"", b""]], [P])
        assert not outs[0].flags & A.SEG_DEAD and outs[0].carry_len == 8 * page
        assert e.pool_stats()[0] == 8
        e.reset_conn(0)
        assert e.pool_stats()[0] == 0
    finally:
        e.close()
