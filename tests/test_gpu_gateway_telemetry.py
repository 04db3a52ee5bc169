"""GPU: the gateway's telemetry tap (ssegw_stream_with_telemetry, gateway.Telemetry). Client responses are written in seeded
pieces, one piece per upstream stream and tick; a response is one upstream stream, or several mode R streams opened one after
another that share one fold (an MCP session, whose tool-call merge and last-four-pieces window span the iterations). The
verdict: every stream's frames are the oracle's; the fold finishes with (0, *orc.telemetry(body)), body being what the client
was sent (the MCP agent's final [DONE], fed by the caller, included), or with 1 when body has an irregular piece (DESIGN.md
§5, deviation 4); a stream whose records include a line past the nesting limit ends after a prefix of the oracle's frames
that reaches that line, and its fold is not compared. Untapped streams keep their old behaviour next to tapped ones."""
import numpy as np
import pytest

from inference_gateway_b200 import _abi as A, synth
from inference_gateway_b200.gateway import Gateway, Telemetry
from tests import folds
from tests.gateway_drive import (Session, assert_folds_saw_something, check_sessions, check_telemetry, drive, expected,
                                 gateway_config)
from tests.util import DONE, ENGINES, TINY_DECODE, TINY_PRODUCE

pytestmark = pytest.mark.gpu

P, R, PP = A.MODE_P, A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE
N_SLOTS = 4


# ------------------------------------------------------------------ workloads
def long_pieces():
    """Segments of more than 64 lines (several runs), and lines longer than a produce window."""
    e = folds.element
    many = b"".join(folds.tc_chunk([e(k % 7, id=b"m%d" % k, name=b"n", args=b"%d," % k)]) for k in range(150)) + folds.STOP
    blanks = (b"data: {}\n" + b"\n" * 70) * 3 + folds.TAIL + folds.STOP
    wide = folds.tc_chunk([e(k, id=b"w%d" % k, name=b"f\\u00e9", args=b"x" * 300) for k in range(30)]) + folds.USAGE + folds.STOP
    return [many, blanks, wide]


def synth_bodies(name, n):
    return [b for b, _, _ in synth.make_config(name, n_streams=n)[0]]


def iteration(tag, k, last):
    """One agent iteration's upstream body: content, tool calls that reuse indices 0 and 1 of the iterations before, usage,
    then finish_reason tool_calls (stop on the last iteration)."""
    e = folds.element
    fin = b"stop" if last else b"tool_calls"
    return (folds.HEAD
            + folds.tc_chunk([e(0, id=b"%s-%d" % (tag, k), name=b"lookup", args=b"q%d" % k)], content=b"step %d" % k)
            + folds.tc_chunk([e(0, args=b"+%d" % k), e(1, id=b"%s-b%d" % (tag, k), name=b"fetch%d" % k, args=b"{}")])
            + b'data: {"choices":[],"usage":{"prompt_tokens":%d,"completion_tokens":%d,"total_tokens":%d}}\n\n' % (10 + k, k, 10 + 2 * k)
            + b'data: {"choices":[{"index":0,"delta":{},"finish_reason":"%s"}]}\n\n' % fin + DONE)


def mcp_sessions(n, seed):
    """n sessions of two or three mode R iterations sharing one fold; some iterations are C4-shaped bodies."""
    rng = np.random.default_rng(seed)
    c4 = synth_bodies("C4", 2 * n)
    out = []
    for i in range(n):
        m = 2 + i % 2
        parts = [iteration(b"s%d" % i, k, k == m - 1) for k in range(m)]
        if i % 3 == 2:
            parts[int(rng.integers(0, m))] = c4[i]
        out.append(Session(parts, R))
    return out


def plain_sessions(bodies, untapped_every=4, proxy_every=5):
    """One session per body in mode P|PARSE with its own fold; every untapped_every-th is untapped (mode P or P|PARSE in
    turn), every proxy_every-th reads through the raw proxy loop."""
    out = []
    for i, b in enumerate(bodies):
        if i % untapped_every == untapped_every - 1:
            out.append(Session([b], (P, PP)[i // untapped_every % 2], tap=False))
        else:
            out.append(Session([b], PP, route="proxy" if i % proxy_every == 0 else "chan"))
    return out


# ------------------------------------------------------------------ 1, 2, 3: handler, proxy route and MCP sessions
@pytest.fixture(scope="module")
def plain_bodies():
    c = folds.corpus(small=True)
    return [b for fam in c.values() for b in fam] + long_pieces() + synth_bodies("C3", 48) + synth_bodies("C4", 48)


@pytest.mark.parametrize("depth", [1, N_SLOTS])
@pytest.mark.parametrize("devices", [[0], [0, 0]], ids=lambda d: f"ctx{len(d)}")
@pytest.mark.parametrize("eng", ["split", "fused"])
def test_tap_on_handler_and_proxy_streams(plain_bodies, eng, devices, depth):
    sessions = plain_sessions(plain_bodies)
    # the tile kernel's lines are at most 49,120 bytes; a smaller slot loosens no bound
    slot = dict(carry_slot_bytes=32768) if eng == "fused" else {}
    g = Gateway(config=gateway_config(len(sessions), worst_case=True, flags=ENGINES[eng], **slot), devices=devices, depth=depth)
    try:
        assert drive(g, sessions, seed=depth + 10 * len(devices)) >= 0
    finally:
        g.close()
    n_limited, compared = check_sessions(sessions, f"{eng} devices {devices} depth {depth}")
    assert n_limited > 0                    # the corpus reaches the nesting limit on tapped streams
    assert_folds_saw_something(compared)
    assert any(s.route == "proxy" for s in sessions)


@pytest.mark.parametrize("devices,depth", [([0], 1), ([0], N_SLOTS), ([0, 0], N_SLOTS)])
def test_mcp_sessions_share_one_fold(devices, depth):
    """Two or three mode R streams per session, each opened once the one before was released, among other sessions' plain
    streams (tapped and untapped). Tool-call indices repeat over the iterations, so telemetry merges across them."""
    c3 = synth_bodies("C3", 40)
    sessions = mcp_sessions(36, seed=depth) + plain_sessions(c3)
    g = Gateway(config=gateway_config(len(sessions), worst_case=True), devices=devices, depth=depth)
    try:
        assert drive(g, sessions, seed=depth) >= 0
    finally:
        g.close()
    n_limited, compared = check_sessions(sessions, f"mcp devices {devices} depth {depth}")
    assert n_limited == 0
    assert_folds_saw_something(compared)
    # a merge that spans iterations: index 0's arguments hold every iteration's pieces
    _, calls = compared[0]
    assert calls[0]["args"] == b"q0+0q1+1"


# ------------------------------------------------------------------ 4: deferral and the line pool
@pytest.mark.parametrize("devices,depth", [([0], N_SLOTS), ([0, 0], 2)])
@pytest.mark.parametrize("eng", ["split", "copy"])
def test_tap_when_batches_defer(eng, devices, depth):
    """SSE_FLAG_DEFER at capacities far below a tick's need: deferred rests go back to their queues, decode arenas grow in
    sse_collect, and every fold still sees each segment once and in order."""
    c = folds.corpus(seed=1, n_adv=24)
    bodies = c["adversarial"] + c["tricky"][::3] + c["merge"] + c["near_misses"][::8] + long_pieces() + synth_bodies("C4", 32)
    sessions = plain_sessions(bodies) + mcp_sessions(12, seed=7)
    cfg = gateway_config(len(sessions), flags=A.FLAG_DEFER | A.FLAG_COUNTERS | ENGINES[eng], **TINY_PRODUCE, **TINY_DECODE)
    g = Gateway(config=cfg, devices=devices, depth=depth)
    try:
        assert drive(g, sessions, seed=3) >= 0
        k = g.counters()
    finally:
        g.close()
    assert k["p_deferred_rounds"] > 0
    _, compared = check_sessions(sessions, f"defer {eng} devices {devices} depth {depth}")
    assert_folds_saw_something(compared)


def long_body(rng, n_lines, size):
    parts = []
    for j in range(n_lines):
        text = bytes(int(x) for x in rng.integers(0x61, 0x7B, size=size + 997 * j))
        parts.append(b'data: {"choices":[{"index":0,"delta":{"content":"' + text + b'"},"finish_reason":null}]}\n\n')
    parts.append(folds.USAGE + b'data: {"choices":[{"index":0,"delta":{},"finish_reason":"stop"}]}\n\ndata: [DONE]\n\n')
    return b"".join(parts)


@pytest.mark.parametrize("devices,depth", [([0], 1), ([0, 0], 1)])
def test_tap_on_line_pool_lines(devices, depth):
    """Lines longer than the carry slot, assembled in the line pool over several ticks, among them the 65,534-65,537-element
    tool-call lines, next to C4 streams, on the worst-case config (which the pool grows by its size)."""
    rng = np.random.default_rng(11)
    longs = [long_body(rng, 3, 100_000 + 20_000 * i) for i in range(4)]
    big = folds.saturated_streams() + longs
    sessions = ([Session([b], PP) for b in big] + [Session([b], R) for b in big]
                + plain_sessions(synth_bodies("C4", 48)))
    g = Gateway(config=gateway_config(len(sessions), worst_case=True), devices=devices, depth=depth,
                line_pool=dict(pool_pages=192, page_bytes=65536, max_line_bytes=512 * 1024))
    try:
        assert drive(g, sessions, seed=depth, n_pieces=12) >= 0
    finally:
        g.close()
    n_limited, compared = check_sessions(sessions, f"pool devices {devices} depth {depth}")
    assert n_limited == 0
    for (_, calls), n in zip(compared, folds.SATURATED):
        assert len(calls) == 4 and calls[-1]["id"] == b"id%d" % (n - 1)      # index 0 ({} elements) has no name


# ------------------------------------------------------------------ 5: released while batches are in flight
def tool_body(tag, n):
    e = folds.element
    out = []
    for j in range(n):
        out.append(b'data: {"choices":[{"index":0,"delta":{"content":"%s %d"},"finish_reason":null}]}\n\n' % (tag, j))
        out.append(folds.tc_chunk([e(j % 3, id=b"%s%d" % (tag, j), name=b"f%d" % (j % 3), args=b"%d," % j)]))
        out.append(b'data: {"choices":[],"usage":{"prompt_tokens":%d,"completion_tokens":%d,"total_tokens":%d}}\n\n'
                   % (j, 2 * j, 3 * j))
    return b"".join(out)


def test_released_tap_gets_nothing_of_batches_in_flight():
    """Tapped streams released while batches still hold their bytes, and their connections reopened at once with new folds:
    an old fold holds the telemetry of exactly the frames its stream received, a new fold sees only its own stream, and the
    streams left open, tapped or not, are the oracle's to the end."""
    n = 64
    g = Gateway(config=gateway_config(n), devices=[0], depth=N_SLOTS)
    try:
        taps = [Telemetry() if i % 4 != 3 else None for i in range(n)]
        sids = [g.stream_chat_completions(PP, telemetry=t) for t in taps]
        assert sids == list(range(n))
        old = tool_body(b"old", 120)
        got = {s: [] for s in sids}

        def drain(s):
            try:
                while (f := g.recv(s)) is not None:
                    got[s].append(f)
            except EOFError:
                return True
            return False

        for r in range(3):                  # several batches in flight, each ending inside a line
            for s in sids:
                assert g.upstream_write(s, old[1200 * r:1200 * (r + 1)]) == 1200
            g.pump()
            for s in sids:
                drain(s)
        released = sids[::2]
        for s in released:
            drain(s)
            g.release(s)
        old_frames = {s: got.pop(s) for s in released}
        new_taps = [Telemetry() for _ in released]
        reopened = [g.stream_chat_completions(PP, telemetry=t) for t in new_taps]
        assert reopened == released
        new = tool_body(b"new", 6) + folds.STOP
        for s in reopened:
            got[s] = []
            assert g.upstream_write(s, new) == len(new)
            g.upstream_close(s)
        rest = {s: old[3600:] for s in sids[1::2]}
        eof = set()
        for _ in range(500):
            for s, left in rest.items():
                rest[s] = left[g.upstream_write(s, left):]
                if not rest[s]:
                    g.upstream_close(s)
            g.pump()
            eof |= {s for s in got if s not in eof and drain(s)}
            if len(eof) == len(got):
                break
        assert len(eof) == len(got) and g.flush() == 0
    finally:
        g.close()
    _, want_old, _ = expected(old, PP)
    for s, t in zip(released, (taps[s] for s in released)):
        fr = old_frames[s]
        assert fr == want_old[:len(fr)] and fr, f"released stream {s}: not a prefix of the oracle's frames"
        check_telemetry(t, b"".join(fr), f"released stream {s}")
    _, want_new, _ = expected(new, PP)
    for s, t in zip(reopened, new_taps):
        assert got[s] == want_new, f"reopened stream {s}: frames differ from the oracle's"
        check_telemetry(t, b"".join(got[s]), f"reopened stream {s}")
    for s in sids[1::2]:
        assert got[s] == want_old, f"open stream {s}: frames differ from the oracle's"
        if taps[s] is not None:
            check_telemetry(taps[s], old, f"open stream {s}")
    for t in [t for t in taps if t is not None] + new_taps:
        t.close()


# ------------------------------------------------------------------ 6: refusals
def test_attach_refusals_and_reattach():
    L = A.load()
    g = Gateway(config=gateway_config(4), devices=[0], depth=2)
    tel, other = Telemetry(), Telemetry()
    try:
        attach = lambda mode, t: L.ssegw_stream_with_telemetry(g.g, mode, t.f if t is not None else None)
        assert attach(P, tel) == A.SSE_ERR_ARG                 # mode P alone produces no records
        assert attach(PP, None) == A.SSE_ERR_ARG
        with pytest.raises(A.SseError) as e:
            g.stream_chat_completions(P, telemetry=tel)
        assert e.value.status == A.SSE_ERR_ARG
        first = g.stream_chat_completions(R, telemetry=tel)
        assert attach(PP, tel) == A.SSE_ERR_BUSY               # one feeder at a time
        with pytest.raises(A.SseError) as e:
            g.proxy_stream(telemetry=tel)
        assert e.value.status == A.SSE_ERR_BUSY
        more = [g.stream_chat_completions(P) for _ in range(3)]
        assert attach(PP, other) == -1                          # no free connection
        with pytest.raises(RuntimeError):
            g.stream_chat_completions(PP, telemetry=other)
        g.release(first)
        assert g.stream_chat_completions(A.MODE_R, telemetry=tel) == first   # reattached to the next iteration's stream
        g.release(more[0])
        assert g.proxy_stream(telemetry=other) == more[0]
        for s in (first, more[0]):
            g.upstream_close(s)
        g.pump()
        assert g.flush() == 0
    finally:
        g.close()
    for t in (tel, other):
        assert t.finish() == (0, (0, 0, 0), [])
        t.close()
