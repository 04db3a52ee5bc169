"""GPU: the gateway's telemetry tap (ssegw_stream_with_telemetry, gateway.Telemetry). Client responses are written in seeded
pieces, one piece per upstream stream and tick; a response is one upstream stream, or several mode R streams opened one after
another that share one fold (an MCP session, whose tool-call merge and last-four-pieces window span the iterations). The
verdict: every stream's frames are the oracle's; the fold finishes with (0, *orc.telemetry(body)), body being what the client
was sent (the MCP agent's final [DONE], fed by the caller, included), or with 1 when body has an irregular piece (DESIGN.md
§5, deviation 4); a stream whose records include a line past the nesting limit ends after a prefix of the oracle's frames
that reaches that line, and its fold is not compared. Untapped streams keep their old behaviour next to tapped ones."""
import ctypes as C

import numpy as np
import pytest

from inference_gateway_b200 import _abi as A, synth
from inference_gateway_b200.gateway import Gateway, Telemetry
from inference_gateway_b200.synth import random_cuts
from oracle import orc
from tests import folds
from tests.util import DONE, ENGINES, TINY_DECODE, TINY_PRODUCE, check_agent, irregular_telemetry

pytestmark = pytest.mark.gpu

P, R, PP = A.MODE_P, A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE
N_SLOTS = 4
MiB = 1 << 20


def worst_case(conns, flags=0):
    cfg = A.Config()
    A.load().sse_worst_case_config(C.byref(cfg), conns, MiB)
    cfg.n_slots, cfg.flags = N_SLOTS, flags
    return cfg


def default(conns, batch=MiB, flags=0, **caps):
    cfg = A.Config()
    A.load().sse_default_config(C.byref(cfg), conns, batch)
    cfg.n_slots, cfg.flags = N_SLOTS, flags
    for k, v in caps.items():
        setattr(cfg, k, v)
    return cfg


class Session:
    """One client response: the upstream bodies of `parts`, each opened once the one before was delivered to the end and
    released, in `mode`, read through the channel ("chan") or the raw proxy loop ("proxy"); its own fold unless tap is
    False."""

    def __init__(self, parts, mode, route="chan", tap=True):
        self.parts, self.mode, self.route = list(parts), mode, route
        self.tel = Telemetry() if tap else None
        self.frames = [[] for _ in self.parts]
        self.agent = [None] * len(self.parts)
        self.k, self.sid, self.done = -1, None, False
        self.queue, self.left, self.upstream_closed = [], b"", False


def open_next(g, s, rng, n_pieces):
    s.k += 1
    s.sid = g.proxy_stream(telemetry=s.tel) if s.route == "proxy" else g.stream_chat_completions(s.mode, telemetry=s.tel)
    s.queue = random_cuts(rng, s.parts[s.k], int(rng.integers(1, n_pieces + 1)))
    s.left, s.upstream_closed = b"", False


def drive(g, sessions, seed, n_pieces=6, max_ticks=5000):
    """Writes every session's streams in seeded pieces, one piece per stream and tick, closes each upstream after the pump that
    took its last piece, and reads every channel after every pump. A stream whose channel ends is released (mode R: after
    its agent state was read) and the session's next stream is opened at once, while the other sessions' batches may still
    be in flight."""
    rng = np.random.default_rng(seed)
    for s in sessions:
        open_next(g, s, rng, n_pieces)
    for _ in range(max_ticks):
        live = [s for s in sessions if not s.done]
        if not live:
            break
        for s in live:
            if not s.left and s.queue:
                s.left = s.queue.pop(0)
            if s.left:
                s.left = s.left[g.upstream_write(s.sid, s.left):]
        g.pump()
        for s in live:
            if not s.upstream_closed and not s.left and not s.queue:
                g.upstream_close(s.sid)
                s.upstream_closed = True
            fn = g.proxy_step if s.route == "proxy" else g.recv
            try:
                while (f := fn(s.sid)) is not None:
                    s.frames[s.k].append(f)
            except EOFError:
                if s.mode & A.MODE_R:
                    s.agent[s.k] = g.agent_state(s.sid)
                g.release(s.sid)
                if s.k + 1 < len(s.parts):
                    open_next(g, s, rng, n_pieces)
                else:
                    s.done = True
    else:
        raise AssertionError("sessions still open after max_ticks")
    assert g.flush() >= 0


def expected(body, mode):
    """The oracle's view of one upstream body, its frames, and how many of them reach its first line past the nesting limit
    (None: no such line)."""
    if mode & A.MODE_R:
        v = orc.reframe(body)
        lines = [(l, l.kind == orc.L_EMITTED) for l in v.lines]
    else:
        v = orc.passthrough(body, parse=bool(mode & A.MODE_PARSE))
        lines = [(l, True) for l in v.lines]
    want, upto = [], None
    for l, emitted in lines:
        if emitted:
            want.append(l.out)
        if upto is None and l.kind != orc.L_UNREAD and l.depth_limited:
            upto = len(want)
    return v, want, upto


def check_telemetry(tel, body, label):
    rc, usage, calls = tel.finish()
    if irregular_telemetry(body):
        assert rc == 1, f"{label}: telemetry finished with {rc} on a body with an irregular piece"
    else:
        assert (rc, usage, calls) == (0, *orc.telemetry(body)), f"{label}: telemetry differs from the oracle's"
    return usage, calls


def check_sessions(sessions, label):
    """The verdict on every session. Returns (sessions ended by a line past the nesting limit, fold results compared)."""
    n_limited, compared = 0, []
    for i, s in enumerate(sessions):
        lab = f"{label} session {i} mode {s.mode} {s.route}{'' if s.tel else ' untapped'}"
        limited = False
        for k, (body, got) in enumerate(zip(s.parts, s.frames)):
            v, want, upto = expected(body, s.mode)
            # a fold that meets such a line closes the stream: the tap, or the agent fold of a mode R stream
            if upto is not None and (s.tel is not None or s.mode & A.MODE_R):
                limited = True
                assert upto <= len(got) <= len(want) and got == want[:len(got)], \
                    f"{lab} part {k}: {len(got)} frames are not a prefix of the oracle's {len(want)} through frame {upto}"
                continue
            assert got == want, f"{lab} part {k}: {len(got)} frames, oracle {len(want)}"
            if s.mode & A.MODE_R:
                check_agent(s.agent[k], v, f"{lab} part {k}")
        n_limited += limited
        if s.tel is not None:
            if not limited:
                body = b"".join(f for part in s.frames for f in part)
                if s.mode & A.MODE_R:
                    s.tel.feed_bytes(DONE)          # the agent's single final [DONE] (agent.go:140-143)
                    body += DONE
                compared.append(check_telemetry(s.tel, body, lab))
            s.tel.close()
    return n_limited, compared


def assert_folds_saw_something(compared):
    assert any(u != (0, 0, 0) for u, _ in compared) and any(c for _, c in compared)


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
    cfg = worst_case(len(sessions), ENGINES[eng])
    if eng == "fused":
        cfg.carry_slot_bytes = 32768        # the tile kernel's lines are at most 49,120 bytes; a smaller slot loosens no bound
    g = Gateway(config=cfg, devices=devices, depth=depth)
    try:
        drive(g, sessions, seed=depth + 10 * len(devices))
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
    g = Gateway(config=worst_case(len(sessions)), devices=devices, depth=depth)
    try:
        drive(g, sessions, seed=depth)
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
    cfg = default(len(sessions), flags=A.FLAG_DEFER | A.FLAG_COUNTERS | ENGINES[eng], **TINY_PRODUCE, **TINY_DECODE)
    g = Gateway(config=cfg, devices=devices, depth=depth)
    try:
        drive(g, sessions, seed=3)
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
    g = Gateway(config=worst_case(len(sessions)), devices=devices, depth=depth,
                line_pool=dict(pool_pages=192, page_bytes=65536, max_line_bytes=512 * 1024))
    try:
        drive(g, sessions, seed=depth, n_pieces=12)
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
    g = Gateway(config=default(n), devices=[0], depth=N_SLOTS)
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
    g = Gateway(config=default(4), devices=[0], depth=2)
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
