"""Drives a Gateway as clients and upstreams do, and the verdict on what it delivered. A client response is a Session: the
upstream bodies of its parts, opened one after another on the stream of a channel or of the raw proxy loop, with its own
telemetry fold or none; a plain stream is a session of one part. drive writes every stream in seeded pieces over many ticks;
check_sessions compares every stream's frames, agent state and telemetry with the CPU oracle."""
import ctypes as C

import numpy as np

from inference_gateway_b200 import _abi as A
from inference_gateway_b200.gateway import Telemetry
from inference_gateway_b200.synth import random_cuts
from oracle import orc
from tests.util import DONE, check_agent, irregular_telemetry


def gateway_config(conns, batch=1 << 20, *, worst_case=False, flags=0, n_slots=4, **caps):
    """The sse_config of a gateway of `conns` connections per context: sse_default_config, or sse_worst_case_config, for
    batches of `batch` input bytes, with n_slots, flags and any other field in caps set."""
    cfg = A.Config()
    L = A.load()
    (L.sse_worst_case_config if worst_case else L.sse_default_config)(C.byref(cfg), conns, batch)
    cfg.n_slots, cfg.flags = n_slots, flags
    for k, v in caps.items():
        setattr(cfg, k, v)
    return cfg


class Session:
    """One client response: the upstream bodies of `parts`, each opened once the one before was delivered to the end and
    released, in `mode`, read through the channel ("chan") or the raw proxy loop ("proxy"); its own fold unless tap is
    False. sid is the id of the stream open for the current part."""

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


def drive(g, sessions, seed, n_pieces=6, max_ticks=5000, after_pump=None):
    """Writes every session's streams in seeded pieces (1 to n_pieces per stream), one piece per stream and tick, closes each
    upstream after the pump that took its last piece, and reads every channel after every pump. A stream whose channel ends
    is released (mode R: after its agent state was read) and the session's next stream is opened at once, while the other
    sessions' batches may still be in flight. after_pump(tick) runs right after each tick's pump. Returns what g.flush()
    returned once every session was done."""
    rng = np.random.default_rng(seed)
    for s in sessions:
        open_next(g, s, rng, n_pieces)
    for tick in range(max_ticks):
        live = [s for s in sessions if not s.done]
        if not live:
            break
        for s in live:
            if not s.left and s.queue:
                s.left = s.queue.pop(0)
            if s.left:
                s.left = s.left[g.upstream_write(s.sid, s.left):]
        g.pump()
        if after_pump is not None:
            after_pump(tick)
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
    return g.flush()


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
    """The verdict on every session: each part's frames are the oracle's, and in mode R so is its agent state; a part with a
    line past the nesting limit, where a fold meets it, ends after a prefix of the oracle's frames that reaches that line;
    a tapped session without such a line has the oracle's telemetry of what its client was sent. Closes every fold.
    Returns (sessions ended by a line past the nesting limit, fold results compared)."""
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
