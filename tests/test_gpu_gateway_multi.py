"""GPU: the gateway over several contexts with batches in flight (ssegw_new_multi). Streams are cut into seeded pieces and
written over many ticks; every stream's delivered frames, agent content, tool calls, finish and has_tool_calls are compared
with the CPU oracle and with a one-context, depth-1 gateway fed the same pieces."""
import ctypes as C

import numpy as np
import pytest

from inference_gateway_b200 import _abi as A, synth
from inference_gateway_b200.gateway import Gateway
from inference_gateway_b200.synth import random_cuts
from oracle import orc
from tests.corpus import adversarial_bodies
from tests.util import TINY_PRODUCE, check_agent

pytestmark = pytest.mark.gpu

P, R, PP = A.MODE_P, A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE
RAW = -1                      # the raw proxy loop: ssegw_proxy_stream / ssegw_proxy_step (mode P)
N_SLOTS = 4


def config(conns, batch=1 << 18, flags=0, **caps):
    cfg = A.Config()
    A.load().sse_default_config(C.byref(cfg), conns, batch)
    cfg.n_slots = N_SLOTS
    cfg.flags = flags
    for k, v in caps.items():
        setattr(cfg, k, v)
    return cfg


class Out:
    def __init__(self, mode):
        self.mode, self.frames, self.eof, self.agent = mode, [], False, None


def drain(g, sid, o):
    fn = g.proxy_step if o.mode == RAW else g.recv
    try:
        while (e := fn(sid)) is not None:
            o.frames.append(e)
    except EOFError:
        o.eof = True


def drive(g, bodies, modes, n_pieces=6, seed=0, max_ticks=5000):
    """Opens one stream per body (in order), writes each body in seeded pieces, one piece per stream and tick, closes the
    upstream right after the pump that took its last piece (its batch may still be in flight), and pumps until every channel
    is closed. Returns ([Out], stream ids)."""
    rng = np.random.default_rng(seed)
    sids = [g.proxy_stream() if m == RAW else g.stream_chat_completions(m) for m in modes]
    outs = [Out(m) for m in modes]
    queue = [random_cuts(rng, b, int(rng.integers(1, n_pieces + 1))) for b in bodies]
    left = [b"" for _ in bodies]
    closed = [False] * len(bodies)
    for _ in range(max_ticks):
        for i, sid in enumerate(sids):
            if not left[i] and queue[i]:
                left[i] = queue[i].pop(0)
            if left[i]:
                left[i] = left[i][g.upstream_write(sid, left[i]):]
        g.pump()
        for i, sid in enumerate(sids):
            if not closed[i] and not left[i] and not queue[i]:
                g.upstream_close(sid)
                closed[i] = True
            drain(g, sid, outs[i])
        if all(o.eof for o in outs):
            break
    else:
        raise AssertionError("streams still open after max_ticks")
    assert g.flush() == 0
    for i, sid in enumerate(sids):
        if modes[i] == R:
            outs[i].agent = g.agent_state(sid)
    return outs, sids


def check_oracle(bodies, modes, outs, label):
    for i, (b, m, o) in enumerate(zip(bodies, modes, outs)):
        if m == R:
            v = orc.reframe(b)
            want = [l.out for l in v.lines if l.kind == orc.L_EMITTED]
            check_agent(o.agent, v, f"{label} stream {i}")
        else:
            want = [l.out for l in orc.passthrough(b, parse=bool(m & A.MODE_PARSE)).lines]
        assert o.frames == want, f"{label} stream {i} mode {m}: {len(o.frames)} frames, oracle {len(want)}"


def check_same(outs, ref, label):
    for i, (o, r) in enumerate(zip(outs, ref)):
        assert o.frames == r.frames and o.agent == r.agent, f"{label} stream {i} differs from the one-context depth-1 gateway"


@pytest.fixture(scope="module")
def workload():
    """C3-shaped synthetic streams, C4-shaped ones (tool calls among them) and adversarial corpus streams, in modes P, R, P|PARSE
    and the raw proxy loop."""
    c3 = [b for b, _, _ in synth.make_config("C3", n_streams=240)[0]]
    c4 = [b for b, _, _ in synth.make_config("C4", n_streams=240)[0]]
    adv = adversarial_bodies(np.random.default_rng(5), 60)
    # the corpus streams run in the modes without an agent fold: some nest past the decoder's limit, which a fold refuses
    modes = [(P, R, PP, RAW)[i % 4] for i in range(len(c3 + c4))] + [(P, PP, RAW)[i % 3] for i in range(len(adv))]
    return c3 + c4 + adv, modes


@pytest.fixture(scope="module")
def reference(workload):
    bodies, modes = workload
    g = Gateway(device=0, config=config(len(bodies)))
    try:
        outs, _ = drive(g, bodies, modes)
    finally:
        g.close()
    check_oracle(bodies, modes, outs, "one context, depth 1")
    return outs


@pytest.mark.parametrize("devices", [[0], [0, 0], [0, 0, 0]], ids=lambda d: f"ctx{len(d)}")
@pytest.mark.parametrize("depth", [1, 2, N_SLOTS])
def test_streams_match_the_oracle_and_depth_one(workload, reference, devices, depth):
    bodies, modes = workload
    g = Gateway(config=config(len(bodies)), devices=devices, depth=depth)
    try:
        outs, sids = drive(g, bodies, modes)
    finally:
        g.close()
    label = f"devices {devices} depth {depth}"
    check_oracle(bodies, modes, outs, label)
    check_same(outs, reference, label)
    per_ctx = np.bincount(np.asarray(sids) // len(bodies), minlength=len(devices))
    assert per_ctx.max() - per_ctx.min() <= 1


@pytest.mark.parametrize("devices,depth", [([0, 0], 2), ([0, 0, 0], N_SLOTS)])
def test_counters_add_up_over_contexts(workload, devices, depth):
    """Passthrough streams (no early termination, so every complete line the device counts is a frame the gateway delivers):
    the gateway's counters hold every context's batches exactly once."""
    bodies, modes = workload
    keep = [i for i, m in enumerate(modes) if m != R]
    bodies, modes = [bodies[i] for i in keep], [modes[i] for i in keep]
    g = Gateway(config=config(len(bodies), flags=A.FLAG_COUNTERS), devices=devices, depth=depth)
    try:
        outs, _ = drive(g, bodies, modes, seed=3)
        k = g.counters()
    finally:
        g.close()
    check_oracle(bodies, modes, outs, f"counters devices {devices} depth {depth}")
    delivered = sum(len(o.frames) for o in outs)
    assert k["p_frames_zero_copy"] + k["p_frames_materialised"] == delivered > 0


@pytest.mark.parametrize("devices,depth", [([0], N_SLOTS), ([0, 0], 2), ([0, 0, 0], N_SLOTS)])
def test_deferral_keeps_each_stream_in_one_batch_in_flight(workload, devices, depth):
    """SSE_FLAG_DEFER with produce capacities far below a tick's need: batches defer, and a stream whose rest goes back to its
    queue is never in a second uncollected batch, so every byte arrives once and in order."""
    bodies, modes = workload
    g = Gateway(config=config(len(bodies), batch=1 << 20, flags=A.FLAG_DEFER | A.FLAG_COUNTERS, **TINY_PRODUCE),
                devices=devices, depth=depth)
    try:
        outs, _ = drive(g, bodies, modes, seed=1)
        k = g.counters()
    finally:
        g.close()
    assert k["p_deferred_rounds"] > 0
    check_oracle(bodies, modes, outs, f"defer devices {devices} depth {depth}")


def long_body(rng, n_lines, size):
    parts = []
    for j in range(n_lines):
        text = bytes(int(x) for x in rng.integers(0x61, 0x7B, size=size + 997 * j))
        parts.append(b'data: {"choices":[{"index":0,"delta":{"content":"' + text + b'"},"finish_reason":null}]}\n\n')
    parts.append(b'data: {"choices":[{"index":0,"delta":{},"finish_reason":"stop"}]}\n\ndata: [DONE]\n\n')
    return b"".join(parts)


@pytest.mark.parametrize("devices,depth", [([0], N_SLOTS), ([0, 0], N_SLOTS)])
def test_line_pool_lines_complete_while_batches_are_in_flight(workload, devices, depth):
    """Lines longer than the 16 KiB carry slot continue in the line pool across ticks while other streams' batches are in
    flight on the same context."""
    bodies, modes = workload
    rng = np.random.default_rng(7)
    longs = [long_body(rng, 3, 100_000 + 20_000 * i) for i in range(8)]
    b2, m2 = list(bodies[:120]) + longs, list(modes[:120]) + [(R, PP)[i % 2] for i in range(len(longs))]
    kw = dict(config=config(len(b2)), line_pool=dict(pool_pages=48))
    g = Gateway(devices=devices, depth=depth, **kw)
    try:
        outs, _ = drive(g, b2, m2, n_pieces=12, seed=2)
    finally:
        g.close()
    check_oracle(b2, m2, outs, f"pool devices {devices} depth {depth}")
    g = Gateway(**kw)
    try:
        ref, _ = drive(g, b2, m2, n_pieces=12, seed=2)
    finally:
        g.close()
    check_same(outs, ref, f"pool devices {devices} depth {depth}")


@pytest.mark.parametrize("mode", [P, R])
def test_reopened_connection_gets_nothing_of_the_old_stream(mode):
    """A stream released while batches still hold its bytes, and its connection reopened at once: the reset is ordered after
    those batches and what they return for the connection goes to nobody, so the new stream sees exactly its own body."""
    n = 64
    g = Gateway(config=config(n), devices=[0], depth=N_SLOTS)
    try:
        sids = [g.stream_chat_completions(mode) for _ in range(n)]
        assert sids == list(range(n))
        old = b'data: {"choices":[{"index":0,"delta":{"content":"old stream"},"finish_reason":null}]}\n\n' * 300
        for _ in range(3):
            for s in sids:                   # several batches in flight, each ending inside a line (and the channel, never
                assert g.upstream_write(s, old[:1200]) == 1200          # drained, below its 100 elements)
            g.pump()
        for s in sids[::2]:
            g.release(s)
        new = [g.stream_chat_completions(mode) for _ in sids[::2]]
        assert new == sids[::2]              # the lowest free connections: the ones just released
        body = (b'data: {"choices":[{"index":0,"delta":{"content":"new"},"finish_reason":null}]}\n\n'
                b'data: {"choices":[{"index":0,"delta":{},"finish_reason":"stop"}]}\n\ndata: [DONE]\n\n')
        for s in new:
            assert g.upstream_write(s, body) == len(body)
            g.upstream_close(s)
        outs = {s: Out(mode) for s in new}
        for _ in range(100):
            g.pump()
            for s in new:
                drain(g, s, outs[s])
            if all(o.eof for o in outs.values()):
                break
        assert g.flush() == 0
        for s in new:
            if mode == R:
                outs[s].agent = g.agent_state(s)
        check_oracle([body] * len(new), [mode] * len(new), [outs[s] for s in new], "reopened")
    finally:
        g.close()


def test_placement_balances_open_streams():
    g = Gateway(config=config(16), devices=[0, 0, 0], depth=2)
    try:
        ctx = lambda s: s // 16
        first = [g.stream_chat_completions(P) for _ in range(3)]
        assert [ctx(s) for s in first] == [0, 1, 2]           # fewest open streams, lowest index on a tie
        more = [g.stream_chat_completions(R) for _ in range(20)]
        live = first + more
        for s in live[::3]:
            g.release(s)
        live = [s for s in live if s not in live[::3]]
        for _ in range(12):
            live.append(g.stream_chat_completions(P))
            counts = np.bincount([ctx(s) for s in live], minlength=3)
        assert counts.max() - counts.min() <= 1 and len(set(live)) == len(live)
        for s in live:
            g.release(s)
        opened = [g.proxy_stream() for _ in range(48)]
        assert sorted(opened) == list(range(48))
        with pytest.raises(RuntimeError):
            g.stream_chat_completions(P)
    finally:
        g.close()
