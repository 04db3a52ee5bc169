"""GPU: the gateway over several contexts with batches in flight (ssegw_new_multi). Streams are cut into seeded pieces and
written over many ticks; every stream's delivered frames, agent content, tool calls, finish and has_tool_calls are compared
with the CPU oracle and with a one-context, depth-1 gateway fed the same pieces."""
import numpy as np
import pytest

from inference_gateway_b200 import _abi as A, synth
from inference_gateway_b200.gateway import Gateway
from tests.corpus import adversarial_bodies
from tests.gateway_drive import Session, check_sessions, drive, gateway_config
from tests.util import TINY_PRODUCE

pytestmark = pytest.mark.gpu

P, R, PP = A.MODE_P, A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE
RAW = -1                      # the raw proxy loop: ssegw_proxy_stream / ssegw_proxy_step (mode P)
N_SLOTS = 4


def sessions(bodies, modes):
    """One untapped session per body; RAW reads through the raw proxy loop."""
    return [Session([b], P, route="proxy", tap=False) if m == RAW else Session([b], m, tap=False) for b, m in zip(bodies, modes)]


def check_same(ss, ref, label):
    for i, (s, r) in enumerate(zip(ss, ref)):
        assert s.frames == r.frames and s.agent == r.agent, f"{label} stream {i} differs from the one-context depth-1 gateway"


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
    ss = sessions(bodies, modes)
    g = Gateway(device=0, config=gateway_config(len(bodies), 1 << 18))
    try:
        assert drive(g, ss, seed=0) == 0
    finally:
        g.close()
    assert check_sessions(ss, "one context, depth 1")[0] == 0
    return ss


@pytest.mark.parametrize("devices", [[0], [0, 0], [0, 0, 0]], ids=lambda d: f"ctx{len(d)}")
@pytest.mark.parametrize("depth", [1, 2, N_SLOTS])
def test_streams_match_the_oracle_and_depth_one(workload, reference, devices, depth):
    bodies, modes = workload
    ss = sessions(bodies, modes)
    g = Gateway(config=gateway_config(len(bodies), 1 << 18), devices=devices, depth=depth)
    try:
        assert drive(g, ss, seed=0) == 0
    finally:
        g.close()
    label = f"devices {devices} depth {depth}"
    assert check_sessions(ss, label)[0] == 0
    check_same(ss, reference, label)
    # one part per session: each sid is the stream id drive opened before its first tick
    per_ctx = np.bincount(np.asarray([s.sid for s in ss]) // len(bodies), minlength=len(devices))
    assert per_ctx.max() - per_ctx.min() <= 1


@pytest.mark.parametrize("devices,depth", [([0, 0], 2), ([0, 0, 0], N_SLOTS)])
def test_counters_add_up_over_contexts(workload, devices, depth):
    """Passthrough streams (no early termination, so every complete line the device counts is a frame the gateway delivers):
    the gateway's counters hold every context's batches exactly once."""
    bodies, modes = workload
    keep = [i for i, m in enumerate(modes) if m != R]
    ss = sessions([bodies[i] for i in keep], [modes[i] for i in keep])
    g = Gateway(config=gateway_config(len(ss), 1 << 18, flags=A.FLAG_COUNTERS), devices=devices, depth=depth)
    try:
        assert drive(g, ss, seed=3) == 0
        k = g.counters()
    finally:
        g.close()
    assert check_sessions(ss, f"counters devices {devices} depth {depth}")[0] == 0
    delivered = sum(len(s.frames[0]) for s in ss)
    assert k["p_frames_zero_copy"] + k["p_frames_materialised"] == delivered > 0


@pytest.mark.parametrize("devices,depth", [([0], N_SLOTS), ([0, 0], 2), ([0, 0, 0], N_SLOTS)])
def test_deferral_keeps_each_stream_in_one_batch_in_flight(workload, devices, depth):
    """SSE_FLAG_DEFER with produce capacities far below a tick's need: batches defer, and a stream whose rest goes back to its
    queue is never in a second uncollected batch, so every byte arrives once and in order."""
    bodies, modes = workload
    ss = sessions(bodies, modes)
    g = Gateway(config=gateway_config(len(bodies), flags=A.FLAG_DEFER | A.FLAG_COUNTERS, **TINY_PRODUCE),
                devices=devices, depth=depth)
    try:
        assert drive(g, ss, seed=1) == 0
        k = g.counters()
    finally:
        g.close()
    assert k["p_deferred_rounds"] > 0
    assert check_sessions(ss, f"defer devices {devices} depth {depth}")[0] == 0


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
    kw = dict(config=gateway_config(len(b2), 1 << 18), line_pool=dict(pool_pages=48))
    ss, ref = sessions(b2, m2), sessions(b2, m2)
    g = Gateway(devices=devices, depth=depth, **kw)
    try:
        assert drive(g, ss, seed=2, n_pieces=12) == 0
    finally:
        g.close()
    assert check_sessions(ss, f"pool devices {devices} depth {depth}")[0] == 0
    g = Gateway(**kw)
    try:
        assert drive(g, ref, seed=2, n_pieces=12) == 0
    finally:
        g.close()
    check_same(ss, ref, f"pool devices {devices} depth {depth}")


@pytest.mark.parametrize("mode", [P, R])
def test_reopened_connection_gets_nothing_of_the_old_stream(mode):
    """A stream released while batches still hold its bytes, and its connection reopened at once: the reset is ordered after
    those batches and what they return for the connection goes to nobody, so the new stream sees exactly its own body."""
    n = 64
    g = Gateway(config=gateway_config(n, 1 << 18), devices=[0], depth=N_SLOTS)
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
        ss = {s: Session([body], mode, tap=False) for s in new}
        eof = set()
        for _ in range(100):
            g.pump()
            for s in new:
                try:
                    while (f := g.recv(s)) is not None:
                        ss[s].frames[0].append(f)
                except EOFError:
                    eof.add(s)
            if len(eof) == len(new):
                break
        assert g.flush() == 0
        for s in new:
            if mode == R:
                ss[s].agent[0] = g.agent_state(s)
        assert check_sessions([ss[s] for s in new], "reopened")[0] == 0
    finally:
        g.close()


def test_placement_balances_open_streams():
    g = Gateway(config=gateway_config(16, 1 << 18), devices=[0, 0, 0], depth=2)
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
