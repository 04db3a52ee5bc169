"""GPU: the extremal loads of tests/capacity.py on every engine.

Measure: each load runs alone on a context with four times the worst-case capacities; the kernels' own counts of frames,
records, work items, runs and tool-call elements must equal capacity.demand(), and out and text bytes must stay within its
bounds. This pins the demand model to the kernels, so that test_capacity_cpu.py's comparison with the config means something.

Hold: the same load, next to two ordinary C4 streams, runs on a context configured exactly by sse_worst_case_config (the two
fused engines with the tile kernel's longest carry slot). No batch may overflow, every batch passes orc_check_result, and
every connection matches the oracle.

Pooled: on the three split engines, lines assembled in the line pool go through both, on contexts with a line pool.

Gateway: a blank-line flood, a stream of [1,1,...] lines and connections completing carried lines share a 1 MiB gateway with
ordinary agent streams, which all get the oracle's frames and one [DONE]."""
import numpy as np
import pytest

from inference_gateway_b200 import SseEngine, _abi as A, synth
from inference_gateway_b200.gateway import Gateway
from oracle import orc
from tests import capacity as K
from tests import seams as S
from tests.capacity import TILE_SLOT, worst
from tests.util import ENGINES, assert_digest_parity, check_result

pytestmark = pytest.mark.gpu
CONNS, BATCH = 10, 1 << 20
N_GOOD = 2
CAPS = ("max_frames", "max_recs", "max_tcs", "max_usages", "text_arena_bytes", "max_runs", "out_arena_bytes")


# the line pool of the pooled loads (split engines): four connections each complete a line of three pages, next to in-batch
# lines of the same kind
POOL = dict(pool_pages=24, page_bytes=65536, max_line_bytes=1 << 20)
POOL_CONNS = 4


def _cfg(name):
    fused = bool(ENGINES[name] & A.FLAG_KERNEL_FUSED)
    return worst(CONNS, BATCH, slot=TILE_SLOT if fused else None), ("tile" if fused else "split")


def _engine(name, scale, pool=None):
    """A context for engine `name` with sse_worst_case_config's capacities times scale (and a line pool's growth on top)."""
    cfg, _ = _cfg(name)
    over = {k: getattr(cfg, k) * scale for k in CAPS}
    return SseEngine(device=0, max_conns=CONNS, bytes_per_batch=BATCH, flags=ENGINES[name], n_slots=1, line_pool=pool,
                     in_arena_bytes=cfg.in_arena_bytes, carry_slot_bytes=cfg.carry_slot_bytes, **over)


def _loads(name, budget, n_conns):
    cfg, _ = _cfg(name)
    return K.generators(budget, n_conns, cfg.carry_slot_bytes)


def _pooled(budget):
    return K.pooled(budget, POOL_CONNS, POOL["pool_pages"] * POOL["page_bytes"] // 2, POOL["page_bytes"])


def _batch(eng, items, digests=None):
    """One checked batch of (conn, mode, bytes) items; folds it into digests (d, carry, flags) when given. Returns
    (status, overflow message, counts) with counts read from the result."""
    slot, arena, segs = eng.acquire()
    try:
        n, nbytes = eng.fill(arena, segs, items)
        eng.submit(slot, n, nbytes)
        try:
            res = eng.collect(slot)
        except A.SseError as e:
            if e.status != A.SSE_ERR_OVERFLOW:
                raise
            return e.status, str(e), None
        check_result(eng, res, segs[:n].copy())
        if digests is not None:
            conn = np.array([c for c, _, _ in items], dtype=np.uint32)
            assert orc.digest_result(res.raw, conn, *digests) == n
        r = res.raw
        counts = dict(frames=r.n_frames, recs=r.n_recs, items=r.n_decoded, runs=r.n_runs, tcs=r.n_tcs, usages=r.n_usages,
                      out=r.out_bytes, text=r.text_bytes)
        return A.SSE_OK, "", counts
    finally:
        eng.release(slot)


def _measure(eng, kind, loads) -> list:
    """Runs each load alone (its prefixes first) and returns where the kernels' counts differ from capacity.demand()."""
    bad = []
    for g in loads:
        eng.reset_all()
        pre = [(i, c.mode, c.prefix) for i, c in enumerate(g.conns) if c.prefix]
        if pre:
            st, msg, _ = _batch(eng, pre)
            assert st == A.SSE_OK, f"{g.name}: prefix batch {msg}"
        st, msg, got = _batch(eng, [(i, c.mode, c.body) for i, c in enumerate(g.conns)])
        assert st == A.SSE_OK, f"{g.name}: {msg}"
        want = K.demand(g, kind)
        for a in K.EXACT:
            if a == "items" and kind == "tile":
                continue                                # the tile kernel has no work items
            if got[a] != want[a]:
                bad.append(f"{g.name}: {a} measured {got[a]}, model {want[a]}")
        for a in ("out", "text"):
            if got[a] > want[a]:
                bad.append(f"{g.name}: {a} measured {got[a]}, above the model's bound {want[a]}")
    return bad


def _good_streams():
    bodies = [b for b, _, _ in synth.make_config("C4", n_streams=N_GOOD)[0]]
    return bodies, [A.MODE_R | A.MODE_PARSE] * N_GOOD


def _hold_budget(cfg):
    """Input bytes a load may take next to the good streams' second pieces, and the cut of each good stream."""
    good, _ = _good_streams()
    cut = [len(b) // 3 for b in good]
    return cfg.in_arena_bytes - sum(S.r16(len(b) - c) for b, c in zip(good, cut)), cut


def _hold(eng, loads, cut) -> list:
    """Runs each load next to the good streams, in two batches (the prefixes and the good streams' first pieces, then the
    rest), and returns the batches that overflowed and the loads that differ from the oracle (assert_digest_parity)."""
    good, gmodes = _good_streams()
    bad = []
    for g in loads:
        att = [(c.mode, c.prefix + c.body) for c in g.conns]
        na = len(att)                                   # the good streams' connections follow the load's
        bodies = [b for _, b in att] + good
        modes = [m for m, _ in att] + gmodes
        d = (orc.new_digests(len(bodies)), np.zeros(len(bodies), np.uint32), np.zeros(len(bodies), np.uint32))
        eng.reset_all()
        first = [(i, c.mode, c.prefix) for i, c in enumerate(g.conns) if c.prefix]
        first += [(na + j, gmodes[j], good[j][:cut[j]]) for j in range(N_GOOD)]
        st, msg, _ = _batch(eng, first, d)
        assert st == A.SSE_OK, f"{g.name}: first batch {msg}"
        second = [(i, c.mode, c.body) for i, c in enumerate(g.conns)]
        second += [(na + j, gmodes[j], good[j][cut[j]:]) for j in range(N_GOOD)]
        st, msg, _ = _batch(eng, second, d)
        if st != A.SSE_OK:
            bad.append(f"{g.name}: {msg}")
            continue
        try:
            assert_digest_parity(d, bodies, modes, g.name)
        except AssertionError as e:
            bad.append(str(e))
    return bad


@pytest.fixture(scope="module")
def engines():
    live = {}

    def get(name, scale, pool=None):
        key = (name, scale, pool is not None)
        if key not in live:
            for e in live.values():
                e.close()
            live.clear()
            live[key] = _engine(name, scale, pool)
        return live[key]
    yield get
    for e in live.values():
        e.close()


@pytest.mark.parametrize("name", list(ENGINES))
def test_measured_demand_equals_the_model(engines, name):
    cfg, kind = _cfg(name)
    bad = _measure(engines(name, 4), kind, _loads(name, cfg.in_arena_bytes, CONNS))
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("name", list(ENGINES))
def test_worst_case_config_holds_every_load(engines, name):
    cfg, _ = _cfg(name)
    budget, cut = _hold_budget(cfg)
    bad = _hold(engines(name, 1), _loads(name, budget, CONNS - N_GOOD), cut)
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("name", [n for n, f in ENGINES.items() if not f & A.FLAG_KERNEL_FUSED])
def test_pooled_loads_measured_and_held(engines, name):
    """Lines assembled in the line pool (the tile kernel has none): the kernels' counts equal the model with four times the
    worst-case capacities, and the worst-case config grown by sse_line_pool_config holds them next to the good streams."""
    cfg, kind = _cfg(name)
    bad = _measure(engines(name, 4, POOL), kind, _pooled(cfg.in_arena_bytes))
    budget, cut = _hold_budget(cfg)
    bad += _hold(engines(name, 1, POOL), _pooled(budget), cut)
    assert not bad, "\n".join(bad)


def test_gateway_holds_floods_tool_call_elements_and_carried_lines():
    """A 1 MiB gateway (sse_worst_case_config): one connection floods 400 KiB of blank lines in one write (6,400 rounds of 64
    lines), one sends 720 KB of [1,1,...] lines, three complete lines of a whole carry slot of {} elements in every other
    batch; three agent streams next to them each get the oracle's frames and one [DONE]."""
    R = A.MODE_R | A.MODE_PARSE
    g = Gateway(device=0, max_conns=8, bytes_per_batch=1 << 20)
    try:
        flood = g.proxy_stream()
        nums = g.stream_chat_completions(K.PP)
        carriers = [g.stream_chat_completions(K.PP) for _ in range(3)]
        good = [g.stream_chat_completions(R) for _ in range(3)]
        ok_body = (b'data: {"choices":[{"index":0,"delta":{"content":"hi"},"finish_reason":null}]}\n\n'
                   b'data: {"choices":[{"index":0,"delta":{},"finish_reason":"stop"}]}\n\n')
        num_line, _ = K.tc_line("numbers", 60000)
        big_line, _ = K.tc_line("objects", 65536)
        streams = {flood: b"\n" * (400 << 10), nums: num_line * 12}
        for s in carriers:
            streams[s] = big_line * 6
        sent = {s: 0 for s in streams}
        got = {s: 0 for s in streams}
        want = {flood: 400 << 10, nums: 12}
        want.update({s: 6 for s in carriers})
        good_out = {s: [] for s in good}
        for s in good:
            assert g.upstream_write(s, ok_body) == len(ok_body)
        for step in range(2000):
            for s, body in streams.items():
                # carriers write half a line per pump, so that every line completes from the carry slot
                piece = 32768 if s in carriers else 1 << 20
                if sent[s] < len(body):
                    sent[s] += g.upstream_write(s, body[sent[s]:sent[s] + piece])
            g.pump()
            while (e := g.proxy_step(flood)) is not None:
                assert e == b"\n"
                got[flood] += 1
            for s in [nums] + carriers:
                while (e := g.recv(s)) is not None:
                    assert e == (num_line if s == nums else big_line)
                    got[s] += 1
            for s in good:
                try:
                    while (e := g.agent_recv(s)) is not None:
                        good_out[s].append(e)
                except EOFError:
                    pass
            if got == want:
                break
        assert got == want
        v = orc.reframe(ok_body)
        exp = [l.out for l in v.lines if l.kind == orc.L_EMITTED] + [b"data: [DONE]\n\n"]
        assert v.terminated and len(exp) == 3
        for s in good:
            assert good_out[s] == exp
    finally:
        g.close()
