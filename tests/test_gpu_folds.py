"""GPU: the agent and telemetry folds fed the kernels' own records of adversarial streams (tests/folds.py), on every engine, in
one batch and in pieces, under SSE_FLAG_DEFER at tiny capacities, with 65,534-65,537 tool-call elements in one line, and through
the gateway. The verdict is tests/util.py::check_folds: the oracle's agent state and telemetry, telemetry's irregular pieces
(DESIGN.md §5, deviation 4) finishing with 1, and SSE_ERR_UNDECODED from both feeds in the piece that completes the first line
past the nesting limit."""
import ctypes as C

import numpy as np
import pytest

from inference_gateway_b200 import SseEngine, _abi as A, synth
from inference_gateway_b200.gateway import Gateway
from inference_gateway_b200.synth import random_cuts
from oracle import orc
from tests import folds
from tests.util import ENGINES, TINY_DECODE, TINY_PRODUCE, check_agent, check_streams, run_deferred, run_streams

pytestmark = pytest.mark.gpu

R, PP = A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE
MiB = 1 << 20


def long_pieces():
    """Segments of more than 64 lines (several runs), and lines longer than a produce window, which pieces cut and the carry
    slot completes."""
    e = folds.element
    many = b"".join(folds.tc_chunk([e(k % 7, id=b"m%d" % k, name=b"n", args=b"%d," % k)]) for k in range(150)) + folds.STOP
    blanks = (b"data: {}\n" + b"\n" * 70) * 3 + folds.TAIL + folds.STOP
    wide = folds.tc_chunk([e(k, id=b"w%d" % k, name=b"f\\u00e9", args=b"x" * 300) for k in range(30)]) + folds.USAGE + folds.STOP
    return [many, blanks, wide]


@pytest.fixture(scope="module")
def bodies():
    c = folds.corpus(small=True)
    return [b for fam in c.values() for b in fam] + long_pieces()


@pytest.mark.parametrize("n_batches", [1, 3, 17])
@pytest.mark.parametrize("mode", [R, PP], ids=["R", "PP"])
def test_folds_on_the_kernels_records(engine, bodies, mode, n_batches):
    outs = run_streams(engine, bodies, [mode] * len(bodies), n_batches=n_batches, seed=n_batches, with_folds=True,
                       keep_codes=True)
    check_streams(bodies, mode, outs, f"folds x{n_batches}", engine.L)
    assert any(r != (A.SSE_OK, A.SSE_OK) for o in outs for _, *r in o.fold_rcs)      # the corpus reaches the depth rule


@pytest.fixture(scope="module", params=["split", "templates", "copy"])
def tiny(request):
    e = SseEngine(device=0, max_conns=512, bytes_per_batch=4 * MiB, flags=A.FLAG_DEFER | ENGINES[request.param],
                  **TINY_PRODUCE, **TINY_DECODE)
    yield e
    e.close()


@pytest.mark.parametrize("n_batches", [1, 17])
def test_folds_when_batches_defer(tiny, n_batches):
    c = folds.corpus(seed=1, n_adv=24)
    b = c["adversarial"] + c["tricky"][::3] + c["merge"] + c["near_misses"][::8] + long_pieces()
    modes = [(R, PP)[i % 2] for i in range(len(b))]
    outs, st = run_deferred(tiny, b, modes, n_batches=n_batches, seed=n_batches, with_folds=True, keep_codes=True)
    check_streams(b, modes, outs, f"deferred x{n_batches}", tiny.L)
    assert st["deferred"] > 0 and st["overflow"]


@pytest.mark.parametrize("mode", [R, PP], ids=["R", "PP"])
@pytest.mark.parametrize("eng", ["split", "templates", "copy"])
def test_saturated_tool_call_chains(eng, mode):
    """Lines of 65,534-65,537 tool-call elements, assembled in the line pool and decoded by the long-line kernel, next to C4
    streams, under SSE_FLAG_DEFER."""
    c4 = [b for b, _, _ in synth.make_config("C4", n_streams=64)[0]]
    b = folds.saturated_streams() + c4
    e = SseEngine(device=0, max_conns=128, bytes_per_batch=4 * MiB, flags=A.FLAG_DEFER | ENGINES[eng],
                  line_pool=dict(pool_pages=64, page_bytes=65536, max_line_bytes=512 * 1024))
    try:
        for nb in (1, 3):
            outs, st = run_deferred(e, b, [mode] * len(b), n_batches=nb, seed=nb, with_folds=True, keep_codes=True)
            check_streams(b, mode, outs, f"saturated x{nb}", e.L)
            for o, n in zip(outs, folds.SATURATED):
                assert max(len(r.get("tcs", ())) for r in o.recs) == n
    finally:
        e.close()


# ------------------------------------------------------------------ the gateway's agent path on the same streams
N_SLOTS = 4


def drive(g, bodies, seed, max_ticks=3000):
    """Mode R streams written in seeded pieces, one piece per stream and tick, closed after their last piece; pumps until every
    channel is closed. Returns (frames per stream, stream ids)."""
    rng = np.random.default_rng(seed)
    sids = [g.stream_chat_completions(R) for _ in bodies]
    queue = [random_cuts(rng, b, int(rng.integers(1, 7))) for b in bodies]
    frames, eof, left, closed = [[] for _ in bodies], [False] * len(bodies), [b""] * len(bodies), [False] * len(bodies)
    for _ in range(max_ticks):
        for i, s in enumerate(sids):
            if not left[i] and queue[i]:
                left[i] = queue[i].pop(0)
            if left[i]:
                left[i] = left[i][g.upstream_write(s, left[i]):]
        g.pump()
        for i, s in enumerate(sids):
            if not closed[i] and not left[i] and not queue[i]:
                g.upstream_close(s)
                closed[i] = True
            try:
                while (f := g.recv(s)) is not None:
                    frames[i].append(f)
            except EOFError:
                eof[i] = True
        if all(eof):
            break
    else:
        raise AssertionError("streams still open after max_ticks")
    assert g.flush() >= 0
    return frames, sids


@pytest.mark.parametrize("depth", [1, N_SLOTS])
@pytest.mark.parametrize("devices", [[0], [0, 0]], ids=lambda d: f"ctx{len(d)}")
def test_gateway_agent_on_adversarial_streams(devices, depth):
    c = folds.corpus(seed=2, n_adv=48)
    b = c["adversarial"] + c["tricky"] + c["merge"]
    cfg = A.Config()
    A.load().sse_worst_case_config(C.byref(cfg), len(b), 1 << 20)
    cfg.n_slots = N_SLOTS
    g = Gateway(config=cfg, devices=devices, depth=depth)
    try:
        frames, sids = drive(g, b, seed=depth)
        n_failed = 0
        for i, (body, got, s) in enumerate(zip(b, frames, sids)):
            v = orc.reframe(body)
            want = [l.out for l in v.lines if l.kind == orc.L_EMITTED]
            # frames up to and including the first line past the nesting limit (None: no such line)
            upto, n = None, 0
            for l in v.lines:
                n += l.kind == orc.L_EMITTED
                if l.kind != orc.L_UNREAD and l.depth_limited:
                    upto = n
                    break
            label = f"devices {devices} depth {depth} stream {i}"
            if upto is None:
                assert got == want, f"{label}: {len(got)} frames, oracle {len(want)}"
                check_agent(g.agent_state(s), v, label)
            else:
                # the stream is failed in the batch that holds its first line past the nesting limit: its channel ends after a
                # prefix of the oracle's frames that reaches that line
                n_failed += 1
                assert upto <= len(got) <= len(want) and got == want[:len(got)], f"{label}: not a prefix through the line"
        assert n_failed
    finally:
        g.close()
