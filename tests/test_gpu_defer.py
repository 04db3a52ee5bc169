"""GPU: SSE_FLAG_DEFER. Batches whose results do not fit the configured capacities are not failed: the produce stage defers what
does not fit to a later batch (sse_seg_result.consumed), the decode stage's arenas grow and the batch is decoded again. Every
stream must still come out bit-exact against the CPU oracle, however often it was deferred."""
import ctypes as C

import numpy as np
import pytest

from inference_gateway_b200 import SseEngine, _abi as A, synth
from inference_gateway_b200.gateway import Gateway
from inference_gateway_b200.synth import random_cuts
from oracle import orc
from tests.corpus import adversarial_bodies
from tests.util import (ENGINES, TINY_DECODE, TINY_PRODUCE, ConnOut, check_streams, fold_segment, process_all_checked,
                        process_checked)

pytestmark = pytest.mark.gpu

P, R, PP = A.MODE_P, A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE
MiB = 1 << 20


def run_deferred(eng, bodies, modes, n_batches=1, seed=0, with_folds=False, n_folds=None):
    """run_streams (tests/util.py) on an engine with SSE_FLAG_DEFER: every micro-batch of pieces is run to the end with
    SseEngine.process_all, which submits deferred remainders again until every byte was taken. The agent and telemetry folds
    are fed for the first n_folds streams (all by default). Returns (outs, stats)."""
    rng = np.random.default_rng(seed)
    L = eng.L
    outs = [ConnOut() for _ in bodies]
    eng.reset_all()
    pieces = [random_cuts(rng, b, n_batches) for b in bodies]
    if with_folds:
        for o in outs[:n_folds]:
            o.agent, o.tele = L.sse_agent_new(), L.sse_telemetry_new()
    stats = dict(batches=0, deferred=0, overflow=0)

    def on_batch(res, conns):
        stats["overflow"] |= res.overflow
        for i, c in enumerate(conns):
            o = outs[c]
            fold_segment(o, res, i)
            stats["deferred"] += bool(int(res.segs[i]["flags"]) & A.SEG_DEFERRED)
            if o.agent is not None:
                A.check(L.sse_agent_feed(o.agent, C.byref(res.raw), i), "sse_agent_feed")
                A.check(L.sse_telemetry_feed(o.tele, C.byref(res.raw), i), "sse_telemetry_feed")

    for b in range(max(len(p) for p in pieces)):
        items = [(c, modes[c], pieces[c][b]) for c in range(len(bodies)) if b < len(pieces[c])]
        stats["batches"] += process_all_checked(eng, items, on_batch)
    return outs, stats


N_C4 = 160


def mixed_bodies(seed, n_c4=N_C4, n_adv=60):
    """C4 streams, then adversarial ones (nesting past the 128-level limit among them: those records are flagged
    SSE_F_DEPTH_LIMIT, which check_stream compares with the oracle's restatement of the limit, and the folds refuse them, so
    only the C4 streams are folded)."""
    streams, _ = synth.make_config("C4", n_streams=n_c4)
    bodies = [b for b, _, _ in streams] + adversarial_bodies(np.random.default_rng(seed), n_adv)
    modes = [(P, R, PP)[i % 3] for i in range(len(bodies))]
    return bodies, modes


@pytest.fixture(scope="module", params=["split", "templates", "copy"])
def tiny(request):
    flags = A.FLAG_DEFER | ENGINES[request.param]
    e = SseEngine(device=0, max_conns=512, bytes_per_batch=4 * MiB, flags=flags, **TINY_PRODUCE)
    yield e
    e.close()


@pytest.mark.parametrize("n_batches", [1, 3, 17])
def test_produce_side_deferral_is_bit_exact(tiny, n_batches):
    bodies, modes = mixed_bodies(n_batches)
    outs, st = run_deferred(tiny, bodies, modes, n_batches=n_batches, seed=n_batches, with_folds=True, n_folds=N_C4)
    check_streams(bodies, modes, outs, f"tiny batches={n_batches}", tiny.L)
    assert st["deferred"] > 0 and st["overflow"] & (A.OVF_OUT | A.OVF_RUNS)
    assert not any(o.flags & A.SEG_DEAD for o in outs)


# ------------------------------------------------------------------ decode side: arenas grow, the batch is decoded again
def _tool_call_body(rng, n):
    parts = []
    for k in range(n):
        tcs = ",".join('{"index":%d,"id":"call_%d","type":"function","function":{"name":"f\\u00e9%d","arguments":"{\\"a\\":%d}"}}'
                       % (j, k, j, j) for j in range(int(rng.integers(1, 6))))
        parts.append(b'data: {"choices":[{"index":0,"delta":{"tool_calls":[%s]},"finish_reason":null}]}\n\n' % tcs.encode())
    parts.append(b'data: {"choices":[{"index":0,"delta":{},"finish_reason":"tool_calls"}]}\n\n')
    parts.append(b'data: {"choices":[],"usage":{"prompt_tokens":3,"completion_tokens":4,"total_tokens":7}}\n\ndata: [DONE]\n\n')
    return b"".join(parts)


def _bad_utf8_body(rng, n):
    parts = []
    for _ in range(n):
        junk = bytes(int(x) for x in rng.integers(0x80, 0x100, size=int(rng.integers(8, 120))))
        parts.append(b'data: {"choices":[{"index":0,"delta":{"content":"' + junk + b'"},"finish_reason":null}],'
                     b'"usage":{"prompt_tokens":1,"completion_tokens":2,"total_tokens":3}}\n\n')
    return b"".join(parts) + b"data: [DONE]\n\n"


@pytest.mark.parametrize("flags", [0, A.FLAG_TEMPLATES], ids=["split", "templates"])
def test_decode_side_arenas_grow_and_the_batch_is_decoded_again(flags):
    rng = np.random.default_rng(3)
    bodies = [_tool_call_body(rng, 30) for _ in range(24)] + [_bad_utf8_body(rng, 20) for _ in range(24)]
    modes = [(R, PP)[i % 2] for i in range(len(bodies))]
    e = SseEngine(device=0, max_conns=64, bytes_per_batch=1 * MiB, flags=A.FLAG_DEFER | flags, n_slots=1, **TINY_DECODE)
    try:
        outs, st = run_deferred(e, bodies, modes, n_batches=2, seed=1, with_folds=True)
        check_streams(bodies, modes, outs, "decode growth", e.L)
        grown = A.OVF_TCS | A.OVF_USAGES | A.OVF_TEXT
        assert st["overflow"] & grown == grown and st["deferred"] == 0
        # the slot keeps what it grew to: the same batches again need no second pass
        outs, st = run_deferred(e, bodies, modes, n_batches=2, seed=1, with_folds=True)
        check_streams(bodies, modes, outs, "decode growth, second run", e.L)
        assert st["overflow"] == 0
    finally:
        e.close()


# ------------------------------------------------------------------ the cases that have to be exactly right
def test_deferral_at_a_first_line_that_starts_in_the_carried_tail():
    """Every segment of the batch continues a line held back by the previous batch, and the first round of each needs 64 frames
    while the batch has 128: almost all of them are deferred before their first line, which starts in the carry. They must take
    nothing (consumed 0) and keep their carry as it was; resubmitted, they come out bit-exact."""
    e = SseEngine(device=0, max_conns=64, bytes_per_batch=1 * MiB, flags=A.FLAG_DEFER, max_frames=128, max_recs=64, max_runs=0)
    try:
        head = b'data: {"choices":[{"index":0,"delta":{"content":"held'
        rest = b'"},"finish_reason":null}]}\n' + b"data: {}\n" * 200
        bodies = [head + rest for _ in range(48)]
        outs = [ConnOut() for _ in bodies]
        e.reset_all()
        slot, res = process_checked(e, [(c, PP, head) for c in range(len(bodies))])
        try:
            assert all(int(res.segs[i]["carry_len"]) == len(head) for i in range(len(bodies)))
        finally:
            e.release(slot)
        seen = []

        def on_batch(res, conns):
            for i, c in enumerate(conns):
                fl = int(res.segs[i]["flags"])
                if fl & A.SEG_DEFERRED and not outs[c].frames and res.consumed(i) == 0:
                    seen.append(int(res.segs[i]["carry_len"]))
                fold_segment(outs[c], res, i)
        process_all_checked(e, [(c, PP, rest) for c in range(len(bodies))], on_batch)
        assert len(seen) >= len(bodies) - 2 and set(seen) == {len(head)}
        check_streams(bodies, PP, outs, "carry")
    finally:
        e.close()


def test_terminating_chunk_before_deferred_bytes_finishes_the_connection():
    """Mode R: the round that holds the terminating chunk is admitted, the next round is deferred (no runs[] entry is free).
    The connection still ends FINISHED, nothing is left to resubmit, and bytes sent anyway are ignored."""
    e = SseEngine(device=0, max_conns=8, bytes_per_batch=1 * MiB, flags=A.FLAG_DEFER, max_runs=0)
    try:
        stop = b'data: {"choices":[{"index":0,"delta":{"content":"bye"},"finish_reason":"stop"}]}\n\n'
        more = b'data: {"choices":[{"index":0,"delta":{"content":"never read"},"finish_reason":null}]}\n\n' * 100
        body = stop + more
        e.reset_all()
        slot, res = process_checked(e, [(0, R, body)])
        try:
            fl = int(res.segs[0]["flags"])
            assert fl & A.SEG_TERMINATED and not fl & A.SEG_DEFERRED and res.consumed(0) == len(body)
            assert res.overflow & A.OVF_RUNS                      # the batch did defer the round after the terminating one
            assert res.seg_frames(0) == [stop]
        finally:
            e.release(slot)
        slot, res = process_checked(e, [(0, R, more)])
        try:
            assert int(res.segs[0]["flags"]) & A.SEG_FINISHED and res.seg_frames(0) == [] and res.consumed(0) == len(more)
        finally:
            e.release(slot)
    finally:
        e.close()


def test_pooled_line_whose_completion_does_not_fit_waits_at_its_newline():
    """Two connections complete a pooled 1 MiB line in the same batch; the out arena holds one. The other line stays in its
    pages, its segment stops at the '\\n' (consumed is the '\\n''s offset, 0), and the next batch completes it. No page leaks."""
    e = SseEngine(device=0, max_conns=64, bytes_per_batch=4 * MiB, flags=A.FLAG_DEFER, out_arena_bytes=1 * MiB,
                  line_pool=dict(pool_pages=40, page_bytes=65536, max_line_bytes=1200 * 1024))
    try:
        assert MiB + 64 < e.cfg.out_arena_bytes < 2 * MiB
        rng = np.random.default_rng(9)
        pre = b'data: {"choices":[{"index":0,"delta":{"tool_calls":[{"index":0,"id":"c","type":"function","function":{"name":"w","arguments":"'
        post = b'"}}]},"finish_reason":null}]}\n'
        body_chars = bytes(int(x) for x in rng.integers(0x61, 0x7B, size=MiB))
        lines = [pre + body_chars[:MiB - k * 100] + post for k in range(2)]
        tails = [b"\n" + b'data: {"choices":[{"index":0,"delta":{},"finish_reason":"stop"}]}\n\n' for _ in lines]
        bodies = [l + t for l, t in zip(lines, tails)]
        outs = [ConnOut() for _ in bodies]
        e.reset_all()
        first = [(c, R, l[:-1]) for c, l in enumerate(lines)]             # everything but the '\n': held in the pool
        second = [(c, R, b"\n" + t) for c, t in enumerate(tails)]
        stops = []

        def on_batch(res, conns):
            for i, c in enumerate(conns):
                fl = int(res.segs[i]["flags"])
                if fl & A.SEG_DEFERRED:
                    stops.append(res.consumed(i))
                fold_segment(outs[c], res, i)
        assert process_all_checked(e, first, on_batch) == 1 and e.pool_stats()[0] > 0
        n = process_all_checked(e, second, on_batch)
        # one line waited, at its '\n' (consumed 0); the other completed, and what followed it may have waited too (the failed
        # reservation left the out-arena counter past the capacity)
        assert n == 2 and stops.count(0) == 1 and all(c in (0, 1) for c in stops)
        check_streams(bodies, R, outs, "pooled")
        assert all(o.terminated for o in outs)
        assert e.pool_stats()[0] == 0
    finally:
        e.close()


@pytest.mark.parametrize("keep", [16383, 16384, 16385, 20480], ids=lambda k: f"keep{k}")
def test_line_whose_newline_would_leave_the_carry_slot_keeps_its_bytes_when_deferred(keep):
    """Lines held in the 16 KiB carry slot across batches whose completion is deferred at the '\\n'. keep = bytes before the
    '\\n': 16384 is the case where the '\\n' is the byte that moves the line out of the slot into pool pages; giving the '\\n'
    back must leave every byte of the line in the slot (the slot had only the bytes of earlier windows). 16383 stays in the slot,
    16385 is in the pool already, 20480 (five 4 KiB pages) is the case where the '\\n' took a page of its own. Eight connections
    finish such a line in the same batch and the out arena holds one completion at a time, so all but one wait at least once."""
    slot = 16384
    e = SseEngine(device=0, max_conns=16, bytes_per_batch=1 * MiB, flags=A.FLAG_DEFER, carry_slot_bytes=slot, out_arena_bytes=24 * 1024,
                  line_pool=dict(pool_pages=64, page_bytes=4096, max_line_bytes=24000))
    try:
        cap = e.cfg.out_arena_bytes
        assert ((keep + 3 + 15) & ~15) + 16 <= cap < 2 * (((16384 + 3 + 15) & ~15) + 16)
        rng = np.random.default_rng(keep)
        pre, post = b'data: {"choices":[{"index":0,"delta":{"content":"', b'"},"finish_reason":null}]}'
        bodies = []
        for c in range(8):
            fill = bytes(int(x) for x in rng.integers(0x61, 0x7B, size=keep - len(pre) - len(post)))
            line = pre + fill + post
            assert len(line) == keep
            bodies.append(line + b"\n" + b'data: {"choices":[{"index":0,"delta":{"content":"end %d"},"finish_reason":"stop"}]}\n\n' % c)
        outs = [ConnOut() for _ in bodies]
        waited, taken, second = set(), [0] * len(bodies), [False]

        def on_batch(res, conns):
            for i, c in enumerate(conns):
                fl = int(res.segs[i]["flags"])
                frames = res.seg_frames(i)
                if second[0]:
                    if fl & A.SEG_DEFERRED and not outs[c].frames and not frames:
                        # the line did not complete: its segment stopped exactly at the line's '\\n'
                        assert taken[c] + res.consumed(i) == keep - 10000, (c, taken[c], res.consumed(i))
                        waited.add(c)
                    taken[c] += res.consumed(i)
                fold_segment(outs[c], res, i)
        e.reset_all()
        # 10,000 bytes without a '\\n': more than a window, so the line is assembled in the slot (not yet in the pool)
        assert process_all_checked(e, [(c, PP, b[:10000]) for c, b in enumerate(bodies)], on_batch) == 1
        assert all(o.carry_len == 10000 for o in outs) and e.pool_stats()[0] == 0
        second[0] = True
        assert process_all_checked(e, [(c, PP, b[10000:]) for c, b in enumerate(bodies)], on_batch) >= 8
        assert len(waited) >= 7 and taken == [len(b) - 10000 for b in bodies]
        check_streams(bodies, PP, outs, f"keep={keep}")
        assert not any(o.flags & A.SEG_DEAD for o in outs)
        assert e.pool_stats()[0] == 0
    finally:
        e.close()


# ------------------------------------------------------------------ gateway mirror on a default-sized config
def test_gateway_on_default_capacities_with_defer_survives_a_blank_line_flood():
    """test_one_stream_of_blank_lines_cannot_starve_or_overflow_the_batch (tests/test_gpu_gateway.py) with sse_default_config
    capacities, far below the worst case: the flood of one-frame-per-byte lines is deferred batch after batch instead of
    failing the batch, every good stream gets the oracle's frames and one [DONE], and the flood is delivered whole."""
    L = A.load()
    cfg = A.Config()
    L.sse_default_config(C.byref(cfg), 8, 1 << 16)
    cfg.flags = A.FLAG_DEFER
    worst = A.Config()
    L.sse_worst_case_config(C.byref(worst), 8, 1 << 16)
    assert cfg.max_frames * 10 < worst.max_frames
    g = Gateway(device=0, config=cfg)
    try:
        evil = g.proxy_stream()
        good = [g.stream_chat_completions(R) for _ in range(3)]
        ok_body = (b'data: {"choices":[{"index":0,"delta":{"content":"hi"},"finish_reason":null}]}\n\n'
                   b'data: {"choices":[{"index":0,"delta":{},"finish_reason":"stop"}]}\n\n')
        flood = b"\n" * 100000
        sent = got_evil = 0
        good_out = {s: [] for s in good}
        for s in good:
            assert g.upstream_write(s, ok_body) == len(ok_body)
        for _ in range(2000):
            if sent < len(flood):
                sent += g.upstream_write(evil, flood[sent:sent + 30000])
            g.pump()
            while (e := g.proxy_step(evil)) is not None:
                assert e == b"\n"
                got_evil += 1
            for s in good:
                try:
                    while (e := g.agent_recv(s)) is not None:
                        good_out[s].append(e)
                except EOFError:      # the iteration is over: terminating chunk seen and its [DONE] delivered
                    pass
            if got_evil == len(flood) and all(len(v) == 3 for v in good_out.values()):
                break
        assert got_evil == len(flood)
        want = [l.out for l in orc.reframe(ok_body).lines if l.kind == orc.L_EMITTED] + [b"data: [DONE]\n\n"]
        for s in good:
            assert good_out[s] == want
    finally:
        g.close()


def test_without_the_flag_the_same_capacities_still_fail_the_batch():
    bodies, modes = mixed_bodies(0, n_c4=64, n_adv=8)
    e = SseEngine(device=0, max_conns=512, bytes_per_batch=4 * MiB, **TINY_PRODUCE)
    try:
        e.reset_all()
        with pytest.raises(A.SseError) as ex:
            slot, _ = e.process([(c, m, b) for c, (b, m) in enumerate(zip(bodies, modes))])
        assert ex.value.status == A.SSE_ERR_OVERFLOW
        e.release(0)
    finally:
        e.close()
