"""GPU: a line pool that grows on demand (sse_line_pool_set_growth, SSE_FLAG_DEFER). A line that finds no free page defers its
segment at the byte that needed the page, sse_collect grows the pool, and the stream goes on bit-exact against the CPU oracle;
at the limit lines fail as without growth. Every batch passes orc_check_result."""
import ctypes as C

import numpy as np
import pytest

from inference_gateway_b200 import SseEngine, _abi as A
from inference_gateway_b200.gateway import Gateway, Telemetry
from inference_gateway_b200.synth import random_cuts
from oracle import orc
from tests import folds
from tests.streams import PAGE, SLOT, chunk, long_line, stream_with
from tests.util import (ENGINES, TINY_DECODE, ConnOut, check_agent, check_folds, check_result, check_stream, check_streams,
                        feed_folds, fold_segment, irregular_telemetry, process_all_checked, run_deferred)

pytestmark = pytest.mark.gpu

P, R, PP = A.MODE_P, A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE
MODES = (P, R, PP)
MiB = 1 << 20
SMALL_PAGE = 4096 + 16
DONE = b"data: [DONE]\n\n"


def engine(pages, max_pages, flags=0, page_bytes=PAGE, conns=64, batch=8 * MiB, n_slots=4, **caps):
    return SseEngine(device=0, max_conns=conns, bytes_per_batch=batch, carry_slot_bytes=SLOT, n_slots=n_slots,
                     flags=A.FLAG_DEFER | flags, **caps,
                     line_pool=dict(pool_pages=pages, page_bytes=page_bytes, max_line_bytes=2 * MiB, max_pages=max_pages))


def burst(n, rng, size=200_000, kinds=("toolcall", "content", "terminal")):
    return [stream_with(long_line(kinds[i % len(kinds)], size + 1009 * i, rng), kinds[i % len(kinds)]) for i in range(n)]


def run_pieces_deferred(eng, pieces, modes):
    """pieces[c][b] goes to connection c in batch b; every batch is run to the end (SseEngine.process_all, checked), its
    deferred rests first in the next batch. Returns (outs, deferrals: (connection, consumed, batch overflow), overflow bits)."""
    outs = [ConnOut() for _ in pieces]
    eng.reset_all()
    deferrals, ovf = [], [0]

    def on_batch(res, conns):
        ovf[0] |= res.overflow
        for i, c in enumerate(conns):
            fold_segment(outs[c], res, i)
            if int(res.segs[i]["flags"]) & A.SEG_DEFERRED:
                deferrals.append((c, res.consumed(i), res.overflow))
    for b in range(max(map(len, pieces))):
        process_all_checked(eng, [(c, modes[c], pieces[c][b]) for c in range(len(pieces)) if b < len(pieces[c])], on_batch)
    return outs, deferrals, ovf[0]


# ------------------------------------------------------------------ 1: a burst far beyond the initial pool
@pytest.mark.parametrize("n_batches", [1, 3, 17])
@pytest.mark.parametrize("mode", MODES, ids=["P", "R", "PP"])
def test_burst_grows_the_pool(mode, n_batches):
    """40 connections complete 200 KB lines (4 pages each) in the same batches; the pool starts at 8 pages, the limit is 1024."""
    e = engine(8, 1024, batch=16 * MiB)
    try:
        rng = np.random.default_rng(n_batches * 7 + mode)
        bodies = burst(40, rng)
        outs, st = run_deferred(e, bodies, [mode] * len(bodies), n_batches=n_batches, seed=n_batches)
        check_streams(bodies, [mode] * len(bodies), outs, f"burst mode {mode} batches {n_batches}")
        assert not any(o.flags & (A.SEG_DEAD | A.SEG_LINE_TOO_LONG) for o in outs)
        assert st["overflow"] & A.OVF_POOL and st["deferred"] > 0
        pages, limit = e.line_pool_capacity()
        assert limit == 1024 and 8 < pages <= 1024
        used, hw = e.pool_stats()
        assert used == 0 and 8 < hw <= pages
    finally:
        e.close()


# ------------------------------------------------------------------ 2: every place a line takes a page
# (page bytes, initial pages, bytes connection 0 holds in the pool, connection 1's line length, where its first deferral lands)
# The second connection's line starts its segment, so its windows end at multiples of 8192 bytes of the line.
PLACES = {
    # no page free when the line leaves the carry slot: the slot is filled to its end
    "slot": (PAGE, 1, 40_000, 100_000, SLOT),
    # the line leaves the slot with the last free page; the next page boundary (65,536 = 8 windows) is a window's end
    "window_end": (PAGE, 2, 40_000, 200_000, PAGE),
    # 10 free pages of 4,112 bytes: the line leaves the slot with all of them and stops at 41,120, 160 bytes into a window
    "inside": (SMALL_PAGE, 20, 40_000, 100_000, 10 * SMALL_PAGE),
    # the line's '\n' is the first byte of a page that is not free: the line waits with exactly one page, the '\n' first
    "newline": (PAGE, 2, 40_000, PAGE + 1, PAGE),
}


@pytest.mark.parametrize("place", list(PLACES))
@pytest.mark.parametrize("mode", [P, R], ids=["P", "R"])
def test_deferral_lands_where_the_page_was_needed(place, mode):
    page, initial, held, length, at = PLACES[place]
    assert at % 8192 == (0 if place in ("slot", "window_end", "newline") else 160)
    e = engine(initial, 256, page_bytes=page)
    try:
        rng = np.random.default_rng(len(place))
        other = stream_with(long_line("toolcall", 300_000, rng), "toolcall")
        start = len(chunk(b"Hello")) + len(chunk(b"world"))
        line = long_line("content", length, rng)
        assert len(line) == length and (place != "newline" or line[PAGE:] == b"\n")
        body = line + b"\n" + chunk(b"bye", '"stop"') + DONE
        pieces = [[other[:start + held], b"", other[start + held:]], [b"", body]]
        outs, deferrals, ovf = run_pieces_deferred(e, pieces, [mode, mode])
        for b, o in ((other, outs[0]), (body, outs[1])):
            check_stream(b, mode, o, f"{place} mode {mode}")
        assert not any(o.flags & (A.SEG_DEAD | A.SEG_LINE_TOO_LONG) for o in outs)
        first = next(d for d in deferrals if d[0] == 1)
        assert first[1] == at and first[2] & A.OVF_POOL, (place, deferrals[:4])
        assert e.line_pool_capacity()[0] > initial and e.pool_stats()[0] == 0
    finally:
        e.close()


# ------------------------------------------------------------------ 3: the limit
def test_limit_stops_growth_and_fails_only_the_unlucky():
    """Twelve 200 KB lines (4 pages each) at once on a pool of 4 pages that may grow to 8: capacity stops at 8, the connections
    that then found no page fail, the others match the oracle."""
    e = engine(4, 8)
    try:
        rng = np.random.default_rng(3)
        bodies = burst(12, rng, kinds=("toolcall",))
        modes = [MODES[i % 3] for i in range(12)]
        outs, st = run_deferred(e, bodies, modes, n_batches=1)
        ok = dead = 0
        for i, (b, m, o) in enumerate(zip(bodies, modes, outs)):
            if o.flags & A.SEG_DEAD:
                assert o.flags & A.SEG_LINE_TOO_LONG
                dead += 1
            else:
                check_stream(b, m, o, f"limit stream {i}")
                ok += 1
        assert ok >= 1 and dead >= 1 and st["overflow"] & A.OVF_POOL
        assert e.line_pool_capacity() == (8, 8)
        for c in range(12):
            e.reset_conn(c)
        used, hw = e.pool_stats()
        assert used == 0 and hw <= 8
    finally:
        e.close()


@pytest.mark.parametrize("limit", [None, 0], ids=["never_set", "set_to_0"])
def test_without_growth_the_pool_fails_as_before(limit):
    """The same shape with growth never enabled, or disabled again: no SSE_OVF_POOL, no pool deferral, the capacity stays,
    and each connection completes bit-exact or fails LINE_TOO_LONG | DEAD."""
    e = engine(8, 0 if limit is None else 64)
    try:
        if limit is not None:
            e.line_pool_growth(0)
        assert e.line_pool_capacity() == (8, 0)
        rng = np.random.default_rng(4)
        bodies = burst(12, rng, kinds=("toolcall",))
        modes = [MODES[i % 3] for i in range(12)]
        outs, st = run_deferred(e, bodies, modes, n_batches=1)
        dead = 0
        for i, (b, m, o) in enumerate(zip(bodies, modes, outs)):
            if o.flags & A.SEG_DEAD:
                assert o.flags & A.SEG_LINE_TOO_LONG
                dead += 1
            else:
                check_stream(b, m, o, f"no growth stream {i}")
        assert dead > 0 and not st["overflow"] & A.OVF_POOL and e.line_pool_capacity() == (8, 0)
    finally:
        e.close()


def test_setter_refusals():
    e = SseEngine(device=0, max_conns=16, bytes_per_batch=MiB, carry_slot_bytes=SLOT, line_pool=dict(pool_pages=8))
    try:
        with pytest.raises(A.SseError):                      # no SSE_FLAG_DEFER
            e.line_pool_growth(64)
    finally:
        e.close()
    e = SseEngine(device=0, max_conns=16, bytes_per_batch=MiB, carry_slot_bytes=SLOT, flags=A.FLAG_DEFER)
    try:
        with pytest.raises(A.SseError):                      # no pool
            e.line_pool_growth(64)
    finally:
        e.close()
    e = engine(8, 0, conns=16, batch=4 * MiB)
    try:
        for bad in (7, 0xFFFFFFFF):                         # below the capacity, SSE_NONE
            with pytest.raises(A.SseError):
                e.line_pool_growth(bad)
        e.line_pool_growth(8)
        assert e.line_pool_capacity() == (8, 8)
    finally:
        e.close()


# ------------------------------------------------------------------ 4: batches in flight
def run_inflight(eng, bodies, modes, depth, n_pieces, seed, between=None, abandon=None):
    """Up to depth uncollected batches. Connection c belongs to group c % depth and a batch takes the ready connections of one
    group (the next group, in turn, that has any), so that depth batches of disjoint connections are uncollected together. A
    connection goes into a batch only while it is in no uncollected one, and a deferred rest goes back to the front of its
    queue when its batch is collected. between(k) runs after submit k; abandon(k) may return (conn, mode, bytes) items for a
    batch that is submitted after submit k and released without being collected.
    Returns (outs, per-batch overflow bits, events): events["grew_in_flight"] counts collects that grew the pool while other
    batches were uncollected (launched with the old pool's arrays), events["stale_pool"] batches that reported SSE_OVF_POOL after
    the pool had grown since their submit, whose collect did not grow it again."""
    rng = np.random.default_rng(seed)
    queue = [random_cuts(rng, b, n_pieces) for b in bodies]
    outs = [ConnOut() for _ in bodies]
    busy, inflight, k, g_next, ovf = set(), [], 0, 0, []
    events = dict(grew_in_flight=0, stale_pool=0, max_in_flight=0)
    eng.reset_all()
    while any(queue) or inflight:
        group = None
        if len(inflight) < depth:
            for j in range(depth):
                g = (g_next + j) % depth
                if any(queue[c] and c not in busy for c in range(g, len(bodies), depth)):
                    group = g
                    break
        if group is not None:
            g_next = group + 1
            items = [(c, modes[c], queue[c].pop(0)) for c in range(group, len(bodies), depth) if queue[c] and c not in busy]
            slot, arena, segs = eng.acquire()
            n, nbytes = eng.fill(arena, segs, items)
            eng.submit(slot, n, nbytes)
            inflight.append((slot, items, segs[:n].copy(), eng.line_pool_capacity()[0]))
            events["max_in_flight"] = max(events["max_in_flight"], len(inflight))
            busy.update(c for c, _, _ in items)
            if between is not None:
                between(k)
            extra = abandon(k) if abandon is not None else None
            if extra:
                s2, a2, g2 = eng.acquire()
                eng.submit(s2, *eng.fill(a2, g2, extra))
                eng.release(s2)
            k += 1
            continue
        slot, items, segs, pages_at_submit = inflight.pop(0)
        try:
            before = eng.line_pool_capacity()[0]
            res = eng.collect(slot)
            after = eng.line_pool_capacity()[0]
            check_result(eng, res, segs)
            ovf.append(res.overflow)
            if after > before and inflight:
                events["grew_in_flight"] += 1
            if res.overflow & A.OVF_POOL and pages_at_submit != before:
                assert after == before, "a batch launched before a growth grew the pool again"
                events["stale_pool"] += 1
            for i, (c, m, data) in enumerate(items):
                fold_segment(outs[c], res, i)
                busy.discard(c)
                if int(res.segs[i]["flags"]) & A.SEG_DEFERRED:
                    queue[c].insert(0, data[res.consumed(i):])
        finally:
            eng.release(slot)
    return outs, ovf, events


@pytest.mark.parametrize("depth", [2, 4])
def test_growth_with_batches_in_flight(depth):
    """depth batches of disjoint connections uncollected together: a collect grows the pool while later batches, launched with
    the old arrays, are still queued; those batches' own SSE_OVF_POOL does not grow it again; every stream matches the oracle."""
    e = engine(8, 2048)
    try:
        rng = np.random.default_rng(depth)
        bodies = burst(36, rng)
        modes = [MODES[i % 3] for i in range(len(bodies))]
        stats = []
        outs, ovf, ev = run_inflight(e, bodies, modes, depth, n_pieces=2, seed=depth, between=lambda k: stats.append(e.pool_stats()))
        check_streams(bodies, modes, outs, f"in flight depth {depth}")
        assert not any(o.flags & A.SEG_DEAD for o in outs) and any(x & A.OVF_POOL for x in ovf)
        assert ev["max_in_flight"] == depth and ev["grew_in_flight"] >= 1 and ev["stale_pool"] >= 1, ev
        assert all(u <= hw for u, hw in stats) and e.line_pool_capacity()[0] > 8 and e.pool_stats()[0] == 0
    finally:
        e.close()


def test_resets_stats_and_an_abandoned_batch_between_submits():
    """sse_reset_conn and sse_line_pool_stats after every submit, and batches of other connections (long lines that take and
    lack pages) released without being collected: the pool grows only at collect, the abandoned connections' pages come back
    with their resets, and the collected streams match the oracle."""
    e = engine(8, 2048, conns=128)
    try:
        rng = np.random.default_rng(8)
        bodies = burst(24, rng)
        modes = [MODES[i % 3] for i in range(len(bodies))]
        junk = burst(8, rng, size=150_000)

        def between(k):
            e.pool_stats()
            e.reset_conn(100 + k % 8)

        def abandon(k):
            return [(100 + j, P, junk[j][:180_000]) for j in range(8)] if k % 3 == 0 else None
        outs, ovf, _ = run_inflight(e, bodies, modes, 3, n_pieces=4, seed=8, between=between, abandon=abandon)
        check_streams(bodies, modes, outs, "resets and abandoned batches")
        assert not any(o.flags & A.SEG_DEAD for o in outs)
        for j in range(8):
            e.reset_conn(100 + j)
        assert e.pool_stats()[0] == 0
    finally:
        e.close()


def test_pool_and_decode_arenas_grow_in_the_same_batch():
    """Tiny tool-call, usage and text arenas: one batch whose long lines lack pages (SSE_OVF_POOL) also grows the tool-call
    and text arenas and is decoded again; streams and folds match the oracle."""
    e = engine(8, 1024, **TINY_DECODE)
    try:
        rng = np.random.default_rng(12)
        tc = b"".join(b'data: {"choices":[{"index":0,"delta":{"tool_calls":[{"index":%d,"id":"c%d","function":{"name":"f",'
                      b'"arguments":"\\u00e9\\n%d"}}]},"finish_reason":null}]}\n\n' % (k, k, k) for k in range(24))
        bodies = [tc + b for b in burst(30, rng)]
        modes = [MODES[i % 3] for i in range(len(bodies))]
        outs = [ConnOut() for _ in bodies]
        for o, b in zip(outs, bodies):      # one piece per stream, fed to both folds
            o.agent, o.tele, o.piece_ends = e.L.sse_agent_new(), e.L.sse_telemetry_new(), [len(b)]
        per_batch = []

        def on_batch(res, conns):
            per_batch.append(res.overflow)
            for i, c in enumerate(conns):
                fold_segment(outs[c], res, i)
                feed_folds(e.L, outs[c], res, i, 0, False)
        e.reset_all()
        process_all_checked(e, [(c, modes[c], bodies[c]) for c in range(len(bodies))], on_batch)
        views = check_streams(bodies, modes, outs, "pool and decode growth")
        for i, (m, o) in enumerate(zip(modes, outs)):
            check_folds(e.L, o, m, views[i], f"pool and decode growth stream {i}")
            e.L.sse_agent_free(o.agent)
            e.L.sse_telemetry_free(o.tele)
        need = A.OVF_POOL | A.OVF_TCS | A.OVF_TEXT
        assert any(x & need == need for x in per_batch), [hex(x) for x in per_batch]
    finally:
        e.close()


# ------------------------------------------------------------------ 5: engines and folds
@pytest.mark.parametrize("name", ["split", "copy", "templates"])
def test_engines_and_folds_on_grown_pages(name):
    """The split engines, each on a pool of 4 pages that grows: saturated tool-call chains (65,534-65,537 elements) and long
    tool-call arguments complete in grown pages; frames and records match the oracle, and the agent and telemetry folds too."""
    e = engine(4, 1024, flags=ENGINES[name], text_arena_bytes=32 * MiB)
    try:
        rng = np.random.default_rng(21)
        big = folds.saturated_streams() + [stream_with(long_line("toolcall", 400_000 + 5000 * i, rng), "toolcall") for i in range(6)]
        bodies = big + big
        modes = [R] * len(big) + [PP] * len(big)
        for nb in (1, 5):
            outs, st = run_deferred(e, bodies, modes, n_batches=nb, seed=nb, with_folds=True)
            views = check_streams(bodies, modes, outs, f"{name} batches {nb}")
            for i, (m, o) in enumerate(zip(modes, outs)):
                check_folds(e.L, o, m, views[i], f"{name} batches {nb} stream {i}")
            assert not any(o.flags & A.SEG_DEAD for o in outs)
            for o in outs:
                e.L.sse_agent_free(o.agent)
                e.L.sse_telemetry_free(o.tele)
        assert e.line_pool_capacity()[0] > 4 and e.pool_stats()[0] == 0
    finally:
        e.close()


# ------------------------------------------------------------------ 6: the gateway
def gw_config(conns, batch=1 << 20):
    cfg = A.Config()
    A.load().sse_default_config(C.byref(cfg), conns, batch)
    cfg.n_slots = 4
    cfg.flags = A.FLAG_DEFER
    return cfg


@pytest.mark.parametrize("tap", [False, True], ids=["plain", "tapped"])
@pytest.mark.parametrize("devices,depth", [([0], 1), ([0], 4), ([0, 0], 1), ([0, 0], 4)])
def test_gateway_grows_its_pools(devices, depth, tap):
    rng = np.random.default_rng(depth * 10 + len(devices))
    bodies = burst(24, rng, size=150_000) + [chunk(b"short %d" % i) + chunk(b"end", '"stop"') + DONE for i in range(8)]
    modes = [(R, PP)[i % 2] for i in range(len(bodies))]
    g = Gateway(config=gw_config(len(bodies)), devices=devices, depth=depth,
                line_pool=dict(pool_pages=4, max_line_bytes=MiB, max_pages=4096))
    taps = [Telemetry() if tap else None for _ in bodies]
    try:
        sids = [g.stream_chat_completions(m, telemetry=t) if t is not None else g.stream_chat_completions(m)
                for m, t in zip(modes, taps)]
        queue = [random_cuts(rng, b, 6) for b in bodies]
        left = [b""] * len(bodies)
        frames = [[] for _ in bodies]
        eof = [False] * len(bodies)
        closed = [False] * len(bodies)
        for _ in range(20000):
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
                try:
                    while not eof[i] and (f := g.recv(sid)) is not None:
                        frames[i].append(f)
                except EOFError:
                    eof[i] = True
            if all(eof):
                break
        else:
            raise AssertionError("streams still open")
        assert g.flush() >= 0
        for i, (b, m, sid) in enumerate(zip(bodies, modes, sids)):
            if m == R:
                v = orc.reframe(b)
                want = [l.out for l in v.lines if l.kind == orc.L_EMITTED]
                check_agent(g.agent_state(sid), v, f"gateway stream {i}")
            else:
                want = [l.out for l in orc.passthrough(b, parse=True).lines]
            assert frames[i] == want, f"gateway {devices} depth {depth} stream {i}: {len(frames[i])} frames, oracle {len(want)}"
            if taps[i] is not None:
                body = b"".join(frames[i]) + (DONE if m == R else b"")
                if m == R:
                    taps[i].feed_bytes(DONE)
                rc, usage, calls = taps[i].finish()
                if irregular_telemetry(body):
                    assert rc == 1
                else:
                    assert (rc, usage, calls) == (0, *orc.telemetry(body)), f"gateway stream {i}: telemetry differs"
            g.release(sid)
    finally:
        g.close()
        for t in taps:
            if t is not None:
                t.close()
