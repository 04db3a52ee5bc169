"""GPU: a line pool that grows on demand (sse_line_pool_set_growth, SSE_FLAG_DEFER). A line that finds no free page defers its
segment at the byte that needed the page, sse_collect grows the pool, and the stream goes on bit-exact against the CPU oracle;
at the limit lines fail as without growth. Every batch passes orc_check_result."""
import numpy as np
import pytest

from inference_gateway_b200 import SseEngine, _abi as A
from inference_gateway_b200.gateway import Gateway
from tests import folds
from tests.gateway_drive import Session, check_sessions, drive, gateway_config
from tests.streams import PAGE, SLOT, burst, chunk, long_line, stream_with
from tests.util import (DONE, ENGINES, TINY_DECODE, ConnOut, check_folds, check_stream, check_streams, feed_folds, fold_segment,
                        pool_engine, process_all_checked, run_deferred, run_inflight, run_pieces_deferred)

pytestmark = pytest.mark.gpu

P, R, PP = A.MODE_P, A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE
MODES = (P, R, PP)
MiB = 1 << 20
SMALL_PAGE = 4096 + 16


# ------------------------------------------------------------------ 1: a burst far beyond the initial pool
@pytest.mark.parametrize("n_batches", [1, 3, 17])
@pytest.mark.parametrize("mode", MODES, ids=["P", "R", "PP"])
def test_burst_grows_the_pool(mode, n_batches):
    """40 connections complete 200 KB lines (4 pages each) in the same batches; the pool starts at 8 pages, the limit is 1024."""
    e = pool_engine(8, 1024, conns=64, batch=16 * MiB)
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
    e = pool_engine(initial, 256, conns=64, batch=8 * MiB, page_bytes=page)
    try:
        rng = np.random.default_rng(len(place))
        other = stream_with(long_line("toolcall", 300_000, rng), "toolcall")
        start = len(chunk(b"Hello")) + len(chunk(b"world"))
        line = long_line("content", length, rng)
        assert len(line) == length and (place != "newline" or line[PAGE:] == b"\n")
        body = line + b"\n" + chunk(b"bye", '"stop"') + DONE
        pieces = [[other[:start + held], b"", other[start + held:]], [b"", body]]
        e.reset_all()
        outs, _, deferrals, _ = run_pieces_deferred(e, pieces, [mode, mode])
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
    e = pool_engine(4, 8, conns=64, batch=8 * MiB)
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
    e = pool_engine(8, 0 if limit is None else 64, conns=64, batch=8 * MiB)
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
    e = pool_engine(8, 0, conns=16, batch=4 * MiB)
    try:
        for bad in (7, 0xFFFFFFFF):                         # below the capacity, SSE_NONE
            with pytest.raises(A.SseError):
                e.line_pool_growth(bad)
        e.line_pool_growth(8)
        assert e.line_pool_capacity() == (8, 8)
    finally:
        e.close()


# ------------------------------------------------------------------ 4: batches in flight
@pytest.mark.parametrize("depth", [2, 4])
def test_growth_with_batches_in_flight(depth):
    """depth batches of disjoint connections uncollected together: a collect grows the pool while later batches, launched with
    the old arrays, are still queued; those batches' own SSE_OVF_POOL does not grow it again; every stream matches the oracle."""
    e = pool_engine(8, 2048, conns=64, batch=8 * MiB)
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
    e = pool_engine(8, 2048, conns=128, batch=8 * MiB)
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
    e = pool_engine(8, 1024, conns=64, batch=8 * MiB, **TINY_DECODE)
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
    e = pool_engine(4, 1024, flags=A.FLAG_DEFER | ENGINES[name], conns=64, batch=8 * MiB, text_arena_bytes=32 * MiB)
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
@pytest.mark.parametrize("tap", [False, True], ids=["plain", "tapped"])
@pytest.mark.parametrize("devices,depth", [([0], 1), ([0], 4), ([0, 0], 1), ([0, 0], 4)])
def test_gateway_grows_its_pools(devices, depth, tap):
    seed = depth * 10 + len(devices)
    rng = np.random.default_rng(seed)
    bodies = burst(24, rng, size=150_000) + [chunk(b"short %d" % i) + chunk(b"end", '"stop"') + DONE for i in range(8)]
    sessions = [Session([b], (R, PP)[i % 2], tap=tap) for i, b in enumerate(bodies)]
    g = Gateway(config=gateway_config(len(sessions), flags=A.FLAG_DEFER), devices=devices, depth=depth,
                line_pool=dict(pool_pages=4, max_line_bytes=MiB, max_pages=4096))
    try:
        assert drive(g, sessions, seed, max_ticks=20000) >= 0
    finally:
        g.close()
    n_limited, _ = check_sessions(sessions, f"gateway {devices} depth {depth}")
    assert n_limited == 0
