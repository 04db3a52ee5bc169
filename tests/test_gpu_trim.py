"""GPU: sse_trim gives back what on-demand growth took. A grown line pool shrinks to max(min, pages held, 1) pages with the held
pages repacked on the device, and lines held across the trim complete bit-exact against the CPU oracle; grown decode arenas go
back to the config at once or at the slot's release; sse_memory_held returns to a fresh context's value. Every batch passes
orc_check_result."""
import ctypes as C

import numpy as np
import pytest

from inference_gateway_b200 import SseEngine, _abi as A
from inference_gateway_b200.gateway import Gateway, Telemetry
from inference_gateway_b200.synth import random_cuts
from oracle import orc
from tests import folds
from tests.streams import PAGE, SLOT, chunk, long_line, stream_with
from tests.util import (TINY_DECODE, ConnOut, check_agent, check_folds, check_result, check_streams, feed_folds, fold_segment,
                        irregular_telemetry, process_all_checked, process_checked)

pytestmark = pytest.mark.gpu

P, R, PP = A.MODE_P, A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE
MODES = (P, R, PP)
MiB = 1 << 20
DONE = b"data: [DONE]\n\n"
INITIAL = 8


def engine(pages=INITIAL, max_pages=1024, flags=A.FLAG_DEFER, conns=128, batch=16 * MiB, n_slots=4, **caps):
    return SseEngine(device=0, max_conns=conns, bytes_per_batch=batch, carry_slot_bytes=SLOT, n_slots=n_slots, flags=flags, **caps,
                     line_pool=dict(pool_pages=pages, page_bytes=PAGE, max_line_bytes=2 * MiB, max_pages=max_pages))


def burst(n, rng, size=200_000, kinds=("toolcall", "content", "terminal")):
    return [stream_with(long_line(kinds[i % len(kinds)], size + 1009 * i, rng), kinds[i % len(kinds)]) for i in range(n)]


def holder(rng, size, kind="toolcall"):
    """A stream with a long line, and where to cut it so that its connection holds `size // 2` bytes of that line in pages."""
    body = stream_with(long_line(kind, size, rng), kind)
    return body, len(chunk(b"Hello")) + len(chunk(b"world")) + size // 2


def feed(eng, outs, pieces, modes, conns):
    """pieces[j][b] goes to connection conns[j] in batch b; each batch is run to the end (process_all_checked), its deferred rests
    first in the next batch. Appends to outs[conns[j]]; returns the OR of the batches' overflow bits."""
    ovf = [0]

    def on_batch(res, cs):
        ovf[0] |= res.overflow
        for i, c in enumerate(cs):
            fold_segment(outs[c], res, i)
    for b in range(max(map(len, pieces))):
        items = [(c, modes[c], p[b]) for c, p in zip(conns, pieces) if b < len(p)]
        process_all_checked(eng, items, on_batch)
    return ovf[0]


# ------------------------------------------------------------------ 1: burst, trim, continue
@pytest.mark.parametrize("n_pieces", [1, 3, 17])
@pytest.mark.parametrize("mode", MODES, ids=["P", "R", "PP"])
def test_burst_trim_continue(mode, n_pieces):
    """40 streams of 200 KB lines grow the pool from 8 pages while 6 more stop inside 300 KB lines; a trim to the initial size
    keeps those pages (repacked), the held lines then complete exactly, and a second burst grows the trimmed pool again."""
    e = engine()
    try:
        rng = np.random.default_rng(n_pieces * 3 + mode)
        first, second = burst(40, rng), burst(40, rng, size=180_000)
        held = [holder(rng, 300_000 + 4099 * i) for i in range(6)]
        bodies = first + [b for b, _ in held] + second
        modes = [mode] * len(bodies)
        outs = [ConnOut() for _ in bodies]
        hold = list(range(40, 46))
        e.reset_all()
        pieces = [random_cuts(rng, b, n_pieces) for b in first] + [random_cuts(rng, b[:cut], n_pieces) for b, cut in held]
        ovf = feed(e, outs, pieces, modes, list(range(46)))
        grown = e.line_pool_capacity()[0]
        used, hw = e.pool_stats()
        assert ovf & A.OVF_POOL and grown > INITIAL and used >= 6 * 3
        e.trim()
        assert e.pool_stats() == (used, hw)
        assert e.line_pool_capacity() == (max(INITIAL, used), 1024)
        rests = [[b[cut:]] for b, cut in held] + [random_cuts(rng, b, n_pieces) for b in second]
        ovf = feed(e, outs, rests, modes, hold + list(range(46, 86)))
        check_streams(bodies, modes, outs, f"trim mode {mode} pieces {n_pieces}")
        assert not any(o.flags & (A.SEG_DEAD | A.SEG_LINE_TOO_LONG) for o in outs)
        assert ovf & A.OVF_POOL and e.line_pool_capacity()[0] > max(INITIAL, used) and e.pool_stats()[0] == 0
    finally:
        e.close()


# ------------------------------------------------------------------ 2: down to the pages held
def test_trim_down_to_the_pages_held():
    """Three connections stop inside long lines while six others complete theirs, on a pool of 2 pages that grows. A trim with
    min_pool_pages=1 leaves exactly the pages held; the first line that then needs a page grows the pool again."""
    e = engine(pages=2)
    try:
        rng = np.random.default_rng(2)
        held = [holder(rng, 300_000 + 777 * i, kind) for i, kind in enumerate(("toolcall", "content", "terminal"))]
        newcomer = stream_with(long_line("content", 200_000, rng), "content")
        done = burst(6, rng)
        bodies = [b for b, _ in held] + [newcomer] + done
        modes = [R, PP, P, R] + [MODES[i % 3] for i in range(6)]
        outs = [ConnOut() for _ in bodies]
        e.reset_all()
        feed(e, outs, [[b[:cut]] for b, cut in held] + [[b] for b in done], modes, [0, 1, 2] + list(range(4, 10)))
        used = e.pool_stats()[0]
        assert used >= 9 and e.line_pool_capacity()[0] > used
        e.trim(1)
        assert e.line_pool_capacity()[0] == used and e.pool_stats()[0] == used
        # the first line that needs a page finds none free: it defers and its collect grows the pool
        assert feed(e, outs, [[newcomer]], modes, [3]) & A.OVF_POOL
        assert e.line_pool_capacity()[0] > used
        feed(e, outs, [[b[cut:]] for b, cut in held], modes, [0, 1, 2])
        check_streams(bodies, modes, outs, "trim to held")
        assert e.pool_stats()[0] == 0
    finally:
        e.close()


# ------------------------------------------------------------------ 3: batches in flight
def run_inflight(eng, bodies, modes, depth, n_pieces, seed, between=None, abandon=None):
    """Up to depth uncollected batches of disjoint connections (connection c in group c % depth, a batch takes the ready
    connections of the next group that has any); a deferred rest goes back to the front of its queue when its batch is collected.
    between(k) runs after submit k; abandon(k) may return items for a batch submitted after submit k and released uncollected.
    The pool's generation counts every change of its capacity (growth or trim). Returns (outs, overflow bits, events):
    stale_pool counts batches that reported SSE_OVF_POOL after the pool changed since their submit (their collect must not grow
    it), trims_shrunk the trims between submit and collect that shrank it."""
    rng = np.random.default_rng(seed)
    queue = [random_cuts(rng, b, n_pieces) for b in bodies]
    outs = [ConnOut() for _ in bodies]
    busy, inflight, k, g_next, ovf = set(), [], 0, 0, []
    gen = [0, eng.line_pool_capacity()[0]]
    events = dict(stale_pool=0, trims_shrunk=0, max_in_flight=0)

    def track():
        cap = eng.line_pool_capacity()[0]
        if cap != gen[1]:
            gen[0] += 1
            gen[1] = cap
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
            inflight.append((slot, items, segs[:n].copy(), gen[0]))
            events["max_in_flight"] = max(events["max_in_flight"], len(inflight))
            busy.update(c for c, _, _ in items)
            if between is not None:
                before = gen[1]
                between(k)
                track()
                events["trims_shrunk"] += gen[1] < before
            extra = abandon(k) if abandon is not None else None
            if extra:
                s2, a2, g2 = eng.acquire()
                eng.submit(s2, *eng.fill(a2, g2, extra))
                eng.release(s2)
            k += 1
            continue
        slot, items, segs, gen_at_submit = inflight.pop(0)
        try:
            before = eng.line_pool_capacity()[0]
            res = eng.collect(slot)
            after = eng.line_pool_capacity()[0]
            check_result(eng, res, segs)
            ovf.append(res.overflow)
            if res.overflow & A.OVF_POOL and gen_at_submit != gen[0]:
                assert after == before, "a batch launched before a trim or growth grew the pool"
                events["stale_pool"] += 1
            track()
            for i, (c, m, data) in enumerate(items):
                fold_segment(outs[c], res, i)
                busy.discard(c)
                if int(res.segs[i]["flags"]) & A.SEG_DEFERRED:
                    queue[c].insert(0, data[res.consumed(i):])
        finally:
            eng.release(slot)
    return outs, ovf, events


@pytest.mark.parametrize("depth", [2, 4])
def test_trim_with_batches_in_flight(depth):
    """A trim after every second submit, while depth batches of disjoint connections are uncollected: the results collected
    after it are exact, and a batch launched before it does not grow the pool with its SSE_OVF_POOL."""
    e = engine(max_pages=2048)
    try:
        rng = np.random.default_rng(depth)
        bodies = burst(36, rng)
        modes = [MODES[i % 3] for i in range(len(bodies))]
        stats = []

        def between(k):
            if k % 2 == 1:
                used = e.pool_stats()[0]
                e.trim()
                stats.append((used, e.pool_stats()[0], e.line_pool_capacity()[0]))
        outs, ovf, ev = run_inflight(e, bodies, modes, depth, n_pieces=3, seed=depth, between=between)
        check_streams(bodies, modes, outs, f"trim in flight depth {depth}")
        assert not any(o.flags & A.SEG_DEAD for o in outs) and any(x & A.OVF_POOL for x in ovf)
        assert all(u == u2 and cap == max(INITIAL, u) for u, u2, cap in stats), stats
        assert ev["max_in_flight"] == depth and ev["trims_shrunk"] >= 1 and ev["stale_pool"] >= 1, ev
        assert e.pool_stats()[0] == 0
    finally:
        e.close()


def test_trims_between_resets_and_an_abandoned_batch():
    """sse_reset_conn and a trim after submits, and batches of other connections (long lines that take and lack pages)
    released without being collected; then sse_reset_all between two trims leaves nothing held and the initial pool."""
    e = engine(max_pages=2048)
    try:
        rng = np.random.default_rng(8)
        bodies = burst(24, rng)
        modes = [MODES[i % 3] for i in range(len(bodies))]
        junk = burst(8, rng, size=150_000)

        def between(k):
            e.reset_conn(100 + k % 8)
            if k % 2 == 0:
                e.trim()

        def abandon(k):
            return [(100 + j, P, junk[j][:180_000]) for j in range(8)] if k % 3 == 0 else None
        outs, _, ev = run_inflight(e, bodies, modes, 3, n_pieces=4, seed=8, between=between, abandon=abandon)
        check_streams(bodies, modes, outs, "trims, resets and abandoned batches")
        assert not any(o.flags & A.SEG_DEAD for o in outs) and ev["trims_shrunk"] >= 1, ev
        # junk the abandoned batches left held, then reset_all between two trims
        s, a, g = e.acquire()
        e.submit(s, *e.fill(a, g, [(100 + j, P, junk[j][:100_000]) for j in range(8)]))
        e.release(s)
        e.trim()
        assert e.pool_stats()[0] > 0
        e.reset_all()
        e.trim()
        assert e.pool_stats()[0] == 0 and e.line_pool_capacity()[0] == INITIAL
        again = burst(12, rng)
        outs = [ConnOut() for _ in again]
        feed(e, outs, [[b] for b in again], [R] * 12, list(range(12)))
        check_streams(again, [R] * 12, outs, "after reset_all and trims")
    finally:
        e.close()


# ------------------------------------------------------------------ 4: decode arenas
def test_decode_arenas_trim_at_release():
    """Saturated tool-call chains grow the tool-call and text arenas of the slot that decodes them. A trim while that slot is
    COLLECTED leaves its lent results exact; its release gives back exactly the grown bytes; a later batch grows them again."""
    e = engine(pages=32, n_slots=2, batch=4 * MiB, **TINY_DECODE)
    try:
        fresh = e.memory_held()
        rng = np.random.default_rng(4)
        bodies = folds.saturated_streams() + [stream_with(long_line("content", 100_000, rng), "content")]
        modes = [R, PP, R, PP, PP]
        for rnd in range(2):
            e.reset_all()
            outs = [ConnOut() for _ in bodies]
            for o, b in zip(outs, bodies):
                o.agent, o.tele, o.piece_ends = e.L.sse_agent_new(), e.L.sse_telemetry_new(), [len(b)]
            slot, res = process_checked(e, [(c, modes[c], bodies[c]) for c in range(len(bodies))])
            try:
                assert res.overflow & (A.OVF_TCS | A.OVF_TEXT) == A.OVF_TCS | A.OVF_TEXT, hex(res.overflow)
                assert not np.any(res.segs["flags"] & A.SEG_DEFERRED)
                grown = e.memory_held()
                assert grown[0] > fresh[0] and grown[1] > fresh[1]
                if rnd == 0:
                    e.trim()
                    assert e.memory_held() == grown        # the slot is COLLECTED: its arenas shrink at its release
                for i in range(len(bodies)):
                    fold_segment(outs[i], res, i)
                    feed_folds(e.L, outs[i], res, i, 0, False)
            finally:
                e.release(slot)
            views = check_streams(bodies, modes, outs, f"decode arenas round {rnd}")
            for i, (m, o) in enumerate(zip(modes, outs)):
                check_folds(e.L, o, m, views[i], f"decode arenas round {rnd} stream {i}")
                e.L.sse_agent_free(o.agent)
                e.L.sse_telemetry_free(o.tele)
            if rnd == 0:
                assert e.memory_held() == fresh            # exactly the grown bytes came back
        assert e.memory_held() == grown                    # round 1 grew them again and kept them (no trim)
    finally:
        e.close()


# ------------------------------------------------------------------ 5: memory accounting
def test_memory_held_returns_to_a_fresh_context():
    e = engine(**TINY_DECODE)
    try:
        fresh = e.memory_held()
        rng = np.random.default_rng(5)
        tc = b"".join(b'data: {"choices":[{"index":0,"delta":{"tool_calls":[{"index":%d,"id":"c%d","function":{"name":"f",'
                      b'"arguments":"\\u00e9\\n%d"}}]},"finish_reason":null}]}\n\n' % (k, k, k) for k in range(24))
        bodies = [tc + b for b in burst(30, rng)]
        modes = [MODES[i % 3] for i in range(len(bodies))]
        outs = [ConnOut() for _ in bodies]
        e.reset_all()
        assert feed(e, outs, [[b] for b in bodies], modes, list(range(len(bodies)))) & (A.OVF_POOL | A.OVF_TCS | A.OVF_TEXT) == \
            A.OVF_POOL | A.OVF_TCS | A.OVF_TEXT
        check_streams(bodies, modes, outs, "accounting burst")
        held = e.memory_held()
        assert held[0] > fresh[0] and held[1] > fresh[1] and e.pool_stats()[0] == 0
        e.trim(INITIAL)
        assert e.memory_held() == fresh and e.line_pool_capacity()[0] == INITIAL
    finally:
        e.close()
    e = engine()
    try:
        fresh = e.memory_held()
        rng = np.random.default_rng(6)
        bodies = burst(12, rng)
        outs = [ConnOut() for _ in bodies]
        e.reset_all()
        assert feed(e, outs, [[b] for b in bodies], [R] * 12, list(range(12))) & A.OVF_POOL
        slot, _ = process_checked(e, [])              # this collect frees the arrays the growths retired
        e.release(slot)
        pages = e.line_pool_capacity()[0]
        assert pages > INITIAL
        assert e.memory_held() == (fresh[0] + (pages - INITIAL) * (PAGE + 8), fresh[1])
    finally:
        e.close()


# ------------------------------------------------------------------ 6: the gateway
def gw_config(conns, flags=A.FLAG_DEFER, batch=1 << 20):
    cfg = A.Config()
    A.load().sse_default_config(C.byref(cfg), conns, batch)
    cfg.n_slots = 4
    cfg.flags = flags
    return cfg


@pytest.mark.parametrize("tap", [False, True], ids=["plain", "tapped"])
@pytest.mark.parametrize("devices,depth", [([0], 1), ([0], 4), ([0, 0], 1), ([0, 0], 4)])
def test_gateway_trims_between_pumps(devices, depth, tap):
    rng = np.random.default_rng(depth * 10 + len(devices) + 100)
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
        for tick in range(20000):
            for i, sid in enumerate(sids):
                if not left[i] and queue[i]:
                    left[i] = queue[i].pop(0)
                if left[i]:
                    left[i] = left[i][g.upstream_write(sid, left[i]):]
            g.pump()
            if tick % 3 == 2:
                g.trim()
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
        g.trim()
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


# ------------------------------------------------------------------ 7: refusals
def test_refusals():
    e = SseEngine(device=0, max_conns=16, bytes_per_batch=MiB, carry_slot_bytes=SLOT, line_pool=dict(pool_pages=8))
    try:
        with pytest.raises(A.SseError) as err:                # no SSE_FLAG_DEFER
            e.trim()
        assert err.value.status == A.SSE_ERR_ARG
        dev, pin = C.c_uint64(7), C.c_uint64(7)
        assert e.L.sse_memory_held(e._ctx, None, C.byref(pin)) == A.SSE_ERR_ARG
        assert e.L.sse_memory_held(e._ctx, C.byref(dev), None) == A.SSE_ERR_ARG and (dev.value, pin.value) == (7, 7)
    finally:
        e.close()
    g = Gateway(max_conns=8, bytes_per_batch=MiB)        # the worst-case config: no SSE_FLAG_DEFER
    try:
        with pytest.raises(A.SseError):
            g.trim()
    finally:
        g.close()
    e = engine(max_pages=0, conns=16, batch=4 * MiB)     # a pool without a growth limit is left as it is
    try:
        with pytest.raises(A.SseError) as err:
            e.trim(A.NONE)
        assert err.value.status == A.SSE_ERR_ARG
        rng = np.random.default_rng(7)
        body, cut = holder(rng, 300_000)
        out = [ConnOut()]
        e.reset_all()
        feed(e, out, [[body[:cut]]], [R], [0])
        mem, used = e.memory_held(), e.pool_stats()[0]
        e.trim(1)
        assert e.line_pool_capacity() == (INITIAL, 0) and e.memory_held() == mem and e.pool_stats()[0] == used
        feed(e, out, [[body[cut:]]], [R], [0])
        check_streams([body], [R], out, "untrimmed pool")
    finally:
        e.close()
