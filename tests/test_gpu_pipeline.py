"""GPU: the batch pipeline with batches in flight, compared with the CPU oracle. sse_config.n_slots lets up to 8 batches be
submitted before the first is collected; they share every connection's state (carry slot, line pool, template cache), and only
the context's last-kernel event orders their kernels. These tests run that path the way callers do: several batches in
flight collected first-in-first-out or newest first, connections reset and slots released between in-flight submits,
SSE_FLAG_DEFER decode passes that run again behind later batches, steady-state ticks at full size, two contexts on one device,
and the device-resident replay path (sse_upload / sse_launch / sse_download) that bench.py times.

bench.py is imported for fill_slot, delivered, dump_outputs, N_SLOTS and N_ROT: importing it only puts the repository root on
sys.path, which tests/conftest.py has already done."""
import numpy as np
import pytest

import bench
from inference_gateway_b200 import SseEngine, _abi as A, synth
from oracle import orc
from tests.streams import PAGE, SLOT, chunk, long_line, stream_with
from tests.util import (CHECKED, ENGINES, TINY_DECODE, ConnOut, PipelinedDigests, assert_digest_parity, check_batch, check_result,
                        check_stream, check_streams, cut_bounds, digest_parity, digest_run, digest_run_pipelined, fill_pieces,
                        fold_segment, one_context_at_a_time, oracle_digests, parity_faults)

pytestmark = pytest.mark.gpu

P, R, PP = A.MODE_P, A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE
MiB = 1 << 20
GROW = A.OVF_TCS | A.OVF_USAGES | A.OVF_TEXT


@pytest.fixture(scope="module")
def contexts():
    """contexts(key, **SseEngine arguments): the context of that key; building one closes the one before, so that one large
    context lives at a time. contexts(None) closes it."""
    yield from one_context_at_a_time(lambda key, **kw: SseEngine(device=0, **kw))


@pytest.fixture(scope="module")
def populations():
    """populations(name, n): the first n bodies of BASELINE config `name` (generated once per name)."""
    made = {}

    def get(name, n=None):
        if name not in made:
            made[name] = [b for b, _, _ in synth.make_config(name, n_streams={"C2": 4096, "C3": 16384, "C4": 65536}[name])[0]]
        return made[name][:n]
    return get


@pytest.fixture(scope="module")
def c4_oracle(populations):
    """The oracle's digests of the whole C4 population in bench.py's mode (3: R + parse)."""
    return oracle_digests(populations("C4"), 3)


def max_batch_bytes(bounds) -> int:
    return int((((np.diff(bounds, axis=1) + 15) & ~15).sum(axis=0)).max())


# ------------------------------------------------------------------ pipeline depth x engine at C3 / C2 size
def _c3_engine(contexts, populations, name):
    bodies = populations("C3")
    return contexts(f"c3-{name}", max_conns=len(bodies), bytes_per_batch=sum(map(len, bodies)) // 4, n_slots=8,
                    carry_slot_bytes=16384, flags=ENGINES[name])


DEPTHS = ([("C3", 16384, R, "split", d, o) for d, o in ((4, "fifo"), (4, "lifo"), (2, "fifo"))]
          + [("C3", 4096, R, "split", 8, o) for o in ("fifo", "lifo")]
          + [("C2", 4096, PP, "split", 4, o) for o in ("fifo", "lifo")]
          + [("C3", 16384, R, e, 4, o) for e in ENGINES if e != "split" for o in ("fifo", "lifo")])


@pytest.mark.parametrize("name,n_streams,mode,engine,depth,order", [pytest.param(*c, id="-".join(map(str, c))) for c in DEPTHS])
def test_batches_in_flight_match_the_oracle(contexts, populations, name, n_streams, mode, engine, depth, order):
    """Every stream cut into 8 seeded pieces (C2: 4); depth batches in flight, collected in `order`, folded in submission order."""
    eng = _c3_engine(contexts, populations, engine)
    bodies = populations(name, n_streams)
    bounds = cut_bounds(bodies, 8 if name == "C3" else 4, seed=2000 + depth)
    assert max_batch_bytes(bounds) <= eng.cfg.in_arena_bytes
    checked = CHECKED[0]
    gd, _, _ = digest_parity(eng, bodies, mode, bounds, f"{name} x{n_streams} {engine} depth {depth} {order}", depth=depth,
                             collect_order=order)
    assert CHECKED[0] - checked == bounds.shape[1] - 1
    assert int(gd["n_recs"].sum()) > 0


def test_fold_order_is_seen_by_the_digests(contexts, populations):
    """The harness's sensitivity: folding batches 2 and 3 the other way round changes exactly the digests of the connections
    that got frames or records from both, and no other."""
    eng = _c3_engine(contexts, populations, "split")
    bodies = populations("C3", 2048)
    bounds = cut_bounds(bodies, 8, seed=77)
    seen = {}

    def on_batch(b, res, slot):
        seen[b] = (res.segs["frame_count"] + res.segs["rec_count"]) > 0
    got = digest_run_pipelined(eng, bodies, R, bounds, 4, fold_order=[0, 1, 3, 2, 4, 5, 6, 7], on_batch=on_batch)
    differ = parity_faults(got, oracle_digests(bodies, R)).get("digests", [])
    shared = seen[2] & seen[3]
    assert shared.sum() > 500
    assert np.array_equal(differ, np.nonzero(shared)[0])


# ------------------------------------------------------------------ long lines in the line pool across in-flight batches
POOL_PAGES = 512
LINE_LENGTHS = [3 * SLOT + 17, 10 * SLOT, MiB, 40 * SLOT - 5]
LINE_KINDS = ["content", "terminal", "crlf", "done"]


def _pool_engine(contexts, name):
    return contexts(f"pool-{name}", max_conns=64, bytes_per_batch=8 * MiB, carry_slot_bytes=SLOT, n_slots=4,
                    text_arena_bytes=8 * MiB, flags=ENGINES[name], line_pool=dict(pool_pages=POOL_PAGES, page_bytes=PAGE))


@pytest.mark.parametrize("engine", ["templates", "copy", "split"])
def test_long_lines_span_batches_in_flight(contexts, engine):
    """Lines of 3 to 40 carry slots (a 1 MiB tool call among them) cut into five pieces, in batches 0-4 of six, with four in
    flight: the line pool holds every line while the batches that wrote it are all uncollected. Every connection is compared
    field by field; sse_line_pool_stats, called between submits, already counts the pages of the batches in flight."""
    eng = _pool_engine(contexts, engine)
    rng = np.random.default_rng(31)
    bodies, modes, starts, lens = [], [], [], []
    for j, n in enumerate(LINE_LENGTHS):
        for kind in ("toolcall", LINE_KINDS[j]):
            line = long_line(kind, n, rng)
            for m in (P, R, PP):
                bodies.append(stream_with(line, kind))
                modes.append(m)
                starts.append(len(chunk(b"Hello") + chunk(b"world")))
                lens.append(n)
    bounds = np.zeros((len(bodies), 7), dtype=np.int64)
    for i, (b, s, n) in enumerate(zip(bodies, starts, lens)):
        cuts = [s + (n * q) // 5 + int(rng.integers(0, 64)) for q in range(1, 5)]
        bounds[i] = [0] + cuts + [s + n + int(rng.integers(0, 40)), len(b)]
    assert max_batch_bytes(bounds) <= eng.cfg.in_arena_bytes
    outs = [ConnOut() for _ in bodies]
    held = {}

    def between(b):
        if b == 3:          # batches 0-3 in flight, nothing collected: every line is held, most of them in pages
            held["stats"] = eng.pool_stats()

    def on_batch(b, res, slot):
        for i, o in enumerate(outs):
            fold_segment(o, res, i)
    digest_parity(eng, bodies, modes, bounds, f"pool {engine}", depth=4, between=between, on_batch=on_batch)
    check_streams(bodies, modes, outs, f"pool {engine}")
    # a line that left its carry slot is held whole in pages (tests/test_gpu_long_lines.py)
    want = sum(-(-int(bounds[i, 4] - s) // PAGE) for i, s in enumerate(starts) if bounds[i, 4] - s > SLOT)
    used, hw = held["stats"]
    assert used == want and hw >= used, (held["stats"], want)
    assert eng.pool_stats()[0] == 0
    eng.reset_all()
    used, hw = eng.pool_stats()
    assert used == 0 and want <= hw <= POOL_PAGES


# ------------------------------------------------------------------ sse_reset_conn between in-flight submits
def _reset_run(eng, others, xs, ys, boundaries, reset_every, modes, seed, pool_check=None):
    """Connections c % reset_every == 0 get the pieces of xs[c][:boundary] in batches 0-2, are reset after submit 2 with
    nothing collected, and get ys[c] in batches 3-5; the others carry on. Returns the reset connections' outputs."""
    rng = np.random.default_rng(seed)
    n = len(others)
    reset = [c for c in range(n) if c % reset_every == 0]
    bodies = list(others)
    bounds = cut_bounds(others, 6, seed=seed)
    for c in reset:
        x, y, cut = xs[c], ys[c], boundaries[c]
        bodies[c] = x[:cut] + y
        u = np.sort(rng.integers(0, cut + 1, size=2))
        v = np.sort(rng.integers(0, len(y) + 1, size=2))
        bounds[c] = [0, u[0], u[1], cut, cut + v[0], cut + v[1], cut + len(y)]
    outs_x = {c: ConnOut() for c in reset}
    outs_y = {c: ConnOut() for c in reset}

    def between(b):
        if b == 2:
            if pool_check is not None:
                pool_check("before")
            for c in reset:
                eng.reset_conn(c)
            if pool_check is not None:
                pool_check("after")

    def on_batch(b, res, slot):
        for c in reset:
            fold_segment((outs_x if b < 3 else outs_y)[c], res, c)
    digest_parity(eng, bodies, modes, bounds, "connections not reset", skip=reset, depth=4, between=between, on_batch=on_batch)
    mode_of = np.broadcast_to(np.asarray(modes, dtype=np.uint8), (n,))
    for c in reset:
        # the reset drops X's unterminated tail: X's frames and records up to the piece boundary, then Y from its start
        check_stream(xs[c][:boundaries[c]], int(mode_of[c]), outs_x[c], label=f"conn {c} before the reset")
        check_stream(ys[c], int(mode_of[c]), outs_y[c], label=f"conn {c} after the reset")
        # an expectation without the reset (X's tail continued by Y) is not what came out
        joined = xs[c][:boundaries[c]] + ys[c]
        v = orc.reframe(joined) if mode_of[c] & A.MODE_R else orc.passthrough(joined, parse=True)
        no_reset = [l.out for l in v.lines if l.kind == orc.L_EMITTED] if mode_of[c] & A.MODE_R else [l.out for l in v.lines]
        assert outs_x[c].frames + outs_y[c].frames != no_reset, c
    return reset


def test_reset_between_in_flight_submits(contexts, populations):
    bodies = populations("C4", 512)
    eng = contexts("reset", max_conns=512, bytes_per_batch=sum(map(len, bodies)), n_slots=4)
    ys = [b for b, _, _ in synth.make_config("C4", n_streams=512, shard=1)[0]]
    # the boundary falls inside an event's payload, a third of the way in: X still has a held-back tail at the reset
    cuts = [b.find(b"\n\n", len(b) // 3) - 5 for b in bodies]
    modes = np.array([(R, PP)[c % 2] for c in range(len(bodies))], dtype=np.uint8)
    _reset_run(eng, bodies, bodies, ys, cuts, 8, modes, seed=5)


def test_reset_between_in_flight_submits_returns_pooled_pages(contexts, populations):
    """As above, with the reset connections in the middle of a 300 KB line held in the line pool: sse_line_pool_stats, called
    between the submits, counts their pages before the reset and none after it."""
    eng = _pool_engine(contexts, "split")
    others = populations("C4", 48)
    rng = np.random.default_rng(8)
    head = chunk(b"a")
    xs = [head + long_line("toolcall", 300_000 + 1000 * c, rng) + b"\n" + chunk(b"b", '"stop"') for c in range(48)]
    cuts = [len(head) + 200_000 + 7 * c for c in range(48)]
    ys = [b for b, _, _ in synth.make_config("C4", n_streams=48, shard=2)[0]]
    reset_every = 4
    want = sum(-(-(cuts[c] - len(head)) // PAGE) for c in range(0, 48, reset_every))
    seen = {}

    def pool_check(when):
        seen[when] = eng.pool_stats()
    modes = np.array([(R, PP)[(c // reset_every) % 2] for c in range(48)], dtype=np.uint8)
    _reset_run(eng, others, xs, ys, cuts, reset_every, modes, seed=6, pool_check=pool_check)
    assert seen["before"][0] == want, (seen, want)
    assert seen["after"][0] == 0, seen
    assert eng.pool_stats()[0] == 0


# ------------------------------------------------------------------ a batch released without being collected
def _seg_outs(res, n):
    out = []
    for i in range(n):
        o = ConnOut()
        fold_segment(o, res, i)
        out.append((o.frames, o.recs, o.carry_len, o.flags))
    return out


def test_abandoned_batch(contexts, populations):
    """b0, b1, b2 submitted; b1 released without being collected. Its kernels still ran, so b0, b2 and b3 (in b1's slot,
    acquired again at once) equal a fully collected run batch for batch, field by field."""
    bodies = populations("C4", 384)
    n = len(bodies)
    eng = contexts("abandon", max_conns=n, bytes_per_batch=sum(map(len, bodies)), n_slots=3)
    bounds = cut_bounds(bodies, 5, seed=12)
    ref = []
    digest_run(eng, bodies, R, bounds, on_batch=lambda b, res: ref.append(_seg_outs(res, n)))

    eng.reset_all()
    held = []

    def submit(b):
        slot, arena, segs = eng.acquire()
        eng.submit(slot, n, fill_pieces(arena, segs, bodies, R, bounds, b))
        held.append(slot)
        return slot, segs[:n].copy()

    def collect(b, slot, segs):
        res = eng.collect(slot)
        try:
            check_result(eng, res, segs)
            got = _seg_outs(res, n)
            for i in range(n):
                assert got[i] == ref[b][i], f"batch {b} connection {i} differs from the fully collected run"
        finally:
            eng.release(slot)
            held.remove(slot)
    try:
        s0, g0 = submit(0)
        s1, _ = submit(1)
        s2, g2 = submit(2)
        eng.release(s1)
        held.remove(s1)
        s3, g3 = submit(3)
        assert s3 == s1
        collect(0, s0, g0)
        collect(2, s2, g2)
        collect(3, s3, g3)
        s4, g4 = submit(4)
        collect(4, s4, g4)
    finally:
        for s in held:
            eng.release(s)


# ------------------------------------------------------------------ SSE_FLAG_DEFER: decode arenas grow behind later batches
EVENTS_PER_BATCH = [1, 2, 2, 3, 5, 8, 11, 17, 26]     # x2.5 or more every three batches: a slot's next batch outgrows it again


def _defer_piece(c, b):
    """Events with tool calls, a usage and invalid UTF-8 (three text bytes per byte): tool calls, usages and text all grow
    with the event count."""
    out = []
    for e in range(EVENTS_PER_BATCH[b]):
        tcs = ",".join('{"index":%d,"id":"call_%d_%d","type":"function","function":{"name":"f\\u00e9%d","arguments":"{\\"a\\":%d}"}}'
                       % (t, b, e, t, t) for t in range(1 + (c + e) % 5))
        junk = bytes(0x80 + (c * 7 + e * 13 + k) % 0x80 for k in range(24))
        out.append(b'data: {"choices":[{"index":0,"delta":{"content":"' + junk + b'","tool_calls":[' + tcs.encode()
                   + b']},"finish_reason":null}],"usage":{"prompt_tokens":%d,"completion_tokens":2,"total_tokens":3}}\n\n' % e)
    return b"".join(out)


@pytest.mark.parametrize("flags", [A.FLAG_DEFER, A.FLAG_DEFER | A.FLAG_TEMPLATES, A.FLAG_DEFER | A.FLAG_COUNTERS],
                         ids=["defer", "defer_templates", "defer_counters"])
def test_deferred_regrowth_behind_later_batches(contexts, flags):
    n = 48
    pieces = [[_defer_piece(c, b) for b in range(len(EVENTS_PER_BATCH))] for c in range(n)]
    bodies = [b"".join(p) for p in pieces]
    bounds = np.zeros((n, len(EVENTS_PER_BATCH) + 1), dtype=np.int64)
    bounds[:, 1:] = np.cumsum([[len(x) for x in p] for p in pieces], axis=1)
    modes = np.array([(R, PP)[c % 2] for c in range(n)], dtype=np.uint8)
    eng = contexts(f"defer-{flags}", max_conns=64, bytes_per_batch=MiB, n_slots=3, flags=flags, **TINY_DECODE)
    counting = bool(flags & A.FLAG_COUNTERS)
    grew, passes, p_lines = {}, {}, []

    def on_batch(b, res, slot):
        assert not np.any(res.segs["flags"] & A.SEG_DEFERRED) and not res.overflow & (A.OVF_OUT | A.OVF_RUNS), b
        grew[b] = res.overflow & GROW
        if counting:
            # batch b is collected while b + 1 and b + 2 are still in flight (FIFO at depth 3)
            k = eng.counters(slot)
            check_batch(k, res, b"".join(p[b] for p in pieces))
            passes[b] = k["decode_passes"]
            p_lines.append(k["p_lines"])
    got = digest_parity(eng, bodies, modes, bounds, f"defer flags {flags}", depth=3, on_batch=on_batch)
    # every batch outgrew its slot, the first use of a slot and every later one (that slot had already grown)
    assert all(grew[b] for b in range(len(EVENTS_PER_BATCH))), grew
    assert all(grew[b] & A.OVF_USAGES for b in range(3, len(EVENTS_PER_BATCH))), grew
    if counting:
        assert all(passes[b] >= 2 for b in grew if grew[b]), passes
        serial = []
        gs = digest_run(eng, bodies, modes, bounds, on_batch=lambda b, res: serial.append(eng.counters(0)["p_lines"]))
        assert sum(p_lines) == sum(serial) == sum(x.count(b"\n") for x in bodies)
        assert all(np.array_equal(x, y) for x, y in zip(gs, got))


# ------------------------------------------------------------------ steady-state ticks at full C4 size
@pytest.mark.parametrize("engine", ["split", "fused", "templates"])
def test_steady_state_ticks_in_flight(contexts, populations, engine):
    """The production batcher's shape: tick t carries event t of every stream (tools/tick_bench.py); every third tick ends
    inside the next event at a seeded offset, so the tail crosses into a batch that is already in flight. Provider hints
    cycle 0-3. Depth 3."""
    evs = [[e + b"\n\n" for e in b.split(b"\n\n") if e] for b in populations("C4")]
    bodies = [b"".join(e) for e in evs]
    n_ticks = max(map(len, evs))
    rng = np.random.default_rng(44)
    bounds = np.zeros((len(bodies), n_ticks + 1), dtype=np.int64)
    for i, ev in enumerate(evs):
        ends = np.cumsum([len(e) for e in ev])
        bounds[i, 1:len(ev) + 1] = ends
        bounds[i, len(ev) + 1:] = ends[-1]
        for t in range(2, len(ev) - 1, 3):
            bounds[i, t + 1] += int(rng.integers(1, len(ev[t + 1])))
    eng = contexts(f"ticks-{engine}", max_conns=len(bodies), bytes_per_batch=max_batch_bytes(bounds), n_slots=3,
                   carry_slot_bytes=16384, flags=ENGINES[engine])
    providers = (np.arange(len(bodies)) % 4).astype(np.uint8)
    digest_parity(eng, bodies, R, bounds, f"ticks {engine}", providers=providers, depth=3)


# ------------------------------------------------------------------ two contexts on one device
def test_two_contexts_interleaved(contexts, populations):
    """A split and a fused context alive together (the decode and tile tables are per device, shared by both), their
    batches interleaved, two in flight in each."""
    contexts(None)
    bodies = populations("C3", 2048)
    engs = [SseEngine(device=0, max_conns=len(bodies), bytes_per_batch=sum(map(len, bodies)) // 2, n_slots=2,
                      flags=f) for f in (0, A.FLAG_KERNEL_FUSED)]
    runs = []
    try:
        runs = [PipelinedDigests(e, bodies, R, cut_bounds(bodies, 6, seed=90 + k), 2) for k, e in enumerate(engs)]
        while any([r.step() for r in runs]):
            pass
        for k, r in enumerate(runs):
            assert_digest_parity(r.finish(), bodies, R, f"context {k}")
    finally:
        for r in runs:
            r.abort()
        for e in engs:
            e.close()


# ------------------------------------------------------------------ the slot state machine
def _busy(fn):
    with pytest.raises(A.SseError) as e:
        fn()
    assert e.value.status == A.SSE_ERR_BUSY


def test_slot_state_machine():
    eng = SseEngine(device=0, max_conns=8, bytes_per_batch=MiB, n_slots=2, flags=A.FLAG_COUNTERS)
    try:
        x = synth.make_config("C4", n_streams=1)[0][0][0]
        cut = x.find(b"\n", len(x) // 2) + 7
        s0, a0, g0 = eng.acquire()
        s1, a1, g1 = eng.acquire()
        _busy(eng.acquire)                                   # past n_slots
        _busy(lambda: eng.collect(s0))                       # acquired, not submitted
        n, nb = eng.fill(a0, g0, [(0, P, x)])
        eng.submit(s0, n, nb)
        _busy(lambda: eng.submit(s0, n, nb))                 # submitted twice
        _busy(lambda: eng.launch(s0, n))
        _busy(lambda: eng.download(s0))
        _busy(lambda: eng.counters(s0))
        res = eng.collect(s0)
        check_result(eng, res, g0[:n].copy())
        _busy(lambda: eng.collect(s0))                       # collected twice
        eng.counters(s0)
        eng.release(s0)
        # release of a submitted slot waits for its kernels and frees the slot: the connection has advanced past x[:cut]
        n, nb = eng.fill(a1, g1, [(1, P, x[:cut])])
        eng.submit(s1, n, nb)
        eng.release(s1)
        slots = [eng.acquire(), eng.acquire()]
        assert sorted(s for s, _, _ in slots) == [0, 1]
        eng.release(slots[1][0])
        s, a, g = slots[0]
        n, nb = eng.fill(a, g, [(1, P, x[cut:])])
        eng.submit(s, n, nb)
        res = eng.collect(s)
        check_result(eng, res, g[:n].copy())
        k = x[:cut].rfind(b"\n") + 1
        assert b"".join(res.seg_frames(0)) == x[k:x.rfind(b"\n") + 1]
        assert int(res.segs[0]["carry_len"]) == len(x) - x.rfind(b"\n") - 1
        eng.release(s)
    finally:
        eng.close()


# ------------------------------------------------------------------ bench.py's e2e loop and its device-resident replay path
def _c4_engine(contexts, bodies, name):
    return contexts(f"c4-{name}", max_conns=len(bodies), bytes_per_batch=sum(map(len, bodies)), n_slots=bench.N_SLOTS,
                    carry_slot_bytes=16384, flags=ENGINES[name])


def _fresh_parity(eng, res, segs, bodies, mode, oracle, label):
    """One batch that holds every stream whole after a reset: checked, folded alone, equal to the oracle."""
    check_result(eng, res, segs)
    n = len(bodies)
    d, carry, flags = orc.new_digests(n), np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint32)
    assert orc.digest_result(res.raw, np.arange(n, dtype=np.uint32), d, carry, flags) == n
    assert_digest_parity((d, carry, flags), bodies, mode, label, oracle=oracle)
    return d, carry, flags


def test_bench_e2e_loop(contexts, populations, c4_oracle):
    """bench.py's e2e measurement call for call: the same pinned input in every slot, depth 3, sse_reset_all(NULL) before each
    submit. Every batch collected is a fresh population's result, and delivers what the one-shot batch delivers."""
    bodies = populations("C4")
    mode, oracle = 3, c4_oracle
    eng = _c4_engine(contexts, bodies, "split")
    slots = [eng.acquire() for _ in range(bench.N_SLOTS)]
    for sl, arena, segs in slots:
        n_segs, in_bytes, _ = bench.fill_slot(eng, arena, segs, bodies, mode)
    segs0 = slots[0][2][:n_segs].copy()
    for sl, _, _ in slots:
        eng.release(sl)
    s, _, _ = eng.acquire()
    eng.reset_all(0)
    eng.submit(s, n_segs, in_bytes)
    try:
        res = eng.collect(s)
        _fresh_parity(eng, res, segs0, bodies, mode, oracle, "one-shot")
        one = bench.delivered(res)
    finally:
        eng.release(s)
    depth, raw = 3, []

    def collect(sl):
        try:
            r = eng.collect(sl)
            _fresh_parity(eng, r, segs0, bodies, mode, oracle, f"e2e batch {len(raw)}")
            assert bench.delivered(r) == one
            raw.append(int(r.raw.n_frames))
        finally:
            eng.release(sl)
    inflight = []
    try:
        for _ in range(7):
            s2, _, _ = eng.acquire()
            eng.reset_all(0)
            eng.submit(s2, n_segs, in_bytes)
            inflight.append(s2)
            if len(inflight) == depth:
                collect(inflight.pop(0))
        while inflight:
            collect(inflight.pop(0))
    finally:
        for sl in inflight:
            eng.release(sl)
    assert len(raw) == 7
    # n_frames counts frames allocated after a terminating chunk and then cut; bench.py's e2e figure sums it
    print(f"\n[e2e] frames per batch: allocated (n_frames) {raw[0]}, delivered {one[0]}, ratio {raw[0] / one[0]:.4f}")


@pytest.mark.parametrize("engine", ["split", "templates", "fused"])
def test_bench_replay_path(contexts, populations, c4_oracle, engine, tmp_path):
    """bench.py's timed steps on a non-default torch stream: N_ROT resident inputs, each step sse_reset_all(stream) and one
    sse_launch, the slots downloaded at the end, launched again many times and downloaded again. Then the segmented
    measurement: one reset, k launches of the pieces on one stream, folded in order."""
    import torch
    bodies = populations("C4")
    mode, oracle = 3, c4_oracle
    eng = _c4_engine(contexts, bodies, engine)
    ts = torch.cuda.Stream()
    stream = ts.cuda_stream
    assert stream != 0
    slots = [eng.acquire() for _ in range(bench.N_SLOTS)]
    try:
        for sl, arena, segs in slots[:bench.N_ROT]:
            n_segs, in_bytes, _ = bench.fill_slot(eng, arena, segs, bodies, mode)
            eng.upload(sl, n_segs, in_bytes, stream)
        segs0 = slots[0][2][:n_segs].copy()
        torch.cuda.synchronize()

        def step(i):
            eng.reset_all(stream)
            eng.launch(slots[i % bench.N_ROT][0], n_segs, stream)
        for i in range(bench.N_ROT):
            step(i)
        first = {}
        for sl, _, _ in slots[:bench.N_ROT]:
            first[sl] = _fresh_parity(eng, eng.download(sl, stream), segs0, bodies, mode, oracle, f"slot {sl} first launch")
        for i in range(bench.N_ROT, 5 * bench.N_ROT + 1):
            step(i)
        for sl, _, _ in slots[:bench.N_ROT]:
            res = eng.download(sl, stream)
            again = _fresh_parity(eng, res, segs0, bodies, mode, oracle, f"slot {sl} relaunched")
            assert all(np.array_equal(x, y) for x, y in zip(again, first[sl])), sl
        # what --dump-outputs writes for a relaunched slot equals what sse_submit / sse_collect of the same input gives
        sl0 = slots[0][0]
        bench.dump_outputs(eng.download(sl0, stream), str(tmp_path / "replay"))
        torch.cuda.synchronize()            # the replay path and sse_submit are ordered only by synchronising in between
        eng.reset_all(0)
        eng.submit(sl0, n_segs, in_bytes)
        res = eng.collect(sl0)
        check_result(eng, res, segs0)
        bench.dump_outputs(res, str(tmp_path / "submit"))
        names = sorted(p.name for p in (tmp_path / "replay").iterdir())
        assert names == sorted(p.name for p in (tmp_path / "submit").iterdir()) and len(names) == 12
        for name in names:
            a, b = np.load(tmp_path / "replay" / name), np.load(tmp_path / "submit" / name)
            assert a.dtype == b.dtype and np.array_equal(a, b), name
        eng.release(sl0)
        slots[0] = eng.acquire()
        assert slots[0][0] == sl0

        # segmented: bench.py's seeded cuts, one piece per slot, launched in order after one reset
        k = bench.N_SLOTS
        rng = np.random.default_rng(0xB200)
        pieces = [synth.random_cuts(rng, b, k) for b in bodies]
        meta = []
        for b_i, (sl, arena, segs) in enumerate(slots[:k]):
            ns, nb, _ = bench.fill_slot(eng, arena, segs, [p[b_i] if b_i < len(p) else b"" for p in pieces], mode)
            eng.upload(sl, ns, nb, stream)
            meta.append((sl, ns, segs[:ns].copy()))
        torch.cuda.synchronize()
        for _ in range(2):
            eng.reset_all(stream)
            for sl, ns, _ in meta:
                eng.launch(sl, ns, stream)
        n = len(bodies)
        d, carry, flags = orc.new_digests(n), np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint32)
        frames = 0
        for sl, ns, g in meta:
            res = eng.download(sl, stream)
            check_result(eng, res, g)
            assert orc.digest_result(res.raw, np.arange(n, dtype=np.uint32), d, carry, flags) == n
            frames += bench.delivered(res)[0]
        assert_digest_parity((d, carry, flags), bodies, mode, f"segmented {engine}", oracle=oracle)
        assert frames == int(oracle[0]["n_frames"].sum())
    finally:
        torch.cuda.synchronize()
        for sl, _, _ in slots:
            eng.release(sl)
