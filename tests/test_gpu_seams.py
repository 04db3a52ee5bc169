"""GPU: both framing engines at their seams (tests/seams.py), against the CPU oracle. The produce kernel's 8 KiB window and
carried front, its in-carry-slot long-line path, its rounds of LT_MAX lines and DONE_MAX "[DONE]" candidates, its zero-copy
decision; the tile kernel's packing, big_segment windows, rounds of LCAP lines, unquote queue of JQ_CAP jobs and template
replay limits; the line-length limit of every engine. Every input is checked to sit on its seam through the restatements,
every batch goes through orc_check_result, and every case runs in one batch and in seeded pieces."""
import numpy as np
import pytest

from inference_gateway_b200 import SseEngine, _abi as A
from inference_gateway_b200.synth import random_cuts
from oracle import orc
from tests import seams as S
from tests.util import ENGINES, check_stream, cut_bounds, digest_parity, line_limit, oracle_digests, run_pieces

pytestmark = pytest.mark.gpu

P, R, PP = A.MODE_P, A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE
MODES = (P, R, PP)
PRODUCE = ("split", "templates", "copy")
TILED = ("fused", "fused_templates")
SLOT = 32768
MAX_CONNS = 4096
BATCH_BYTES = 48 << 20


@pytest.fixture(scope="module")
def engines():
    made = {}

    def get(name):
        if name not in made:
            made[name] = SseEngine(device=0, max_conns=MAX_CONNS, bytes_per_batch=64 << 20, carry_slot_bytes=SLOT, n_slots=2,
                                   flags=ENGINES[name])
        return made[name]
    yield get
    for e in made.values():
        e.close()


def _bounds(cases) -> np.ndarray:
    """One row per case: its explicit batch boundaries, padded with empty pieces to the longest list."""
    nb = max(len(c.cuts) for c in cases) + 1
    return np.array([[0, *c.cuts] + [len(c.body)] * (nb - len(c.cuts)) for c in cases], dtype=np.int64)


def _groups(bodies):
    i = 0
    while i < len(bodies):
        j, size = i, 0
        while j < len(bodies) and j - i < MAX_CONNS and size + len(bodies[j]) < BATCH_BYTES:
            size += len(bodies[j]) + 16
            j += 1
        yield i, j
        i = j


def bulk(eng, cases, label, modes=MODES, seed=0):
    """Every case in one batch, in its explicit pieces (when it has any) and in four seeded pieces, in every mode."""
    for i, j in _groups([c.body for c in cases]):
        part = cases[i:j]
        bodies = [c.body for c in part]
        runs = [("1 batch", cut_bounds(bodies, 1, 0)), ("4 pieces", cut_bounds(bodies, 4, seed + i))]
        if any(c.cuts for c in part):
            runs.append(("explicit pieces", _bounds(part)))
        for m in modes:
            ref = oracle_digests(bodies, m)
            for name, b in runs:
                digest_parity(eng, bodies, m, b, f"{label} [{i}:{j}] mode {m} {name}", oracle=ref)


def focused(eng, cases, label, modes=MODES, seed=0, alone=False):
    """run_pieces + check_stream, field by field: one batch, the explicit pieces, three seeded pieces. alone: each case on its
    own, so that a tile holds its lines and nobody else's (the tile kernel's rounds and unquote queue are per tile)."""
    if alone:
        for k, c in enumerate(cases):
            focused(eng, [c], label, modes, seed + k)
        return
    rng = np.random.default_rng(seed)
    for m in modes:
        for split in ("one", "explicit", "seeded"):
            pieces = [[c.body] if split == "one" else c.pieces() if split == "explicit" else random_cuts(rng, c.body, 3)
                      for c in cases]
            if split == "explicit" and not any(c.cuts for c in cases):
                continue
            outs = run_pieces(eng, pieces, [m] * len(cases))
            for c, o in zip(cases, outs):
                check_stream(c.body, m, o, label=f"{label} {c.meta} mode {m} {split}")


# ------------------------------------------------------------------ produce kernel (and the same inputs on the tile kernel)
@pytest.mark.parametrize("name", PRODUCE + TILED)
def test_carried_front_and_window_end(engines, name):
    cases = S.produce_carry_cases()
    offs = set()
    for c in cases:
        Rb = c.body[len(S.FIRST):]
        w = S.produce_windows(Rb[:c.meta["t"]], Rb[c.meta["t"]:])
        assert w[0].offset(c.meta["nl"]) == c.meta["o"] and ((c.meta["nl"] in w[0].lines) == (c.meta["o"] < S.BUF))
        offs.add(c.meta["o"])
    assert offs == set(range(S.BUF - 32, S.BUF + 9)) and {c.meta["t"] for c in cases} == set(S.CARRIES)
    bulk(engines(name), cases, "window_end")


@pytest.mark.parametrize("name", PRODUCE + TILED)
def test_long_line_threshold(engines, name):
    cases = S.produce_long_cases()
    longs = [S.produce_windows(b"", c.body)[0].to_long for c in cases]
    assert 0 < sum(longs) < len(cases) and {c.meta["a"] for c in cases} == set(range(16))
    bulk(engines(name), cases, "long_threshold")


@pytest.mark.parametrize("name", PRODUCE + TILED)
def test_tokens_split_across_window_and_batch_ends(engines, name):
    cases = S.produce_split_cases()
    for c in cases:
        if c.label == "produce.split_window":
            Rb = c.body[len(S.FIRST):]
            assert S.produce_windows(Rb[:c.meta["t"]], Rb[c.meta["t"]:])[0].s1 == c.meta["at"] + c.meta["j"]
        else:
            assert c.cuts[1] == c.meta["at"] + c.meta["j"] and c.body[c.meta["at"]:c.meta["at"] + len(S.SPLIT_TOKENS[c.meta["tok"]])] == S.SPLIT_TOKENS[c.meta["tok"]]
    bulk(engines(name), cases, "split")
    focused(engines(name), [c for c in cases if c.meta["tok"] == "nlnl" and c.meta["j"] == 1][:16], "split nlnl", modes=(R,))


@pytest.mark.parametrize("name", PRODUCE + TILED)
def test_rounds_termination_and_done_candidates(engines, name):
    cases = S.produce_round_cases()
    seen = set()
    for c in cases:
        w = S.produce_windows(b"", c.body)
        assert len(w) == 1
        if c.label == "produce.rounds":
            assert len(w[0].lines) == c.meta["n_lines"]
            seen.add(c.meta["n_lines"])
        elif c.label == "produce.terminate_round":
            assert b'"stop"' in c.body[w[0].lines[c.meta["line"] - 1] + 1:w[0].lines[c.meta["line"]]]
        else:
            assert c.body[:w[0].lines[min(S.LT_MAX, len(w[0].lines)) - 1]].count(b"[DONE]") >= c.meta["k"]
    assert {S.LT_MAX - 1, S.LT_MAX, S.LT_MAX + 1, 2 * S.LT_MAX, 2 * S.LT_MAX + 1} <= seen
    focused(engines(name), cases, "rounds")


# ------------------------------------------------------------------ tile kernel (and the same inputs on the produce kernel)
def _batch_parity(eng, bt, label):
    bodies = bt.bodies
    runs = [("1 batch", cut_bounds(bodies, 1, 0)), ("3 pieces", cut_bounds(bodies, 3, len(bodies)))]
    if bt.first_cut is not None:
        runs.append(("explicit", np.array([[0, c, len(b)] for b, c in zip(bodies, bt.first_cut)], dtype=np.int64)))
    for m in MODES:
        ref = oracle_digests(bodies, m)
        for name, b in runs:
            digest_parity(eng, bodies, m, b, f"{label} {bt.meta} mode {m} {name}", oracle=ref)


@pytest.mark.parametrize("name", TILED + PRODUCE)
def test_tile_packing(engines, name):
    for bt in S.tile_pack_batches():
        n = len(bt.bodies)
        if bt.first_cut is None:
            tiles = S.plan_tiles([0] * n, [len(b) for b in bt.bodies], [1] * n)
            if bt.label == "tile.pack_count":
                assert tiles[0] == (0, min(n, S.MAX_TSEGS))
            elif bt.label == "tile.pack_sum":
                assert sum(S.r16(len(b)) for b in bt.bodies[:3]) == S.TILE + bt.meta["d"] and tiles[0][1] == (3 if bt.meta["d"] <= 0 else 2)
            elif bt.label == "tile.pack_group":
                assert (S.PLAN_GROUP in [f for f, _ in tiles]) == (n > S.PLAN_GROUP)
            elif bt.label == "tile.pack_whole":
                assert tiles[1] == (3, 1) and S.r16(len(bt.bodies[3])) == S.TILE + bt.meta["extra"]
        else:
            live = [not orc.reframe(b[:c]).terminated for b, c in zip(bt.bodies, bt.first_cut)]
            carry = [orc.passthrough(b[:c]).tail_len for b, c in zip(bt.bodies, bt.first_cut)]
            tiles = S.plan_tiles(carry, [len(b) - c for b, c in zip(bt.bodies, bt.first_cut)], live)
            assert tiles[0] == (0, S.MAX_TSEGS) and live[:S.MAX_TSEGS].count(False) == 32
        _batch_parity(engines(name), bt, bt.label)


@pytest.mark.parametrize("name", TILED + PRODUCE)
def test_big_segment_windows(engines, name):
    cases = S.big_segment_cases()
    for c in cases:
        t = c.meta.get("t", 0)
        Rb = c.body[len(S.FIRST):] if c.cuts else c.body
        w = S.tile_windows(Rb[:t], Rb[t:])
        if c.label == "tile.big_window_end":
            assert w[c.meta["win"]].s1 + c.meta["d"] == c.meta["nl"]
        elif c.label == "tile.big_no_newline":
            assert w[-1].no_newline
        else:
            assert len(w) >= 3 if c.label == "tile.big_4mib" else c.meta["at"] >= w[1].s0
    ok = [c for c in cases if c.label != "tile.big_no_newline"]
    bulk(engines(name), ok, "big_segment", seed=7)
    eng = engines(name)
    dead = [c for c in cases if c.label == "tile.big_no_newline"][0]
    a = dead.meta["line"][0]
    for m in MODES:
        outs = run_pieces(eng, [[dead.body], random_cuts(np.random.default_rng(m), dead.body, 4)], [m, m])
        for o in outs:
            assert o.flags & A.SEG_LINE_TOO_LONG and o.flags & A.SEG_DEAD
            check_stream(dead.body[:a], m, o, label=f"no newline mode {m}")


@pytest.mark.parametrize("name", TILED + PRODUCE)
def test_tile_line_rounds(engines, name):
    cases = S.tile_round_cases()
    for c in cases:
        w = S.tile_windows(b"", c.body)
        assert len(w) == 1
        if c.label == "tile.rounds":
            assert len(w[0].lines) == c.meta["n_lines"]
    assert {c.meta["n_lines"] - S.END.count(b"\n") for c in cases if c.label == "tile.rounds"} == {511, 512, 513, 1024, 1025}
    focused(engines(name), cases, "tile rounds", alone=True)
    eng = engines(name)
    firsts = set()             # lines of the first segment: the round boundary inside the second, at the boundary, inside the first
    for bt in S.tile_round_batches():
        firsts.add(bt.bodies[0].count(b"\n"))
        assert S.plan_tiles([0, 0], [len(b) for b in bt.bodies], [1, 1]) == [(0, 2)]
        for m in MODES:
            outs = run_pieces(eng, [[b] for b in bt.bodies], [m, m])
            for b, o in zip(bt.bodies, outs):
                check_stream(b, m, o, label=f"round at segment boundary {bt.meta} mode {m}")
    assert min(firsts) < S.LCAP and S.LCAP in firsts and max(firsts) > S.LCAP


@pytest.mark.parametrize("name", TILED + PRODUCE)
def test_unquote_queue(engines, name):
    cases = S.unquote_cases()
    for c in cases:
        assert len(S.tile_windows(b"", c.body)) == 1
        if c.label == "tile.unquote":
            assert c.body.count(b"\\n") == c.meta["n_jobs"]          # one string to unquote per line
    assert {c.meta["n_jobs"] for c in cases if c.label == "tile.unquote"} == {S.JQ_CAP - 1, S.JQ_CAP, S.JQ_CAP + 1, 300}
    focused(engines(name), cases, "unquote", alone=True)
    focused(engines(name), cases, "unquote, many jobs per tile")


@pytest.mark.parametrize("name", TILED + PRODUCE)
def test_template_limits(engines, name):
    cases = S.template_cases()
    learnt = lambda c: S.template_words(c.body[6:c.body.index(b"\n")])      # the shape batch 0 teaches (t_build restated)
    assert sorted(c.meta["stops"] for c in cases if "stops" in c.meta) == [S.W_STOPS - 1, S.W_STOPS, S.W_STOPS + 1]
    assert all(learnt(c) for c in cases if "stops" in c.meta)
    # t_build takes up to T_SEG_MAX structural stops and REC_MAX wildcards: one case on each side of both limits
    assert S.T_SEG_MAX == S.W_STRUCT - 1
    struct = {c.meta["struct"]: learnt(c) for c in cases if "struct" in c.meta}
    assert sorted(struct) == [S.T_SEG_MAX - 1, S.T_SEG_MAX, S.T_SEG_MAX + 1]
    assert struct[S.T_SEG_MAX][1] == S.T_SEG_MAX and struct[S.T_SEG_MAX + 1] is None
    wild = {c.meta["wild"]: learnt(c) for c in cases if "wild" in c.meta}
    assert sorted(wild) == [S.REC_MAX - 1, S.REC_MAX, S.REC_MAX + 1]
    assert wild[S.REC_MAX][2] == S.REC_MAX and wild[S.REC_MAX + 1] is None and wild[S.REC_MAX][1] <= S.T_SEG_MAX
    assert [c.meta["n_shapes"] for c in cases if "n_shapes" in c.meta][0] > S.NREC
    focused(engines(name), cases, "templates")


@pytest.mark.parametrize("name", TILED + PRODUCE)
def test_template_store_fills(name):
    """A fresh context (an empty store) and one segment larger than a tile: its windows record up to NREC templates per round,
    and the templates its shapes give (t_build restated) hold more words than the recorder may fill (TS_WORDS - 360), even at
    NREC per round. The same bytes then go through the full store again, in one batch and in pieces."""
    body = S.template_store_body()
    words = [S.template_words(S._store_line(k)[6:-1]) for k in range(S.STORE_SHAPES)]
    assert all(w is not None for w in words) and len({S._store_line(k)[6:60] for k in range(S.STORE_SHAPES)}) == S.STORE_SHAPES
    room = S.TS_WORDS - 360 - 1                      # (word 0 of the store is not a template's)
    wins = S.tile_windows(b"", body)
    assert sum(w[0] for w in words) > room
    assert len(wins) * S.NREC * min(w[0] for w in words) > room and all(len(w.lines) <= S.LCAP for w in wins)
    eng = SseEngine(device=0, max_conns=16, bytes_per_batch=4 << 20, carry_slot_bytes=SLOT, n_slots=2, flags=ENGINES[name])
    try:
        rng = np.random.default_rng(3)
        for m in MODES:
            for pieces in ([body], random_cuts(rng, body, 5)):
                outs = run_pieces(eng, [pieces, [S.FIRST + body]], [m, m])
                check_stream(body, m, outs[0], label=f"template store mode {m} {len(pieces)} pieces")
                check_stream(S.FIRST + body, m, outs[1], label=f"template store mode {m} second connection")
    finally:
        eng.close()


# ------------------------------------------------------------------ line-length limit, every engine
NEIGHBOURS = [S.chunk(b"left") * 3 + S.END, S.data_line(5000) + S.END]


@pytest.mark.parametrize("slot", [16384, 32768])
@pytest.mark.parametrize("name", list(ENGINES))
def test_line_length_limit(name, slot):
    eng = SseEngine(device=0, max_conns=64, bytes_per_batch=4 << 20, carry_slot_bytes=slot, n_slots=2, flags=ENGINES[name])
    try:
        limit = line_limit(eng)
        assert limit == slot
        cases = S.limit_cases(limit)
        assert {c.meta["n"] for c in cases} >= {limit - 1, limit, limit + 1}
        for c in cases:
            if c.label == "limit.big_tail":
                w = S.tile_windows(b"", c.body)
                assert len(w) >= 2 and w[-1].carried == c.meta["line"][0]       # the last window holds the tail back
            if c.label == "limit.big_carry":
                assert S.r16(c.cuts[0] - len(S.FIRST)) + S.r16(len(c.body) - c.cuts[0]) > S.TILE
            if c.label == "limit.big_window":
                assert c.meta["line"][0] >= S.tile_windows(b"", c.body)[1].s0
            if c.label == "limit.from_carry":
                assert c.meta["line"][0] < c.cuts[0] < c.meta["line"][1]
        rng = np.random.default_rng(slot)
        for c in cases:
            for m in MODES:
                pieces = c.pieces()
                nb = len(pieces)
                nbp = [random_cuts(rng, nb_body, nb) for nb_body in NEIGHBOURS]
                outs = run_pieces(eng, [pieces] + nbp, [m] * 3)
                o = outs[0]
                too_long = c.meta["n"] > limit
                label = f"{name} slot {slot} {c.label} {c.meta['n']} mode {m}"
                assert bool(o.flags & A.SEG_LINE_TOO_LONG) == too_long, label
                assert bool(o.flags & A.SEG_DEAD) == too_long, label
                if too_long:
                    check_stream(c.body[:c.meta["line"][0]], m, o, label=label)
                else:
                    check_stream(c.body, m, o, label=label)
                for b, ob in zip(NEIGHBOURS, outs[1:]):
                    assert not ob.flags & (A.SEG_DEAD | A.SEG_LINE_TOO_LONG)
                    check_stream(b, m, ob, label=label + " neighbour")
    finally:
        eng.close()
