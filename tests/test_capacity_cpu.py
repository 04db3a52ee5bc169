"""CPU: sse_worst_case_config holds every extremal load of tests/capacity.py, and every load is what it claims to be.

For a grid of batch shapes, with and without a line pool, each generator's demand on each arena must fit the capacity the
worst-case config gives that arena, on both engine kinds (the two fused engines run with the tile kernel's longest carry slot).
The claims the demand model makes of the inputs (frames, records, rounds, elements per line) are checked here against the
oracle and the window restatements of tests/seams.py; what the kernels allocate for them is checked on the GPU
(test_gpu_capacity.py).

The grid compares the library's capacities with the demand model, and the model states what the current kernels allocate (for
example no tool-call element after a type error). A kernel that allocates more than the model says is therefore invisible
here: only test_gpu_capacity.py, which measures the kernels' own counts against the model, tells a kernel regression from a
model that is right. test_legacy_bounds_are_broken_by_the_loads shows that the loads would break the earlier formulas and
the earlier kernels' allocation rates, restated here."""
import functools
import json

import pytest

from inference_gateway_b200 import _abi as A
from oracle import orc
from tests import capacity as K
from tests import seams as S
from tests.capacity import TILE_SLOT, worst

GRID = [(8, 64 << 10), (8, 1 << 20), (8, 16 << 20), (64, 64 << 10), (64, 1 << 20), (256, 4 << 20), (1024, 64 << 10),
        (1024, 1 << 20), (1024, 16 << 20), (10, 1 << 20)]
POOL = dict(pool_pages=64, page_bytes=65536)


@functools.lru_cache(None)
def demands(budget: int, conns: int, line_max: int, engine: str):
    return [(g.name, g.arena, K.demand(g, engine)) for g in K.generators(budget, conns, line_max) if not (g.split_only and engine == "tile")]


@pytest.mark.parametrize("pool", [False, True], ids=["no_pool", "pool"])
@pytest.mark.parametrize("conns,batch", GRID, ids=[f"{c}x{b >> 10}KiB" for c, b in GRID])
def test_worst_case_config_holds_every_extremal_load(conns, batch, pool):
    bad = []
    for engine in ("split", "tile"):
        if engine == "tile" and pool:
            continue                                        # the tile kernel has no line pool
        cfg = worst(conns, batch, POOL if pool else None, TILE_SLOT if engine == "tile" else None)
        cap = K.bound(cfg)
        loads = demands(cfg.in_arena_bytes, conns, cfg.carry_slot_bytes, engine)
        if pool:
            loads = loads + [(g.name, g.arena, K.demand(g, engine))
                             for g in K.pooled(cfg.in_arena_bytes, conns, POOL["pool_pages"] * POOL["page_bytes"], POOL["page_bytes"])]
        for name, _, d in loads:
            for a in K.ARENAS:
                if d[a] > cap[a]:
                    bad.append(f"{engine} {name}: {a} needs {d[a]}, the config gives {cap[a]}")
    assert not bad, f"{conns} connections, {batch} bytes per batch:\n" + "\n".join(bad)


# ------------------------------------------------------------------ every generator is what it claims
SMALL = 1 << 18


def _oracle(c: K.Conn):
    whole = c.prefix + c.body
    v = orc.reframe(whole) if c.mode & A.MODE_R else orc.passthrough(whole, parse=bool(c.mode & A.MODE_PARSE))
    return v


PAGE = 65536


def _claim_loads(engine):
    """(load, longest line) of every generator at a small size; the pooled loads on the split engines only."""
    line_max = 65536 if engine == "split" else TILE_SLOT
    out = [(g, line_max) for g in K.generators(SMALL, 4, line_max)]
    if engine == "split":
        out += [(g, 1 << 20) for g in K.pooled(SMALL, 2, 8 * PAGE, PAGE)]
    return out


@pytest.mark.parametrize("engine", ["split", "tile"])
def test_generators_sit_where_they_claim(engine):
    for g, line_max in _claim_loads(engine):
        frames = recs = items = 0
        for c in g.conns:
            assert b"\n" not in c.prefix and len(c.prefix) < line_max, g.name
            v = _oracle(c)
            if c.mode & A.MODE_R:
                frames += sum(l.kind == orc.L_EMITTED for l in v.lines)
                recs += sum(l.kind in (orc.L_EMITTED, orc.L_DONE, orc.L_DONE_EXACT) for l in v.lines)
                items += sum(l.kind in (orc.L_EMITTED, orc.L_DONE) for l in v.lines)
                assert not v.terminated, g.name
            else:
                frames += len(v.lines)
                recs += sum(l.chunk is not None for l in v.lines)
                items += sum(l.chunk is not None for l in v.lines)
            assert max((len(l) + 1 for l in (c.prefix + c.body).split(b"\n")[:-1]), default=0) <= line_max, g.name
        assert (frames, recs, items) == (g.frames, g.recs, g.items), g.name
        assert g.in_bytes() <= SMALL, g.name


def test_round_counts_match_the_window_restatements():
    """split_runs_calls / tile_runs_calls count what seams.produce_windows / seams.tile_windows lay out."""
    for g, _ in _claim_loads("split") + _claim_loads("tile"):
        for c in g.conns:
            in_long = len(c.prefix) > S.BUF
            wins = S.produce_windows(c.prefix, c.body, in_long)
            want = sum(len(w.rounds()) + (w.long_end is not None) for w in wins)
            assert K.split_runs_calls(c.prefix, c.body, in_long) == want, g.name
            if len(c.prefix) <= TILE_SLOT:
                tw = S.tile_windows(c.prefix, c.body)
                assert K.tile_runs_calls(c.prefix, c.body) == sum(len(w.rounds()) for w in tw), g.name


def test_the_extremal_rates():
    """The loads sit at the rates the config's formulas are written for: a round per 64 bytes of blank lines, 128 rounds per
    8,160 bytes with the carried 17-byte tail, a tool-call element per 3 bytes of "{}," and per 2 bytes of "1,", three text
    bytes per invalid byte."""
    d = K.demand(K.generators(1 << 20, 1, 65536)[0], "split")
    assert d["runs"] == (1 << 20) // 64 - 1 and d["frames"] == 1 << 20
    g = {x.name: x for x in K.generators(1 << 20, 8, 65536)}
    part = g["runs.partial_rounds"]
    n = len(part.conns[0].body)
    assert K.demand(part, "split")["runs"] == 128 * ((n - 8192) // 8160 + 1) - 1 > n // 64 + 60
    line, k = K.tc_line("objects", 65536)
    assert len(line) <= 65536 and 3 * k > len(line) - 60 and json.loads(line[6:])["choices"][0]["delta"]["tool_calls"] == [{}] * k
    line, k = K.tc_line("numbers", 65536)
    assert 2 * k > len(line) - 60 and K.tc_alloc("numbers", k, legacy=True)["split"] == k
    for kind in ("repeat_tool_calls", "repeat_choices"):
        line, k = K.tc_line(kind, 4096)
        assert line.count(b'"tool_calls"') == k and len(line) <= 4096
    line, text, _ = K.text_line("content", 65536)
    assert text >= 3 * (len(line) - 60) and len(line) == 65536
    line, text, k = K.text_line("ids", 65536)
    assert text == 4 * k and line.count(b"\xff") == k
    # one JSON_OK chunk with a usage, whose "usage" object reopens after null once per 24 bytes
    line, k = K.usage_reset_line(TILE_SLOT)
    ck = orc.passthrough(line, parse=True).lines[0].chunk
    assert ck.json_ok and ck.usage is not None and 24 * k > len(line) - 60
    # carried: every connection decodes a whole slot beyond its share of the batch
    t = g["text.content.carried"]
    assert all(len(c.prefix) == 65535 for c in t.conns) and t.text > 4 * 8 * 65535 * 3 // 4


def test_legacy_bounds_are_broken_by_the_loads():
    """Where the earlier worst-case config and kernels broke: runs at (8, 1 MiB), one tool-call element per 2 bytes at
    (8, 64 KiB), carried payloads at (8, 64 KiB), and on the tile kernel one usage per 24 bytes of a carried line at
    (64, 64 KiB)."""
    cfg = worst(8, 1 << 20)
    flood = K.demand(K.generators(cfg.in_arena_bytes, 8, 65536)[0], "split")
    assert flood["runs"] > cfg.in_arena_bytes // 256 + 2 * 8 + 1024
    cfg = worst(8, 1 << 16)
    g = {x.name: x for x in K.generators(cfg.in_arena_bytes, 8, 65536, legacy=True)}
    assert K.demand(g["tcs.numbers"], "split")["tcs"] > cfg.in_arena_bytes // 3 + 64
    assert K.demand(g["text.content.carried"], "split")["text"] > 4 * cfg.in_arena_bytes + 65536
    assert K.demand(g["tcs.objects.carried"], "split")["tcs"] > cfg.in_arena_bytes // 3 + 64
    # the tile decoder once took a new sse_usage for every "usage" object after a null: a usage per 24 payload bytes
    cfg = worst(64, 1 << 16, slot=TILE_SLOT)
    g = {x.name: x for x in K.generators(cfg.in_arena_bytes, 64, TILE_SLOT, legacy=True)}
    assert K.demand(g["usages.reset.carried"], "tile")["usages"] > cfg.max_usages
