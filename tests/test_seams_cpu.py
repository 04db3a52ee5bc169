"""CPU: the framing seams of tests/seams.py -- the constants they were designed for, the tile plan restated on hand-worked
examples, deterministic generators that land on their seams, and the oracle against the independent stream model on every seam
stream."""
import collections

import pytest

from oracle import orc
from tests import go_stream_model as sm
from tests import seams as S


def test_constants_are_the_designed_ones():
    assert (S.BUF, S.LT_MAX, S.DONE_MAX) == (8192, 64, 16)
    assert (S.TILE, S.MAX_TSEGS, S.LCAP, S.PLAN_GROUP, S.JQ_CAP) == (49152, 96, 512, 1024, 64)
    assert (S.W_STOPS, S.W_STRUCT, S.REC_MAX, S.NREC, S.TS_WORDS) == (96, 64, 40, 6, 3328)


def test_plan_tiles_hand_worked():
    T = S.TILE
    live = [1] * 200
    assert S.plan_tiles([0] * 96, [16] * 96, live) == [(0, 96)]
    assert S.plan_tiles([0] * 97, [16] * 97, live) == [(0, 96), (96, 1)]
    # TILE - 16, TILE and TILE + 16 over three regions, then a 32-byte one
    assert S.plan_tiles([0] * 4, [16384, 16384, 16368, 32], live) == [(0, 3), (3, 1)]
    assert S.plan_tiles([0] * 4, [16384, 16384, 16384, 32], live) == [(0, 3), (3, 1)]
    assert S.plan_tiles([0] * 4, [16384, 16384, 16400, 32], live) == [(0, 2), (2, 2)]
    # the carry and the bytes are padded to 16 each: 8 + 16376 takes 16 + 16384
    assert S.plan_tiles([8, 0, 0], [16376, 16384, 16368], live) == [(0, 3)]
    assert S.plan_tiles([8, 0, 0], [16376, 16384, 16384], live) == [(0, 2), (2, 1)]
    # a finished connection has no region but takes one of the 96 places
    assert S.plan_tiles([0] * 97, [1000] + [16] * 96, [0] + [1] * 96) == [(0, 96), (96, 1)]
    # a region of exactly TILE is an ordinary tile; 16 bytes more goes alone to big_segment
    assert S.plan_tiles([0] * 3, [32, T, 32], live) == [(0, 1), (1, 1), (2, 1)]
    assert S.plan_tiles([0] * 3, [32, T + 1, 32], live) == [(0, 1), (1, 1), (2, 1)]
    assert S.plan_tiles([0] * 2, [T - 32, 32], live) == [(0, 2)]
    assert S.plan_tiles([0, 16], [T - 32, 16], live) == [(0, 2)]
    assert S.plan_tiles([0, 17], [T - 32, 1], live) == [(0, 1), (1, 1)]
    # groups of PLAN_GROUP segments are planned apart: 48 regions of 1,008 bytes fill a tile, 1,024 = 21 * 48 + 16
    tiles = S.plan_tiles([0] * 1100, [1008] * 1100, [1] * 1100)
    assert (1008, 16) in tiles and (1024, 48) in tiles and sum(n for _, n in tiles) == 1100
    assert all(f // 1024 == (f + n - 1) // 1024 for f, n in tiles)


def test_produce_windows_hand_worked():
    w = S.produce_windows(b"", b"a" * 100 + b"\n" + b"b" * 9000)
    assert (w[0].s0, w[0].s1, w[0].lines) == (0, 8192, [100]) and w[0].to_long is False
    assert w[1].s0 == 101 and w[1].base == r16m(8192 - 101) and w[1].to_long and w[-1].carried is None
    w = S.produce_windows(b"", b"a" * 100 + b"\n" + b"b" * 8000 + b"\n" + b"c" * 500)
    assert w[0].lines == [100, 8101] and (w[1].s0, w[1].base, w[1].carried) == (8102, 6, 8102) and not w[0].to_long
    w = S.produce_windows(b"c" * 5, b"d" * 10000 + b"\n")
    assert w[0].base == 11 and w[0].s1 == 5 + 8192 - 16 and w[0].to_long and w[1].long_end == 10005
    w = S.produce_windows(b"", b"x\n" * 129)
    assert w[0].rounds() == [64, 64, 1]


def r16m(n):
    return S.r16(n) - n


def test_tile_windows_hand_worked():
    w = S.tile_windows(b"", b"y" * 100 + b"\n")
    assert len(w) == 1 and w[0].lines == [100]
    body = S.filler(S.TILE + 5000)
    w = S.tile_windows(b"z" * 20, body)
    assert w[0].s0 == 0 and w[0].base == 12 and w[0].s1 == 20 + S.TILE - 32
    assert w[1].s0 == w[0].restart and w[1].base == (w[0].restart - 20) & 15
    assert w[1].s1 == 20 + ((w[0].restart - 20) & ~15) + S.TILE or w[1].carried is not None
    w = S.tile_windows(b"", b"q" * 10 + b"\n" + b"r" * (2 * S.TILE))
    assert w[1].no_newline


GENERATORS = {
    "produce.window_end": (S.produce_carry_cases, 3000),
    "produce.long_threshold": (S.produce_long_cases, 16 * 49),
    "produce.split_window": (S.produce_split_cases, 16 * 20),
    "produce.split_batch": (S.produce_split_cases, 16 * 20),
    "produce.rounds": (S.produce_round_cases, 10),
    "produce.terminate_round": (S.produce_round_cases, 2),
    "produce.done_candidates": (S.produce_round_cases, 12),
    "tile.big_window_end": (S.big_segment_cases, 2 * 7 * len(S.BIG_CARRIES)),
    "tile.big_4mib": (S.big_segment_cases, 3),
    "tile.rounds": (S.tile_round_cases, 5),
    "tile.terminate_round": (S.tile_round_cases, 2),
    "tile.unquote": (S.unquote_cases, 8),
    "tile.unquote_dup": (S.unquote_cases, 16),
    "tpl.stops": (S.template_cases, 3),
    "tpl.struct": (S.template_cases, 3),
    "tpl.wild": (S.template_cases, 3),
}


@pytest.mark.parametrize("gen", sorted({g.__name__ for g, _ in GENERATORS.values()}))
def test_generators_are_deterministic_and_full(gen):
    fn = getattr(S, gen)
    a, b = fn(), fn()
    assert [(c.label, c.body, c.cuts, c.meta) for c in a] == [(c.label, c.body, c.cuts, c.meta) for c in b]
    got = collections.Counter(c.label for c in a)
    for label, (g, n) in GENERATORS.items():
        if g is fn:
            assert got[label] >= n, (label, got[label])


def test_produce_cases_land_on_their_seams():
    for c in S.produce_carry_cases():
        R = c.body[len(S.FIRST):]
        w = S.produce_windows(R[:c.meta["t"]], R[c.meta["t"]:])
        p = c.meta["nl"]
        if c.meta["o"] < S.BUF:
            assert w[0].s0 <= p < w[0].s1 and p in w[0].lines and w[0].offset(p) == c.meta["o"], c.meta
        else:
            assert p >= w[0].s1 and w[0].offset(p) == c.meta["o"], c.meta
    sides = collections.Counter()
    for c in S.produce_long_cases():
        a, e = c.meta["line"]
        w = S.produce_windows(b"", c.body)
        sides[w[0].to_long] += 1
        assert w[0].to_long == (e > S.BUF and S.BUF - a >= S.BUF - 32)
        assert w[0].offset(a) == c.meta["a"]
    assert sides[True] > 100 and sides[False] > 100
    for c in S.produce_split_cases():
        if c.label == "produce.split_window":
            R = c.body[len(S.FIRST):]
            t = c.meta["t"]
            w = S.produce_windows(R[:t], R[t:])
            assert w[0].s1 == c.meta["at"] + c.meta["j"], c.meta       # the first c.meta["j"] token bytes end the window
        else:
            assert c.cuts[1] == c.meta["at"] + c.meta["j"]
    rounds_seen = set()
    for c in S.produce_round_cases():
        w = S.produce_windows(b"", c.body)
        if c.label == "produce.rounds":
            n = c.meta["n_lines"]
            assert len(w) == 1 and len(w[0].lines) == n and w[0].rounds() == [S.LT_MAX] * (n // S.LT_MAX) + [n % S.LT_MAX] * (n % S.LT_MAX > 0)
            rounds_seen.add(n)
        elif c.label == "produce.terminate_round":
            assert w[0].lines[c.meta["line"]] == len(S.SHORT) * c.meta["line"] + len(S.STOP_LINE) - 1
        else:
            first = c.body[:w[0].lines[S.LT_MAX - 1] + 1] if len(w[0].lines) >= S.LT_MAX else c.body
            assert first.count(b"[DONE]") >= c.meta["k"]
    assert {63, 64, 65, 128, 129} <= rounds_seen


def test_tile_cases_land_on_their_seams():
    for c in S.big_segment_cases():
        t = c.meta.get("t", 0)
        R = c.body[len(S.FIRST):] if c.cuts else c.body
        w = S.tile_windows(R[:t], R[t:])
        assert len(w) >= 2 or c.label == "tile.big_no_newline"
        if c.label == "tile.big_window_end":
            win = w[c.meta["win"]]
            assert win.s1 + c.meta["d"] == c.meta["nl"]
            assert (c.meta["nl"] in win.lines) == (c.meta["d"] < 0)
            if c.meta["d"] <= -2:
                assert win.restart == c.meta["nl"] + 1 and win.s1 - win.restart <= 16
        elif c.label == "tile.big_no_newline":
            assert w[-1].no_newline
        elif c.label in ("tile.big_terminate", "tile.big_done_exact"):
            assert c.meta["at"] >= w[1].s0
    for c in S.tile_round_cases():
        w = S.tile_windows(b"", c.body)
        assert len(w) == 1
        if c.label == "tile.rounds":
            assert len(w[0].lines) == c.meta["n_lines"]
        else:
            assert w[0].lines[c.meta["line"]] == len(S.SHORT) * c.meta["line"] + len(S.STOP_LINE) - 1
    for c in S.unquote_cases():
        w = S.tile_windows(b"", c.body)
        assert len(w) == 1 and len(w[0].lines) <= S.LCAP
    for c in S.template_cases():
        if "stops" in c.meta:
            assert c.meta["stops"] in (S.W_STOPS - 1, S.W_STOPS, S.W_STOPS + 1)
    assert sorted(c.meta["stops"] for c in S.template_cases() if "stops" in c.meta) == [95, 96, 97]
    assert sorted(c.meta["struct"] for c in S.template_cases() if "struct" in c.meta) == [62, 63, 64]
    assert sorted(c.meta["wild"] for c in S.template_cases() if "wild" in c.meta) == [39, 40, 41]


def test_template_words_hand_worked():
    # "a" key: 2 stops, literal segments "{" (1 byte), ":" ... ; "x" value: a wildcard; 4 stops in all
    assert S.template_words(b'{"a":"x"}') == (7 + 5 + 0 + 1, 4, 1)
    assert S.template_words(b'{"key1":12345}') == (7 + 3 + 2 + 1, 2, 1)          # "key1" and ":" + "}" around the integer
    assert S.template_words(b'{"a":[1,2]}') is None                                # two integers in one segment
    assert S.template_words(b'{"' + b"k" * 256 + b'":1}') is None                 # a literal segment longer than 255 bytes
    assert S.template_words(S._wild_line(S.REC_MAX - 1)[6:-1])[2] == S.REC_MAX
    assert S.template_words(S._wild_line(S.REC_MAX)[6:-1]) is None
    line = b"{" + b",".join(b'"k%d":0' % i for i in range(31)) + b"}"               # 62 stops, then 64
    assert S.template_words(line)[1] == 62
    assert S.template_words(line[:-1] + b',"z":0}') is None


def test_pack_batches_land_on_their_seams():
    seen = collections.Counter()
    for b in S.tile_pack_batches():
        n = len(b.bodies)
        if b.first_cut is None:
            tiles = S.plan_tiles([0] * n, [len(x) for x in b.bodies], [1] * n)
        else:
            carry = [orc.passthrough(x[:c]).tail_len for x, c in zip(b.bodies, b.first_cut)]
            live = [not orc.reframe(x[:c]).terminated for x, c in zip(b.bodies, b.first_cut)]
            tiles = S.plan_tiles(carry, [len(x) - c for x, c in zip(b.bodies, b.first_cut)], live)
            assert tiles[0] == (0, S.MAX_TSEGS) and sum(1 - x for x in live[:S.MAX_TSEGS]) == 32
            seen["finished"] += 1
            continue
        if b.label == "tile.pack_sum":
            assert tiles[0] == (0, 3 if b.meta["d"] <= 0 else 2)
            assert sum(S.r16(len(x)) for x in b.bodies[:3]) == S.TILE + b.meta["d"]
        elif b.label == "tile.pack_count":
            assert tiles[0] == (0, min(n, S.MAX_TSEGS)) and len(tiles) == -(-n // S.MAX_TSEGS)
        elif b.label == "tile.pack_group":
            firsts = [f for f, _ in tiles]
            assert (S.PLAN_GROUP in firsts) == (n > S.PLAN_GROUP)
        elif b.label == "tile.pack_whole":
            assert tiles[1] == (3, 1) and S.r16(len(b.bodies[3])) == S.TILE + b.meta["extra"]
        seen[b.label] += 1
    assert seen == {"tile.pack_sum": 3, "tile.pack_count": 5, "tile.pack_group": 4, "tile.pack_whole": 2, "finished": 1}


def test_limit_cases_sit_on_the_limit():
    for limit in (16384, 32768):
        cs = S.limit_cases(limit)
        assert sorted({c.meta["n"] for c in cs}) == [limit - 2, limit - 1, limit, limit + 1]
        for c in cs:
            a, e = c.meta["line"]
            assert e - a == c.meta["n"]
            if c.label == "limit.big_tail":
                w = S.tile_windows(b"", c.body)
                assert len(w) >= 2 and w[-1].carried == c.meta["line"][0]       # the last window holds the tail back
            if c.label == "limit.big_carry":
                assert S.r16(c.cuts[0] - len(S.FIRST)) + S.r16(len(c.body) - c.cuts[0]) > S.TILE
            if c.label == "limit.big_window":
                w = S.tile_windows(b"", c.body)
                assert a >= w[1].s0


def _model_agrees(body: bytes):
    v = orc.reframe(body)
    m = sm.run_with_stream(body)
    assert [ln.out for ln in v.lines if ln.kind == orc.L_EMITTED] == m["frames"]
    assert v.builder == m["builder"] and v.acc_content == m["content"]
    assert v.has_tool_calls == m["has_tool_calls"] and v.terminated == m["terminated"]
    assert [ln.payload for ln in v.lines if ln.kind in (orc.L_EMITTED, orc.L_DONE, orc.L_DONE_EXACT)] == sm.decoded_payloads(body, True)
    p = orc.passthrough(body, parse=True)
    assert [ln.out for ln in p.lines] == sm.lines(body)
    assert [ln.payload for ln in p.lines if ln.chunk is not None] == sm.decoded_payloads(body, False)
    return v.terminated


def test_oracle_and_stream_model_agree_on_every_seam_stream():
    bodies = {c.body for c in S.all_cases()}
    bodies |= {b for bt in S.tile_pack_batches() for b in bt.bodies}
    bodies |= {b for bt in S.tile_round_batches() for b in bt.bodies}
    bodies.add(S.template_store_body())
    n_term = sum(_model_agrees(b) for b in sorted(bodies))
    assert len(bodies) > 1000 and n_term > 300
