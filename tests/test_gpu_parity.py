"""GPU parity: libssegpu.so (through its C ABI) vs the CPU oracle, bit-exact, on the same inputs.

Covers SURVEY.md Appendix B vectors, the reference's own fixtures (tests/golden/ref_fixtures.json), the
BASELINE.json configs at reduced stream counts, ragged/edge inputs and a JSON mutation fuzz.
"""
import ctypes as C
import json
import os

import numpy as np
import pytest

from inference_gateway_b200 import _abi as A
from inference_gateway_b200 import synth
from oracle import orc
from tests.corpus import TRICKY, mutate as _mutate
from tests.util import agent_results, check_agent, check_streams, run_streams

pytestmark = pytest.mark.gpu

P, R, PP = A.MODE_P, A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "ref_fixtures.json")))["fixtures"]


def _run_and_check(engine, bodies, modes, n_batches=1, seed=0, folds=False):
    outs = run_streams(engine, bodies, modes, n_batches=n_batches, seed=seed, with_folds=folds)
    views = check_streams(bodies, modes, outs, f"batches {n_batches}")
    return outs, views


# ------------------------------------------------------------------ SURVEY.md Appendix B
APPENDIX_P = [
    (b'data: {"a":1}\n\ndata: [DONE]\n\n', b'data: {"a":1}\n\ndata: [DONE]\n\n'),      # P1
    (b"data: x\r\n\r\ndata: y", b"data: x\r\n\r\n"),                                  # P2: tail dropped
    (b"", b""),                                                                       # P3
    (b": ping\n\nevent: x\ndata: 1\n\n", b": ping\n\nevent: x\ndata: 1\n\n"),          # P4
    (b"x" * 10000 + b"\n", b"x" * 10000 + b"\n"),                                     # P5: > bufio's 4096
]


def test_appendix_b_passthrough(engine):
    bodies = [i for i, _ in APPENDIX_P]
    outs, _ = _run_and_check(engine, bodies, [P] * len(bodies))
    for (inp, exp), o in zip(APPENDIX_P, outs):
        assert b"".join(o.frames) == exp
    # P1 is delivered as 4 channel elements (provider.go:322-334)
    assert outs[0].frames == [b'data: {"a":1}\n', b"\n", b"data: [DONE]\n", b"\n"]


APPENDIX_R = [
    (b'data: {"choices":[{"index":0,"delta":{"content":"Hi"},"finish_reason":null}]}\n',
     [b'data: {"choices":[{"index":0,"delta":{"content":"Hi"},"finish_reason":null}]}\n\n']),     # R1
    (b'\n: ping\nevent: m\ndata:{"x":1}\ndata: \n', []),                                           # R2
    (b'  data: {"x":1} \r\n', [b'data: {"x":1}\n\n']),                                             # R3
    (b'data:  {"x":1}\n', [b'data:  {"x":1}\n\n']),                                                # R4
    (b"data: [DONE]\n", []),                                                                       # R5
    (b'data: {"choices":[{"index":0,"delta":{"content":"say [DONE]"},"finish_reason":null}]}\n', []),  # R6
    (b"data: {oops\n", [b"data: {oops\n\n"]),                                                      # R7
    (b'data: {"choices":[{"index":0,"delta":{},"finish_reason":"stop"}]}\n\ndata: {"choices":[],"usage":{"prompt_tokens":1,"completion_tokens":2,"total_tokens":3}}\n\ndata: [DONE]\n\n',
     [b'data: {"choices":[{"index":0,"delta":{},"finish_reason":"stop"}]}\n\n']),                   # R8
]


def test_appendix_b_reframe(engine):
    bodies = [i for i, _ in APPENDIX_R]
    outs, _ = _run_and_check(engine, bodies, [R] * len(bodies))
    for (inp, exp), o in zip(APPENDIX_R, outs):
        assert o.frames == exp, inp
    assert outs[7].terminated


# ------------------------------------------------------------------ reference fixtures
def _fixture_bodies(fx):
    for it in fx["iterations"]:
        if fx["kind"] == "channel_elements":
            yield ("\n".join(it) + "\n").encode()
        else:
            body = it[0]
            yield (body if body.endswith("\n") else body + "\n").encode()


@pytest.mark.parametrize("fx", [f for f in GOLD if "content" in f["expect"]], ids=lambda f: f["name"])
def test_reference_fixtures_agent(engine, fx):
    """The semantic assertions the reference tests make on these streams (cited in the golden file)."""
    bodies = list(_fixture_bodies(fx))
    outs, views = _run_and_check(engine, bodies, [R] * len(bodies), n_batches=3, seed=7, folds=True)
    exp = fx["expect"]
    fin_names = {1: "stop", 2: "tool_calls"}
    for i, o in enumerate(outs):
        content, has, term, fin, calls = agent_results(engine.L, o.agent)
        assert content.decode() == exp["content"][i]
        assert term and fin_names[fin] == exp["finish"][i]
        want = exp["tool_calls"][i]
        assert has == bool(want)
        got = [dict(id=c["id"].decode(), name=c["name"].decode(), args=c["args"].decode()) for c in calls]
        assert got == want
        # frames never contain [DONE]; the agent appends exactly one at the very end (agent.go:140-143)
        assert all(b"[DONE]" not in f for f in o.frames)
        # same answers from the oracle's own restatement of agent.go:377-481
        ocalls = orc.parse_tool_calls(views[i].builder)
        assert [dict(id=c["id"].decode(), name=c["name"].decode(), args=c["args"].decode()) for c in ocalls] == want
        assert views[i].acc_content.decode() == exp["content"][i]
        if exp["usage"][i] is not None:
            usage_recs = [r for r in o.recs if r.get("usage")]
            assert usage_recs and list(usage_recs[-1]["usage"]) == exp["usage"][i]


@pytest.mark.parametrize("fx", [f for f in GOLD if "parsed" in f["expect"]], ids=lambda f: f["name"])
def test_reference_fixtures_builder(engine, fx):
    body = (fx["iterations"][0][0] + "\n").encode()
    outs, views = _run_and_check(engine, [body], [R], folds=True)
    _, _, _, _, calls = agent_results(engine.L, outs[0].agent)
    got = [dict(id=c["id"].decode(), name=c["name"].decode(), args=c["args"].decode()) for c in calls]
    assert got == fx["expect"]["parsed"]


@pytest.mark.parametrize("fx", [f for f in GOLD if "frames" in f["expect"]], ids=lambda f: f["name"])
def test_reference_fixtures_dropped_elements(engine, fx):
    """tests/middlewares/mcp_test.go:537: an element without the "data: " prefix is dropped by the agent (agent.go:186-188)."""
    bodies = list(_fixture_bodies(fx))
    outs, views = _run_and_check(engine, bodies, [R] * len(bodies), n_batches=2, seed=3, folds=True)
    for o in outs:
        assert o.frames == [] and o.recs == [] and not o.terminated
        content, has, term, fin, calls = agent_results(engine.L, o.agent)
        assert content == b"" and not has and not term and calls == []


# ------------------------------------------------------------------ BASELINE.json configs (reduced stream counts)
@pytest.mark.parametrize("name,n_streams,n_batches", [
    ("C1", 1, 1), ("C1", 1, 9), ("C2", 256, 1), ("C2", 256, 4), ("C3", 256, 1), ("C3", 256, 5),
    ("C4", 512, 1), ("C4", 512, 6)])
def test_configs(engine, name, n_streams, n_batches):
    streams, mode = synth.make_config(name, n_streams=n_streams)
    bodies = [b for b, _, _ in streams]
    if mode is None:    # C1: both modes
        for m in (P, R, PP):
            _run_and_check(engine, bodies, [m] * len(bodies), n_batches=n_batches, seed=11)
    else:
        _run_and_check(engine, bodies, [mode] * len(bodies), n_batches=n_batches, seed=13)


def test_mixed_modes_and_folds(engine):
    streams, _ = synth.make_config("C4", n_streams=300)
    bodies = [b for b, _, _ in streams]
    modes = [(R, PP, P)[i % 3] for i in range(len(bodies))]
    outs = run_streams(engine, bodies, modes, n_batches=4, seed=3, with_folds=True)
    # mode R: telemetry over what the MCP path would have written (frames + the final [DONE] the host writes, mcp.go:253-299,
    # agent.go:140-143); telemetry.go:190-277 over the body the client got
    check_streams(bodies, modes, outs, "mixed", engine.L)


def test_bare_done_line_does_not_stop_tool_call_parsing(engine):
    """agent.go:181-184 swallows every line that contains "[DONE]", but parseStreamingToolCalls only breaks on the exact line
    "data: [DONE]" (agent.go:394-396): after a bare "[DONE]" (no prefix, or padded) later tool-call chunks still count; after
    "data: [DONE]" they do not."""
    tc1 = b'data: {"choices":[{"delta":{"tool_calls":[{"index":0,"id":"a","function":{"name":"first","arguments":"{"}}]}}]}\n\n'
    tc2 = b'data: {"choices":[{"delta":{"tool_calls":[{"index":0,"function":{"arguments":"}"}},{"index":1,"id":"b","function":{"name":"second"}}]}}]}\n\n'
    fin = b'data: {"choices":[{"delta":{},"finish_reason":"tool_calls"}]}\n\n'
    bodies = [tc1 + b"[DONE]\n\n" + tc2 + fin, tc1 + b"  [DONE]  \n\n" + tc2 + fin, tc1 + b"data: [DONE]\n\n" + tc2 + fin,
              tc1 + b"data: [DONE] \n\n" + tc2 + fin, b"[DONE]\n" + tc1 + tc2 + fin]
    for nb in (1, 4):
        outs, views = _run_and_check(engine, bodies, [R] * len(bodies), n_batches=nb, seed=nb, folds=True)
        names = []
        for o, v in zip(outs, views):
            state = agent_results(engine.L, o.agent)
            check_agent(state, v, f"bare [DONE] x{nb}")
            content, has, term, fin_code, calls = state
            assert term and fin_code == 2
            names.append([c["name"] for c in calls])
        # "data: [DONE] " trims to the exact line too (strings.TrimSpace first, agent.go:178)
        assert names == [[b"first", b"second"], [b"first", b"second"], [b"first"], [b"first"], [b"first", b"second"]]


# ------------------------------------------------------------------ ragged / edge inputs
def test_edges(engine):
    nl = b"\n"
    bodies = [
        b"", nl, nl * 200, b"\r\n" * 50, b"no newline at all",
        b"data: a\n" * 150,                                   # > 64 lines in one segment: several runs
        (b"data: " + b"y" * 9000 + b"\n") * 3 + b"data: tail",   # lines longer than the window
        b"data: " + b"z" * 30000 + b"\n\n" + b'data: {"choices":[{"delta":{"content":"after"}}]}\n\n',
        ("　  data: {\"x\":1}  \n").encode(),   # unicode TrimSpace
        b"\xc2\xa0data: x\xe2\x80\n",                         # incomplete UTF-8 space is not trimmed
        b"data: [DONE] [DONE] [DONE]\n" * 40,                 # more [DONE] hits than the per-round list holds
        b'data: {"a":"[DONE"}\ndata: {"b":"DONE]"}\ndata: [DONE\n',
        b"DATA: x\ndata:x\ndata: \ndata:  \ndata: \t\n",
    ]
    for m in (P, R, PP):
        for nb in (1, 3, 8):
            _run_and_check(engine, bodies, [m] * len(bodies), n_batches=nb, seed=nb)


def test_line_longer_than_carry_slot_fails_loudly(engine):
    big = b"data: " + b"q" * 100000 + b"\n" + b"data: after\n"
    outs = run_streams(engine, [big], [P], n_batches=1)
    assert outs[0].flags & A.SEG_LINE_TOO_LONG and outs[0].flags & A.SEG_DEAD
    outs = run_streams(engine, [big, b"data: ok\n"], [R, R], n_batches=4)
    assert outs[0].flags & A.SEG_DEAD
    assert outs[1].frames == [b"data: ok\n\n"]


def test_reset_conn_starts_a_new_stream(engine):
    body = b'data: {"choices":[{"delta":{"content":"a"},"finish_reason":"stop"}]}\n\ndata: {"choices":[{"delta":{"content":"unread"}}]}\n\n'
    engine.reset_all()
    slot, res = engine.process([(5, R, body)])
    assert len(res.seg_frames(0)) == 1 and int(res.segs[0]["flags"]) & A.SEG_TERMINATED
    engine.release(slot)
    slot, res = engine.process([(5, R, body)])       # finished: bytes are never read (agent.go:169)
    assert res.seg_frames(0) == [] and int(res.segs[0]["flags"]) & A.SEG_FINISHED
    engine.release(slot)
    engine.reset_conn(5)                              # next agent iteration / new request
    slot, res = engine.process([(5, R, body)])
    assert len(res.seg_frames(0)) == 1
    engine.release(slot)


# ------------------------------------------------------------------ JSON decoding fuzz
def test_json_decoding_tricky(engine):
    body = b"".join(b"data: " + d.replace(b"\n", b" ") + b"\n" for d in TRICKY)
    # each document on its own connection so that early termination cannot hide later ones
    bodies = [b"data: " + d.replace(b"\n", b" ") + b"\n" for d in TRICKY]
    _run_and_check(engine, bodies, [R] * len(bodies))
    _run_and_check(engine, [body], [PP], n_batches=5, seed=2)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_json_decoding_fuzz(engine, seed):
    rng = np.random.default_rng(1000 + seed)
    streams, _ = synth.make_config("C4", n_streams=60)
    docs = []
    for b, _, _ in streams:
        for ev in b.split(b"\n\n"):
            if ev.startswith(b"data: {"):
                docs.append(ev[6:])
    docs += TRICKY
    mutated = [_mutate(rng, docs[int(rng.integers(0, len(docs)))]) for _ in range(3000)]
    bodies = [b"data: " + d + b"\n" for d in mutated]
    _run_and_check(engine, bodies, [R] * len(bodies))
    # and as a single passthrough+parse stream cut into pieces (no early termination in mode P)
    _run_and_check(engine, [b"".join(bodies)], [PP], n_batches=7, seed=seed)


def test_product_does_not_use_oracle():
    import inference_gateway_b200
    root = os.path.dirname(inference_gateway_b200.__file__)
    for dirpath, _, files in os.walk(root):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                src = open(os.path.join(dirpath, f), encoding="utf-8").read()
                assert "import oracle" not in src and "from oracle" not in src and "sse_oracle" not in src, f


# ------------------------------------------------------------------ chains of near-identical lines (split pipeline)
def test_line_chains(engine):
    """Consecutive chunks that differ only inside the content string are derived from the previous parse; every other
    kind of difference has to fall back to a full decode. All of it must stay bit-exact."""
    env = '{"id":"chatcmpl-%s","object":"chat.completion.chunk","created":%s,"model":"m","choices":[{"index":0,"delta":{%s},"finish_reason":%s}]%s}'

    def ev(content=None, cid="abc123", created="1700000000", fin="null", tail="", extra=""):
        delta = extra + ('"content":"%s"' % content if content is not None else "")
        return ("data: " + env % (cid, created, delta, fin, tail) + "\n\n").encode()

    streams = [
        # plain content deltas of different lengths (the common case)
        b"".join(ev(w) for w in ["Hello", " there", ", this is a much longer piece of plain content that spans more than sixteen bytes",
                                 "", "x", " and some more words to keep the chain going for a while", "!"]) + ev(fin='"stop"'),
        # identical consecutive lines, then a line that only differs in `created`, then in the id
        ev("same") + ev("same") + ev("same", created="1700000001") + ev("same", cid="abc124") + ev("other"),
        # escapes, quotes, unicode and control escapes inside the content break the chain at that line only
        ev("plain one") + ev('with \\"quotes\\"') + ev("plain two") + ev("café") + ev("plain three") + ev("tab\\tchar") + ev("plain four"),
        # the difference extends past the content string (finish_reason changes, usage appears)
        ev("a") + ev("b", fin='"length"') + ev("c") + ev("d", tail=',"usage":{"prompt_tokens":1,"completion_tokens":2,"total_tokens":3}') + ev("e"),
        # tool-call argument fragments: plain differences inside `arguments`, not inside content
        b"".join(ev(None, extra='"tool_calls":[{"index":0,"function":{"arguments":"%s"}}]' % a) for a in ["abc", "defgh", "i", "jklmnopqrstuvwxyz0123456789"]),
        # content key twice, role key present, content null
        ev("x", extra='"content":"first",') + ev("y", extra='"content":"first",') + ev("z", extra='"role":"assistant",') + ev("w", extra='"role":"assistant",'),
        # very long plain content (several windows of skip) and a chain across it
        ev("p" * 3000) + ev("q" * 2500) + ev("r" * 10) + ev("s" * 3500),
        # invalid JSON lines in a chain
        ev("ok") + b'data: {"choices":[{"delta":{"content":"broken"}}\n\n' + b'data: {"choices":[{"delta":{"content":"brokeN"}}\n\n' + ev("ok again"),
    ]
    for m in (R, PP):
        for nb in (1, 2, 5):
            _run_and_check(engine, streams, [m] * len(streams), n_batches=nb, seed=40 + nb)


def test_overflow_is_reported_not_hidden():
    """A result arena that is too small fails the batch loudly and says which capacity to raise."""
    from inference_gateway_b200 import SseEngine
    eng = SseEngine(device=0, max_conns=8, bytes_per_batch=1 << 16, max_frames=4, max_recs=4)
    try:
        body = b"data: {\"choices\":[]}\n\n" * 50
        slot, arena, segs = eng.acquire()
        n, nb = eng.fill(arena, segs, [(0, R, body)])
        eng.submit(slot, n, nb)
        with pytest.raises(A.SseError) as e:
            eng.collect(slot)
        assert e.value.status == A.SSE_ERR_OVERFLOW and "overflow mask 0x1" in str(e.value)
        eng.release(slot)
    finally:
        eng.close()


# ------------------------------------------------------------------ zero-copy frames (arena offsets >= in_base)
def _one_batch(eng, items):
    slot, res = eng.process(items)
    try:
        offs = [[int(res.frames[k]["off"]) for ff, fc, _, _ in res.seg_runs(i) for k in range(ff, ff + fc)] for i in range(len(items))]
        frames = [res.seg_frames(i) for i in range(len(items))]
        return offs, frames, int(res.raw.out_bytes), res.in_base
    finally:
        eng.release(slot)


def test_zero_copy_frames_are_spans_of_the_input_arena():
    """Default path: a frame whose bytes already stand in the input arena is returned as a span of it (nothing is written to
    the out arena, nothing comes back over PCIe); anything that had to be assembled is materialised. SSE_FLAG_COPY_OUT
    materialises every frame. The bytes are the oracle's either way."""
    from inference_gateway_b200 import SseEngine
    ev = b'data: {"choices":[{"index":0,"delta":{"content":"hello"},"finish_reason":null}]}'
    usual = (ev + b"\n\n") * 7 + b"data: [DONE]\n\n"
    crlf = (ev + b"\r\n\r\n") * 3                      # reframing changes the bytes: materialised in mode R
    padded = b"  " + ev + b" \n\n" + ev + b"\n\n"       # first event is trimmed at the end: materialised; second is not
    nosep = ev + b"\n" + ev + b"\n\n"                   # first line has no blank separator: "\n\n" must be synthesised
    for flags in (0, A.FLAG_COPY_OUT):
        eng = SseEngine(device=0, max_conns=16, bytes_per_batch=1 << 20, flags=flags)
        try:
            eng.reset_all()
            offs, frames, out_bytes, in_base = _one_batch(eng, [(0, R, usual), (1, P, usual), (2, R, crlf), (3, P, crlf),
                                                                (4, R, padded), (5, R, nosep)])
            for i, (body, mode) in enumerate([(usual, R), (usual, P), (crlf, R), (crlf, P), (padded, R), (nosep, R)]):
                v = orc.reframe(body) if mode & A.MODE_R else orc.passthrough(body)
                exp = [l.out for l in v.lines if l.kind == orc.L_EMITTED] if mode & A.MODE_R else [l.out for l in v.lines]
                assert frames[i] == exp
            zc = [[o >= in_base for o in oo] for oo in offs]
            if flags & A.FLAG_COPY_OUT:
                assert not any(any(z) for z in zc) and out_bytes > 0
            else:
                assert all(zc[0]) and all(zc[1]) and all(zc[3])          # usual framing, and every mode P line
                assert not any(zc[2])                                    # \r\n lines are rewritten by the reframe
                assert zc[4] == [False, True] and zc[5] == [False, True]
            # second micro-batch: the first line of each segment continues a held-back tail -> assembled -> materialised
            eng.reset_all()
            cut = len(ev) // 2
            _one_batch(eng, [(0, R, usual[:cut]), (1, P, usual[:cut])])
            offs, frames, _, in_base = _one_batch(eng, [(0, R, usual[cut:]), (1, P, usual[cut:])])
            assert frames[0][0] == ev + b"\n\n" and frames[1][0] == ev + b"\n"
            if not flags:
                assert offs[0][0] < in_base and offs[1][0] < in_base
                assert all(o >= in_base for o in offs[0][1:]) and all(o >= in_base for o in offs[1][1:])
        finally:
            eng.close()


def test_provider_hint_only_schedules(engine):
    """sse_seg.provider feeds the decode kernel's work-item sort (lanes of a batch walk alike lines); results never depend on it."""
    streams, _ = synth.make_config("C4", n_streams=96)
    bodies = [b for b, _, _ in streams]
    got = []
    for hint in (0, 1, 2):
        engine.reset_all()
        slot, arena, segs = engine.acquire()
        n, nb = engine.fill(arena, segs, [(c, R, b) for c, b in enumerate(bodies)])
        segs["provider"][:n] = {0: 0, 1: np.arange(n) % 4, 2: np.random.default_rng(5).integers(0, 256, n)}[hint]
        engine.submit(slot, n, nb)
        res = engine.collect(slot)
        try:
            from tests.util import rec_to_dict
            got.append([(res.seg_frames(i), [{k: v for k, v in rec_to_dict(res, r).items() if k != "frame"} for r in res.seg_recs(i)],
                         int(res.segs[i]["flags"])) for i in range(n)])   # frame indices are bump-allocated: not comparable across runs
        finally:
            engine.release(slot)
    assert got[0] == got[1] == got[2]
    for i, b in enumerate(bodies):
        v = orc.reframe(b)
        assert got[0][i][0] == [l.out for l in v.lines if l.kind == orc.L_EMITTED]


def test_finish_reason_is_case_sensitive(engine):
    """Keys match case-insensitively, finish_reason values do not: "STOP" or "Tool_Calls" is some other reason, and does not end
    the stream (agent.go:235-242 compares with "stop" / "tool_calls")."""
    after = b'data: {"choices":[{"delta":{"content":"after"}}]}\n\n'
    bodies = [b'data: {"choices":[{"delta":{},"finish_reason":"%s"}]}\n\n' % f + after
              for f in (b"STOP", b"Stop", b"TOOL_CALLS", b"Tool_Calls", b"LENGTH", b"stop")]
    outs, _ = _run_and_check(engine, bodies, [R] * len(bodies))
    assert [o.terminated for o in outs] == [False] * 5 + [True]
    assert [r["finish"] for o in outs[:5] for r in o.recs[:1]] == [7] * 5


def test_done_marker_at_every_alignment(engine):
    """agent.go:181 is a substring test: "[DONE]" anywhere in the trimmed line swallows it. The produce scan finds candidates
    16 bytes per lane ('[' followed by 'D', with the chunk's last byte handled conservatively): every alignment of the
    marker relative to the 16-byte chunks, near misses, and markers split by a batch boundary must agree with the oracle."""
    bodies = []
    for pad in range(0, 40):
        fill = "x" * pad
        for marker in ("[DONE]", "[DONE", "[D", "[", "[DONEE]", "[done]", "[[DONE]]", "[D[DONE]"):
            bodies.append(('data: {"choices":[{"delta":{"content":"%s%s tail"}}]}\n\n' % (fill, marker)).encode() +
                          b'data: {"choices":[{"delta":{"content":"next"}}]}\n\n')
    bodies.append(b"data: " + b"[" * 70 + b"DONE]\n\n" + b"data: {}\n\n")
    bodies.append(b"[DONE]\n[DONE]\n\ndata: x[DONE]\n\n   data: [DONE]   \n\ndata: {\"a\":1}\n\n")
    for nb in (1, 2, 3):
        _run_and_check(engine, bodies, [R] * len(bodies), n_batches=nb, seed=60 + nb)
