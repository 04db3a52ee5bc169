"""CPU: the agent and telemetry folds (csrc/sse_fold.cpp) on the oracle's records of adversarial streams, laid out as the
kernels lay them out (tests/folds.py::Layout: several runs per segment, zero-copy frames and spans, spans in all three arenas,
a stream's records over several results), against the oracle's agent.go and telemetry.go restatements."""
import ctypes as C

import pytest

from inference_gateway_b200 import _abi as A
from oracle import orc
from tests import folds, go_model
from tests.util import DONE, agent_results, check_agent, chunk_to_dict, irregular_telemetry, telemetry_results

R, PP = A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE
# (results a stream's records are spread over, longest run in lines)
LAYOUTS = [(1, 64), (3, 64), (17, 5)]


def judge(L, body, mode, layout, label):
    """Both folds fed every result of the layout, against the oracle: the fold verdict of tests/util.py::check_folds, per
    result instead of per piece. Returns the agent fold's state (mode R, no line past the nesting limit) or None."""
    mode_r = bool(mode & A.MODE_R)
    v = orc.reframe(body) if mode_r else orc.passthrough(body, parse=True)
    lay = folds.Layout(v, mode_r, *layout, seed=len(body))
    ag, te, rcs = folds.feed(L, lay, mode_r)
    try:
        want = [(A.SSE_ERR_UNDECODED,) * 2 if u else (A.SSE_OK,) * 2 for u in lay.undecoded]
        assert rcs == want, f"{label}: feed codes {rcs}, want {want}"
        if any(lay.undecoded):
            return None
        state = None
        out = v.out
        if mode_r:
            state = agent_results(L, ag)
            check_agent(state, v, label)
            A.check(L.sse_telemetry_feed_bytes(te, DONE, len(DONE)), "sse_telemetry_feed_bytes")
            out += DONE
        rc, usage, calls = telemetry_results(L, te)
        if irregular_telemetry(out):
            assert rc == 1, f"{label}: telemetry finished with {rc} on a body with an irregular piece"
        else:
            assert (rc, usage, calls) == (0, *orc.telemetry(out)), f"{label}: telemetry differs"
        return state
    finally:
        L.sse_agent_free(ag)
        L.sse_telemetry_free(te)


@pytest.fixture(scope="module")
def corpus():
    return folds.corpus(small=True)


@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda x: f"results{x[0]}-runs{x[1]}")
@pytest.mark.parametrize("mode", [R, PP], ids=["R", "PP"])
@pytest.mark.parametrize("family", ["adversarial", "tricky", "tc_strings", "near_misses", "merge"])
def test_folds_match_the_oracle(corpus, family, mode, layout):
    L = A.load()
    n_limited = n_irregular = 0
    for i, body in enumerate(corpus[family]):
        judge(L, body, mode, layout, f"{family} stream {i} mode {mode} layout {layout}")
        v = orc.passthrough(body, parse=True)
        n_limited += any(l.depth_limited for l in v.lines)
        n_irregular += irregular_telemetry(v.out)
    if family == "adversarial":          # the corpus reaches both exceptions to the plain verdict
        assert n_limited and n_irregular


def test_the_layouts_reach_every_place_a_fold_reads():
    """The layouts put frames in both arenas, strings in all three, segments over several runs and results."""
    L = A.load()
    body = folds.merge_streams()[2]
    lay = folds.Layout(orc.reframe(body), True, 3, 5, seed=1)
    frames_in = spans_text = spans_out = spans_in = runs = 0
    for res, s in lay.results:
        runs += res.n_runs
        for k in range(res.n_frames):
            frames_in += res.frames[k].off >= folds.IN_BASE
        for k in range(res.n_tcs):
            t = res.tcs[k]
            if t.id_len:
                spans_text += bool(t.flags & A.TC_ID_TEXT)
                spans_out += not t.flags & A.TC_ID_TEXT and t.id_off < folds.IN_BASE
                spans_in += t.id_off >= folds.IN_BASE
    assert frames_in and spans_text and spans_out and spans_in and runs > 10
    assert judge(L, body, R, (3, 5), "layout")[4][99]["id"] == b"id99"


@pytest.mark.parametrize("mode", [R, PP], ids=["R", "PP"])
@pytest.mark.parametrize("n", folds.SATURATED)
def test_saturated_tool_call_chains_are_walked_to_their_end(n, mode):
    """tc_count saturates at 0xFFFF: a chunk of 65,536 or more elements must not lose the ones past it in either fold."""
    L = A.load()
    body = folds.HEAD + folds.saturated_line(n) + folds.USAGE + folds.STOP + DONE
    for layout in ((1, 64), (2, 3)):
        state = judge(L, body, mode, layout, f"{n} elements mode {mode}")
        if mode & A.MODE_R:
            calls = state[4]
            assert [c["id"] for c in calls[1:]] == [b"id%d" % k for k in range(n - 4, n)]
            assert [c["args"] for c in calls[1:]] == [b"a%d" % k for k in range(n - 4, n)]


def test_empty_choices_array_starts_choice_zero_anew():
    """decode.go array(): "choices":[] sets a fresh slice of capacity 0, so a later "choices" array's element 0 starts empty
    and the agent keeps nothing of the chunk's first array."""
    first = b'{"choices":[{"delta":{"content":"a"},"finish_reason":"stop"}],'
    cases = {
        first + b'"choices":[],"choices":[{"delta":{}}]}': dict(n_choices=1, content=b"", finish=0),
        first + b'"choices":[],"choices":null}': dict(n_choices=0),
        first + b'"choices":[]}': dict(n_choices=0),
        b'{"choices":[{"delta":{"tool_calls":[{"index":0,"id":"c","function":{"name":"f","arguments":"x"}}]},'
        b'"finish_reason":"tool_calls"}],"choices":[ ],"choices":[{"delta":{"content":"b"}}]}':
            dict(n_choices=1, content=b"b", finish=0, tcs=[], tc_nonnil=False),
        b'{"choices":[{"delta":{"content":"a"}}],"choices":[],"choices":[{"finish_reason":"stop"}],'
        b'"choices":[{"delta":{"content":"c"}}]}': dict(n_choices=1, content=b"c", finish=orc.FIN_STOP),
    }
    L = A.load()
    for doc, want in cases.items():
        got = chunk_to_dict(orc.unmarshal(doc))
        assert got["json_ok"] and {k: got[k] for k in want} == want, doc
        assert go_model.unmarshal(doc) == got, doc
        body = folds.HEAD + b"data: " + doc + b"\n\n" + folds.TAIL + folds.STOP
        v = orc.reframe(body)
        terminates = want.get("finish") == orc.FIN_STOP
        assert v.acc_content == b"before " + want.get("content", b"") + (b"" if terminates else b"after")
        assert v.terminated and v.term_finish == (orc.FIN_STOP if terminates else orc.FIN_TOOL_CALLS)
        assert judge(L, body, R, (1, 64), doc)[:4] == (v.acc_content, v.has_tool_calls, True, v.term_finish)


def test_a_line_past_the_nesting_limit_makes_both_feeds_refuse_their_result():
    L = A.load()
    deep = b"data: " + b"[" * 129 + b"]" * 129 + b"\n\n"
    body = folds.HEAD + folds.TAIL * 80 + deep + folds.TAIL * 80 + folds.STOP
    for mode in (R, PP):
        for layout in LAYOUTS:
            assert judge(L, body, mode, layout, "deep") is None
