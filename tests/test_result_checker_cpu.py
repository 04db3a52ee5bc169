"""CPU: the structural checker of one batch result (oracle/orc_check.c::orc_check_result) on hand-made sse_result arrays. A
well-formed result passes; each case breaks exactly one rule and the checker must name it first."""
import ctypes as C

import numpy as np
import pytest

from inference_gateway_b200 import _abi as A
from inference_gateway_b200.engine import FRAME_DT, REC_DT, RUN_DT, SEG_DT, SEGRES_DT, TC_DT, USAGE_DT
from oracle import orc

IN_BASE = 1024
OUT_BYTES, TEXT_BYTES = 64, 16
R, PP = A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE
N = A.NONE
OK, DONE = A.F_JSON_OK, A.F_DONE_LINE
STOP = 1 << A.F_FINISH_SHIFT


def well_formed() -> dict:
    """Two segments.
    seg 0, mode R, input [0, 200): the inline run has frames 0-1 and records 0-2, then runs[0] has frame 2 and record 3.
      rec 0 -> frame 0 (zero-copy), usage 0, a chain of two tool calls, decoded content in the text arena;
      rec 1: a swallowed [DONE] line (no frame), its content a span of the out arena;
      rec 2 -> frame 1 (materialised in the out arena), decoded content;
      rec 3 -> frame 2 (zero-copy), content a span of its own payload, finish_reason stop: terminates the segment.
    seg 1, mode P|PARSE, input [208, 308), 5 bytes held back: frames 3 (": ping") and 4, rec 4 -> frame 4.
    runs[1], frame 5 and record 5 are holes no run refers to (SSE_FLAG_DEFER leaves such holes)."""
    frames = np.zeros(6, FRAME_DT)
    frames[0] = (IN_BASE + 0, 30)        # "data: " + 22 payload bytes + "\n\n"
    frames[1] = (0, 40)                  # out arena, 32 payload bytes
    frames[2] = (IN_BASE + 50, 20)       # 12 payload bytes
    frames[3] = (IN_BASE + 208, 7)       # ": ping\n"
    frames[4] = (IN_BASE + 215, 27)      # "data: " + 20 payload bytes + "\n"
    frames[5] = (IN_BASE + 260, 9)
    recs = np.zeros(6, REC_DT)
    #            frame flags                                              c_off            c_len tc_first tc_count n_ch usage pay
    recs[0] = (0, OK | A.F_HAS_USAGE | A.F_CONTENT_TEXT | A.F_TC_NONNIL, 0, 5, 0, 2, 1, 0, 22)
    recs[1] = (N, OK | DONE, 48, 4, N, 0, 1, N, 10)
    recs[2] = (1, OK | A.F_CONTENT_TEXT, 5, 4, N, 0, 1, N, 32)
    recs[3] = (2, OK | STOP | A.F_TERMINATES, IN_BASE + 56 + 2, 5, N, 0, 1, N, 12)
    recs[4] = (4, OK, 0, 0, N, 0, 0, N, 20)
    recs[5] = (N, 0, 0, 0, N, 0, 0, N, 0)
    tcs = np.zeros(2, TC_DT)
    tcs[0] = (0, A.TC_HAS_ID | A.TC_HAS_FUNC | A.TC_ID_TEXT | A.TC_NAME_TEXT, 1, 9, 2, 0, 0, 11, 3, 0, 0)
    tcs[1] = (1, A.TC_HAS_FUNC | A.TC_ARGS_TEXT, N, 0, 0, 0, 0, 0, 0, 14, 2)
    usages = np.array([(1, 2, 3)], USAGE_DT)
    runs = np.zeros(2, RUN_DT)
    runs[0] = (2, 1, 3, 1, N)
    runs[1] = (5, 1, 5, 1, N)
    segres = np.zeros(2, SEGRES_DT)
    segres[0] = (0, 2, 0, 3, 0, 0, A.SEG_TERMINATED, 200)
    segres[1] = (3, 2, 4, 1, N, 5, 0, 100)
    segs = np.zeros(2, SEG_DT)
    segs[0] = (0, 0, 200, R, 0, 0)
    segs[1] = (1, 208, 100, PP, 0, 0)
    return dict(frames=frames, recs=recs, tcs=tcs, usages=usages, runs=runs, segres=segres, segs=segs,
                engine_flags=0, max_line=32768)


def check(b: dict):
    keep = []

    def ptr(arr, ctype):
        a = np.ascontiguousarray(arr)
        keep.append(a)
        return C.cast(C.c_void_p(a.ctypes.data), C.POINTER(ctype))

    res = A.Result()
    res.status = 0
    res.n_segs = len(b["segres"])
    res.n_frames, res.n_recs, res.n_tcs = len(b["frames"]), len(b["recs"]), len(b["tcs"])
    res.n_usages, res.n_runs = len(b["usages"]), len(b["runs"])
    res.out_bytes, res.text_bytes, res.in_base = OUT_BYTES, TEXT_BYTES, IN_BASE
    res.frames, res.recs, res.tcs = ptr(b["frames"], A.Frame), ptr(b["recs"], A.Rec), ptr(b["tcs"], A.Tc)
    res.usages, res.runs, res.segs = ptr(b["usages"], A.Usage), ptr(b["runs"], A.Run), ptr(b["segres"], A.SegResult)
    return orc.check_result(res, b["segs"], b["engine_flags"], b["max_line"])


def test_well_formed_result_passes():
    assert check(well_formed()) == (0, "")


def _set(**kw):
    """Mutation: table.field[index] = value for every key 'table__field__index'."""
    def f(b):
        for k, v in kw.items():
            table, fld, idx = k.split("__")
            b[table][fld][int(idx)] = v
    return f


def _both(*fs):
    def f(b):
        for g in fs:
            g(b)
    return f


def _engine(flags=0, max_line=None):
    def f(b):
        b["engine_flags"] = flags
        if max_line is not None:
            b["max_line"] = max_line
    return f


def test_allowed_variants_pass():
    """What the rules allow: a deferred segment that took part of its input (SSE_FLAG_DEFER), DESIGN.md §5 deviation 3's
    LINE_TOO_LONG | DEAD on a segment that terminated, a record without a frame whose spans lie in its segment's input."""
    b = well_formed()
    _both(_engine(A.FLAG_DEFER), _set(segres__flags__1=A.SEG_DEFERRED, segres__consumed__1=40))(b)
    assert check(b) == (0, "")
    b = well_formed()
    _set(segres__flags__0=A.SEG_TERMINATED | A.SEG_LINE_TOO_LONG | A.SEG_DEAD)(b)
    assert check(b) == (0, "")
    b = well_formed()
    _set(recs__content_off__1=IN_BASE + 100)(b)
    assert check(b) == (0, "")


# (rule the checker must name first, mutation, violations it causes)
CASES = {
    # runs
    # (the terminating record of seg 0 is in runs[0]: cut off from it, SEG_TERMINATED has no record: term.seg too)
    "run.next": ("run.next", _set(segres__next__0=7), 2),
    "run.shared": ("run.shared", _set(segres__next__1=0), 1),
    "run.cycle": ("run.shared", _set(runs__next__0=0), 1),
    "run.frames": ("run.frames", _set(runs__frame_count__0=10), 2),
    "run.recs": ("run.recs", _set(runs__rec_first__0=100), 2),
    "frame.shared": ("frame.shared", _set(segres__next__1=1, runs__frame_first__1=4, runs__rec_count__1=0), 1),
    "rec.shared": ("rec.shared", _set(segres__next__1=1, runs__rec_first__1=4, runs__frame_count__1=0), 1),
    # frames
    "frame.out": ("frame.out", _set(frames__off__1=40), 1),
    "frame.in": ("frame.in", _set(frames__off__4=IN_BASE + 0), 1),             # identical bytes of another connection
    "frame.copy_out": ("frame.copy_out", _engine(A.FLAG_COPY_OUT), 4),
    # record links
    "link.range": ("link.range", _set(recs__frame__3=1), 2),                     # ... and frame 2 has no record
    "link.order": ("link.order", _set(recs__frame__0=1, recs__payload_len__0=32, recs__frame__2=0, recs__payload_len__2=22), 1),
    "link.done": ("link.done", _set(recs__frame__1=1, recs__payload_len__1=32, recs__content_off__1=10, recs__frame__2=N), 1),
    "link.unique": ("link.unique", _set(recs__frame__2=N), 1),
    "link.missing": ("link.missing", _set(recs__frame__4=N), 1),
    "rec.mode_p": ("rec.mode_p", _set(segs__mode__1=A.MODE_P), 1),
    # payload length against the frame
    "payload.len.R": ("payload.len", _set(recs__payload_len__0=23), 1),
    "payload.len.P": ("payload.len", _set(recs__payload_len__4=21), 1),
    # spans
    "span.text": ("span.text", _set(recs__content_off__0=14), 1),
    "span.tc_text": ("span.text", _set(tcs__args_off__1=15), 1),
    "span.frame": ("span.frame", _set(recs__content_off__3=IN_BASE + 52), 1),    # inside "data: ", not the payload
    "span.arena": ("span.arena", _set(recs__content_off__1=IN_BASE + 210), 1),   # another segment's input
    "span.content_text": ("span.content_text", _set(recs__content_len__2=0), 1),
    # sentinels
    "usage.flag": ("usage.flag", _set(recs__flags__0=OK | A.F_CONTENT_TEXT | A.F_TC_NONNIL), 1),
    "usage.range": ("usage.range", _set(recs__usage__0=1), 1),
    "usage.shared": ("usage.shared", _set(recs__usage__2=0, recs__flags__2=OK | A.F_CONTENT_TEXT | A.F_HAS_USAGE), 1),
    "tc.first": ("tc.first", _set(recs__tc_first__0=N), 1),
    "tc.short": ("tc.short", _set(recs__tc_count__0=3), 1),
    "tc.end": ("tc.end", _set(recs__tc_count__0=1), 1),
    "tc.range": ("tc.range", _set(tcs__next__0=5), 1),
    "tc.shared": ("tc.shared", _set(recs__tc_first__2=1, recs__tc_count__2=1), 1),
    "rec.not_ok": ("rec.not_ok", _set(recs__flags__1=DONE), 1),
    "rec.too_long": ("rec.too_long", _set(recs__flags__2=OK | A.F_CONTENT_TEXT | A.F_TOO_LONG), 1),
    "rec.depth": ("rec.depth", _set(recs__flags__2=OK | A.F_CONTENT_TEXT | A.F_DEPTH_LIMIT), 1),
    "rec.flags": ("rec.flags", _set(recs__flags__2=OK | A.F_CONTENT_TEXT | 0x400), 1),
    "rec.done_exact": ("rec.done_exact", _set(recs__flags__1=OK | DONE | A.F_DONE_EXACT), 1),
    # termination
    "term.flag.missing": ("term.flag", _set(recs__flags__3=OK | STOP), 2),       # ... and SEG_TERMINATED has no record
    "term.flag.mode_p": ("term.flag", _set(recs__flags__4=OK | A.F_TERMINATES), 3),   # ... and term.seg, term.carry
    "term.flag.done_line": ("term.flag", _set(recs__flags__1=OK | DONE | STOP | A.F_TERMINATES), 2),   # ... and term.count
    "term.count": ("term.count", _set(recs__flags__2=OK | A.F_CONTENT_TEXT | STOP | A.F_TERMINATES), 1),
    "term.last": ("term.last", _set(recs__flags__2=OK | A.F_CONTENT_TEXT | STOP | A.F_TERMINATES, recs__flags__3=OK), 1),
    "term.seg": ("term.seg", _set(segres__flags__0=0), 1),
    "term.carry": ("term.carry", _set(segres__carry_len__0=3), 1),
    "term.consumed": ("term.consumed", _both(_engine(A.FLAG_DEFER), _set(segres__consumed__0=150)), 1),
    # segments
    "seg.flags.unknown": ("seg.flags", _set(segres__flags__1=0x20), 1),
    "seg.flags.too_long": ("seg.flags", _set(segres__flags__1=A.SEG_LINE_TOO_LONG), 1),
    "seg.flags.dead_terminated": ("seg.flags", _set(segres__flags__0=A.SEG_TERMINATED | A.SEG_DEAD), 1),
    "seg.consumed": ("seg.consumed", _set(segres__consumed__1=99), 1),
    "seg.consumed.defer": ("seg.consumed", _both(_engine(A.FLAG_DEFER), _set(segres__consumed__1=101)), 1),
    "seg.deferred": ("seg.deferred", _set(segres__flags__1=A.SEG_DEFERRED), 1),
    "seg.finished": ("seg.finished", _set(segres__flags__1=A.SEG_FINISHED), 1),
    "seg.carry": ("seg.carry", _engine(0, max_line=4), 1),
}


@pytest.mark.parametrize("case", list(CASES))
def test_checker_names_the_broken_rule(case):
    rule, mutate, n_expected = CASES[case]
    b = well_formed()
    mutate(b)
    n, msg = check(b)
    assert msg.startswith(rule + ":"), (case, n, msg)
    assert n == n_expected, (case, n, msg)
