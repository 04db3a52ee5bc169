"""Streams that stress the agent and telemetry folds (csrc/sse_fold.cpp), and an sse_result builder that lays out the oracle's
records of a stream the way the kernels do. Shared by the CPU and GPU fold tests."""
import ctypes as C

import numpy as np

from inference_gateway_b200 import _abi as A
from oracle import orc
from tests.corpus import STRING_FIELDS, TRICKY, adversarial_bodies, string_alignment_docs, template_near_misses

DONE = b"data: [DONE]\n\n"
HEAD = b'data: {"choices":[{"index":0,"delta":{"content":"before "},"finish_reason":null}]}\n\n'
TAIL = (b'data: {"choices":[{"index":0,"delta":{"content":"after","tool_calls":[{"index":0,"id":"t","function":{"name":"tail",'
        b'"arguments":"{}"}}]},"finish_reason":null}]}\n\n')
USAGE = b'data: {"choices":[],"usage":{"prompt_tokens":3,"completion_tokens":4,"total_tokens":7}}\n\n'
STOP = b'data: {"choices":[{"index":0,"delta":{},"finish_reason":"tool_calls"}]}\n\n'


def stream_of(docs, sep=b"\n\n") -> bytes:
    return b"".join(b"data: " + d.replace(b"\n", b" ") + sep for d in docs) + DONE


def tricky_streams() -> list:
    """Every TRICKY document as a stream, between a content chunk and a chunk with content and a tool call: a document that
    terminates the agent where the reference does not, or the reverse, changes what the agent keeps."""
    return [HEAD + b"data: " + d.replace(b"\n", b" ") + b"\n\n" + TAIL + USAGE + DONE for d in TRICKY]


def tool_call_string_streams(per=24, step=1) -> list:
    """The string-alignment documents whose string is a tool call's id, name, arguments or thought signature, `per` to a
    stream (every `step`-th document)."""
    heads = [t[:t.index(b"%s")] for f, t in STRING_FIELDS.items() if f in ("id", "name", "arguments", "thought_signature")]
    docs = [d for d in string_alignment_docs() if any(d.startswith(h) for h in heads)][::step]
    return [stream_of(docs[i:i + per]) for i in range(0, len(docs), per)]


def near_miss_streams(per=30, step=1) -> list:
    canon, miss = template_near_misses()
    docs = (canon + miss)[::step]
    return [stream_of(docs[i:i + per]) for i in range(0, len(docs), per)]


def element(index, id=None, name=None, args=None, type=None) -> bytes:
    """One element of delta.tool_calls (index given as written: an int or the literal bytes)."""
    parts = [b'"index":%s' % (index if isinstance(index, bytes) else str(index).encode())]
    if id is not None:
        parts.append(b'"id":"%s"' % id)
    if type is not None:
        parts.append(b'"type":"%s"' % type)
    if name is not None or args is not None:
        fn = ([b'"name":"%s"' % name] if name is not None else []) + ([b'"arguments":"%s"' % args] if args is not None else [])
        parts.append(b'"function":{%s}' % b",".join(fn))
    return b"{" + b",".join(parts) + b"}"


def tc_chunk(elements, content=None, finish=None) -> bytes:
    delta = b'"tool_calls":[%s]' % b",".join(elements)
    if content is not None:
        delta = b'"content":"%s",' % content + delta
    fin = b'"%s"' % finish if finish else b"null"
    return b'data: {"choices":[{"index":0,"delta":{%s},"finish_reason":%s}]}\n\n' % (delta, fin)


def merge_streams() -> list:
    """Streams built for parseStreamingToolCalls' merge (agent.go:377-481) and telemetry's (telemetry.go:240-274)."""
    e = element
    out = [
        # one index again and again, in separate chunks and twice in one chunk (each element with a function appends the
        # arguments of every element of its index)
        b"".join(tc_chunk([e(0, id=b"c%d" % k, name=b"f", args=b"a%d" % k)]) for k in range(5))
        + tc_chunk([e(0, args=b"x"), e(0, name=b"g", args=b"y"), e(1, id=b"one", name=b"h")]) + STOP + USAGE + DONE,
        # negative, gapped and int64-extreme indices; an index past int64 makes its line a type error
        tc_chunk([e(-1, id=b"neg", name=b"n"), e(0, id=b"zero", name=b"z"), e(2, id=b"two", name=b"t")])
        + tc_chunk([e(5, id=b"five", name=b"f")]) + tc_chunk([e(b"9223372036854775807", id=b"max", name=b"m")])
        + tc_chunk([e(b"-9223372036854775808", id=b"min", name=b"m")]) + tc_chunk([e(b"9223372036854775808", id=b"over")])
        + tc_chunk([e(1, id=b"one", name=b"o", args=b"{}")]) + STOP + DONE,
        # more than 64 merged calls: 100 in one chunk, then 90 more over separate chunks
        tc_chunk([e(k, id=b"id%d" % k, name=b"n%d" % k, args=b"a%d" % k) for k in range(100)])
        + b"".join(tc_chunk([e(100 + k, id=b"late%d" % k, name=b"m%d" % k)]) for k in range(90)) + USAGE + STOP + DONE,
        # tool calls on lines that contain [DONE]: swallowed by the reframe, still parsed for tool calls
        tc_chunk([e(0, id=b"a", name=b"first", args=b"{")], content=b"[DONE]") + tc_chunk([e(0, args=b"}")], content=b"x [DONE] y")
        + tc_chunk([e(1, id=b"b", name=b"second")]) + STOP,
    ]
    # bare [DONE] and data: [DONE] with whitespace around them: only the line that trims to "data: [DONE]" stops the merge
    for done in (b"[DONE]\n\n", b"  [DONE]  \n\n", b"\t[DONE]\r\n\r\n", b"data: [DONE]\n\n", b"  data: [DONE] \n\n",
                 b"data: [DONE]\r\n", b"data:  [DONE]\n\n", b"data: [DONE]x\n\n"):
        out.append(tc_chunk([e(0, id=b"a", name=b"first", args=b"{")]) + done + tc_chunk([e(0, args=b"}"), e(1, id=b"b", name=b"s")])
                   + USAGE + STOP)
    return out


def saturated_line(n: int) -> bytes:
    """One chunk with n tool-call elements: n - 4 of {} (index 0), then 4 with indices 1-4 and their own id, name and
    arguments. tc_count saturates at 65,535: from n = 65,536 the last elements lie past it."""
    tail = [element(k - n + 5, id=b"id%d" % k, name=b"n%d" % k, args=b"a%d" % k, type=b"function") for k in range(n - 4, n)]
    return tc_chunk([b"{}"] * (n - 4) + tail)


SATURATED = (65534, 65535, 65536, 65537)


def saturated_streams() -> list:
    return [HEAD + saturated_line(n) + USAGE + STOP + DONE for n in SATURATED]


def corpus(seed=0, n_adv=48, small=False) -> dict:
    """Every family of the fold corpus but the saturated lines: {family: [bodies]}. small: a sample of the two large
    families."""
    return dict(adversarial=adversarial_bodies(np.random.default_rng(seed), n_adv), tricky=tricky_streams(),
                tc_strings=tool_call_string_streams(step=7 if small else 1), near_misses=near_miss_streams(step=5 if small else 1),
                merge=merge_streams())


# ------------------------------------------------------------------ batch results laid out as the kernels do
IN_BASE = 1 << 26


class Layout:
    """The records of one stream (an oracle view) over n_results sse_results, the way the kernels lay them out:
    - a result holds the lines between two seeded cuts; its lines go in runs of 1 to run_lines (at most 64) lines, chained
      through runs[], with a decoy frame and a decoy record (flagged SSE_F_DEPTH_LIMIT) between two runs and a decoy segment
      before the stream's own: a fold that leaves its runs meets them;
    - frames lie in the out arena or, zero-copy, in the input arena at or above in_base, chosen per frame;
    - strings lie in the text arena (flagged *_TEXT), the out arena or the input arena, in turn;
    - a line past the nesting limit gets SSE_F_DEPTH_LIMIT and no decoded fields, as the kernels give it.
    results[k] is (sse_result, segment index); undecoded[k]: result k holds such a record."""

    def __init__(self, view: orc.StreamView, mode_r: bool, n_results=1, run_lines=64, seed=0):
        rng = np.random.default_rng(seed)
        lines = [l for l in view.lines if l.kind != orc.L_UNREAD]
        cuts = np.sort(rng.integers(0, len(lines) + 1, size=n_results - 1)) if n_results > 1 else []
        bounds = [0, *map(int, cuts), len(lines)]
        self.keep, self.results, self.undecoded = [], [], []
        self.turn = 0
        for k in range(n_results):
            self._result(lines[bounds[k]:bounds[k + 1]], mode_r, run_lines, rng)

    def _arr(self, cls, rows):
        a = (cls * max(1, len(rows)))()
        for i, r in enumerate(rows):
            a[i] = cls(*r)
        self.keep.append(a)
        return C.cast(a, C.POINTER(cls))

    def _bytes(self, b: bytearray):
        a = (C.c_uint8 * max(1, len(b))).from_buffer_copy(bytes(b) or b"\0")
        self.keep.append(a)
        return C.cast(a, C.POINTER(C.c_uint8))

    def _result(self, lines, mode_r, run_lines, rng):
        out, inn, text = bytearray(b"\0" * 16), bytearray(b"\0" * 16), bytearray(b"\0")
        frames, recs, tcs, usages, runs = [], [], [], [], []

        def put(b: bytes):
            """(offset, length, in the text arena) of a string, placed in the next arena of the rotation."""
            if not b:
                return 0, 0, False
            self.turn += 1
            where = self.turn % 3
            if where == 0:
                o = len(text); text.extend(b); return o, len(b), True
            if where == 1:
                o = len(out); out.extend(b); return o, len(b), False
            o = len(inn); inn.extend(b); return IN_BASE + o, len(b), False

        def decoy():
            frames.append((len(out), 3)); out.extend(b"x\n\n")
            recs.append((len(frames) - 1, A.F_DEPTH_LIMIT, 0, 0, A.NONE, 0, 0, A.NONE, 1))

        decoy()
        seg0 = A.Run(0, 1, 0, 1, A.NONE)
        undecoded = False
        i, first = 0, None
        while i < len(lines) or first is None:
            if first is not None:
                decoy()
            n = int(rng.integers(1, run_lines + 1))
            f0, r0 = len(frames), len(recs)
            for l in lines[i:i + n]:
                undecoded |= self._line(l, mode_r, frames, recs, tcs, usages, out, inn, put, rng)
            i += n
            run = [f0, len(frames) - f0, r0, len(recs) - r0, A.NONE]
            if first is None:
                first = run
            else:
                (first if not runs else runs[-1])[4] = len(runs)
                runs.append(run)
        res = A.Result()
        res.status, res.n_segs = 0, 2
        res.n_frames, res.n_recs, res.n_tcs, res.n_usages, res.n_runs = len(frames), len(recs), len(tcs), len(usages), len(runs)
        res.out_bytes, res.text_bytes = len(out), len(text)
        res.out, res.in_, res.text, res.in_base = self._bytes(out), self._bytes(inn), self._bytes(text), IN_BASE
        res.frames, res.recs, res.tcs = self._arr(A.Frame, frames), self._arr(A.Rec, recs), self._arr(A.Tc, tcs)
        res.usages, res.runs = self._arr(A.Usage, usages), self._arr(A.Run, runs)
        segs = (A.SegResult * 2)()
        segs[0].run = seg0
        segs[1].run = A.Run(*first)
        self.keep.append(segs)
        res.segs = C.cast(segs, C.POINTER(A.SegResult))
        self.keep.append(res)
        self.results.append((res, 1))
        self.undecoded.append(undecoded)

    def _line(self, l, mode_r, frames, recs, tcs, usages, out, inn, put, rng) -> bool:
        fidx = A.NONE
        if l.kind == orc.L_EMITTED:
            fidx = len(frames)
            if rng.random() < 0.5:
                frames.append((len(out), len(l.out))); out.extend(l.out)
            else:
                frames.append((IN_BASE + len(inn), len(l.out))); inn.extend(l.out)
        if l.kind == orc.L_DONE_EXACT:
            recs.append((A.NONE, A.F_DONE_LINE | A.F_DONE_EXACT, 0, 0, A.NONE, 0, 0, A.NONE, 6))
            return False
        ck = l.chunk
        if ck is None:
            return False
        fl = A.F_DONE_LINE if l.kind == orc.L_DONE else 0
        if l.depth_limited:
            recs.append((fidx, fl | A.F_DEPTH_LIMIT, 0, 0, A.NONE, 0, 0, A.NONE, l.payload_len))
            return True
        co = cl = 0
        tcf, tcc, nch, ui = A.NONE, 0, 0, A.NONE
        if ck.json_ok:
            fl |= A.F_JSON_OK
            nch = min(ck.n_choices, 0xFFFF)
            if ck.usage is not None:
                fl |= A.F_HAS_USAGE; ui = len(usages); usages.append(ck.usage)
            if nch > 0:
                fl |= ck.finish << A.F_FINISH_SHIFT
                co, cl, t = put(ck.content)
                fl |= A.F_CONTENT_TEXT if t else 0
                fl |= (A.F_TC_NONNIL if ck.tool_calls_nonnil else 0) | (A.F_TC_VALID if ck.has_valid_tool_call else 0)
                if mode_r and fidx != A.NONE and ck.finish in (orc.FIN_STOP, orc.FIN_TOOL_CALLS):
                    fl |= A.F_TERMINATES
                tcc = min(len(ck.tool_calls), 0xFFFF)
                for k, tc in enumerate(ck.tool_calls):
                    tf = (A.TC_HAS_ID if tc.id is not None else 0) | (A.TC_HAS_TYPE if tc.type is not None else 0)
                    tf |= A.TC_HAS_FUNC if tc.function else 0
                    spans = []
                    for bit, s in zip((A.TC_ID_TEXT, A.TC_TYPE_TEXT, A.TC_NAME_TEXT, A.TC_ARGS_TEXT),
                                      (tc.id or b"", tc.type or b"", tc.name, tc.args)):
                        o, n, t = put(s)
                        tf |= bit if t else 0
                        spans += [o, n]
                    if k == 0:
                        tcf = len(tcs)
                    else:
                        tcs[-1][2] = len(tcs)
                    tcs.append([tc.index, tf, A.NONE, *spans])
        recs.append((fidx, fl, co, cl, tcf, tcc, nch, ui, l.payload_len))
        return False


def feed(L, layout: Layout, mode_r: bool):
    """Both folds fed every result of a layout. Returns (agent fold, telemetry fold, [(agent rc, telemetry rc) per result])."""
    ag, te = L.sse_agent_new(), L.sse_telemetry_new()
    rcs = [(L.sse_agent_feed(ag, C.byref(r), s), L.sse_telemetry_feed(te, C.byref(r), s)) for r, s in layout.results]
    return ag, te, rcs
