"""What a batch asks of each result arena, and the inputs that ask the most per byte.

sse_worst_case_config promises capacities under which no batch can overflow a result arena. This module builds, for each
arena, the input that uses the most of it per input byte (the extremal generators), states what such a batch asks of every
arena (demand: exact counts of frames, records, work items, runs and tool-call elements, upper bounds of out and text bytes),
and reads the capacity each arena gets from a config (bound). The CPU test compares demand with bound over a grid of batch
shapes; the GPU test runs every generator and checks the kernels' own counters against demand.

A load is one batch of one or more connections. A connection may hold an unterminated line from an earlier batch (`prefix`,
sent alone first): the batch under test completes it from the carry slot (or the line pool), so its payload is decoded
although its bytes are not in the batch. Every line a generator builds emits a frame (mode P) or a record (mode R lines that
hold "[DONE]"), so every round of lines takes a run."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from inference_gateway_b200 import _abi as A
from inference_gateway_b200.engine import make_line_pool
from tests import seams as S

PP = A.MODE_P | A.MODE_PARSE
R = A.MODE_R | A.MODE_PARSE
ARENAS = ("frames", "recs", "items", "runs", "tcs", "usages", "out", "text")
EXACT = ("frames", "recs", "items", "runs", "tcs", "usages")     # demand() counts these exactly; out and text are bounds
TILE_SLOT = S.TILE - 32       # the longest carry slot the tile kernel accepts (sse_fused_max_line)


def worst(conns: int, batch: int, pool=None, slot=None):
    """sse_worst_case_config for conns connections and batch bytes, with carry_slot_bytes = slot when given and grown by
    sse_line_pool_config for a line pool of make_line_pool(**pool) when given."""
    cfg = A.Config()
    A.load().sse_worst_case_config(C.byref(cfg), conns, batch)
    if slot is not None:
        cfg.carry_slot_bytes = slot
    if pool is not None:
        p = make_line_pool(**pool)
        A.load().sse_line_pool_config(C.byref(cfg), C.byref(p))
    return cfg


def r4(n: int) -> int:
    return (n + 3) & ~3


# ------------------------------------------------------------------ rounds of lines (the runs[] entries a segment takes)
def _nl(stream: np.ndarray, lo: int, hi: int):
    """(count, last position + 1 or lo) of the '\\n' bytes in stream[lo:hi]."""
    if hi <= lo:
        return 0, lo
    w = stream[lo:hi] == 10
    c = int(np.count_nonzero(w))
    return c, (lo + int(np.flatnonzero(w)[-1]) + 1) if c else lo


def split_runs_calls(carry: bytes, body: bytes, in_long: bool) -> int:
    """append_run calls of the produce kernel for one segment (seams.produce_windows, counting only): a round of up to LT_MAX
    lines per call, and one for a line completed from the carry slot."""
    stream = np.frombuffer(carry + body, dtype=np.uint8)
    n, c = len(body), len(carry)
    pend = 0 if in_long else c
    consumed = calls = 0
    while True:
        a = S.r16(pend)
        nload = min(n - consumed, S.BUF - a)
        s0 = c + consumed - pend
        consumed += nload
        s1 = c + consumed
        pos = s0
        if in_long:
            k, end = _nl(stream, s0, s1)
            if not k:
                pend = 0
                if consumed >= n:
                    return calls
                continue
            first = s0 + int(np.argmax(stream[s0:s1] == 10)) + 1
            calls += 1
            in_long = False
            pos = first
        k, end = _nl(stream, pos, s1)
        calls += -(-k // S.LT_MAX)
        tail = s1 - (end if k else pos)
        if consumed >= n:
            return calls
        if tail >= S.BUF - 32:
            in_long = True
            pend = 0
            continue
        pend = tail


def tile_runs_calls(carry: bytes, body: bytes) -> int:
    """Runs of the tile kernel for one segment alone in its tile or tiles (seams.tile_windows, counting only): a run per round
    of up to LCAP lines."""
    stream = np.frombuffer(carry + body, dtype=np.uint8)
    c, n = len(carry), len(body)
    if S.r16(c) + S.r16(n) <= S.TILE:
        return -(-_nl(stream, 0, c + n)[0] // S.LCAP)
    calls, src, cl, front = 0, 0, c, 0
    while True:
        aw = S.r16(cl)
        nbytes = min(n - src, S.TILE - aw)
        d0 = 0 if cl else c + src + front
        e = c + src + nbytes
        k, ts = _nl(stream, d0, e)
        calls += -(-k // S.LCAP)
        if src + nbytes >= n or not k:
            return calls
        x = ts - c
        src, front, cl = x & ~15, x & 15, 0


# ------------------------------------------------------------------ loads
@dataclass
class Conn:
    mode: int
    body: bytes                 # the bytes of the batch under test
    prefix: bytes = b""         # an unterminated line start sent in an earlier batch (held in the carry slot or line pool)


@dataclass
class Load:
    name: str
    arena: str                  # the arena the load is extremal for
    conns: list
    # by construction: frames, records, work items (records not of a bare `data: [DONE]`); usages and tool-call elements per
    # engine kind; text bytes (an upper bound)
    frames: int = 0
    recs: int = 0
    items: int = 0
    usages: dict = field(default_factory=dict)   # {"split": n, "tile": n}: sse_usage slots the decoders allocate
    tcs: dict = field(default_factory=dict)   # {"split": n, "tile": n}: elements the decoders allocate
    text: int = 0
    split_only: bool = False    # needs the line pool, which the tile kernel does not have

    def in_bytes(self) -> int:
        return sum(S.r16(len(c.body)) for c in self.conns)


def _each(n: int, per: int) -> list:
    """n connections' shares of a budget of per bytes each (16-byte multiples)."""
    return [per & ~15] * n


def _lines(line: bytes, budget: int) -> int:
    return max(0, budget // len(line))


TC_HEAD = b'data: {"choices":[{"delta":{"tool_calls":['
TC_TAIL = b']}}]}\n'


def _tc_line(elem: bytes, k: int) -> bytes:
    """A chunk whose choices[0].delta.tool_calls holds k copies of elem."""
    return TC_HEAD + b",".join([elem] * k) + TC_TAIL


def _fit(make, per_elem: int, length: int):
    """The largest k with len(make(k)) <= length; returns (line, k)."""
    k = max(1, (length - len(make(0))) // per_elem)
    while k > 1 and len(make(k)) > length:
        k -= 1
    return make(k), k


# tool-call elements: bytes per element and elements allocated per line of k elements, by engine kind. The split decoder
# allocates an element when it ends and the tile decoder when it begins; neither allocates once the line has a type error
# (the first number in [1,...] sets it when it ends, after the tile decoder already took the first element).
TC_KINDS = {
    "numbers": (b"1", lambda k: {"split": 0, "tile": 1}),
    "objects": (b"{}", lambda k: {"split": k, "tile": k}),
    "nulls": (b"null", lambda k: {"split": k, "tile": k}),
}
LEGACY_TCS = {"numbers": lambda k: {"split": k, "tile": k}}     # before a type error stopped the allocations


def tc_line(kind: str, length: int):
    """(line of at most length bytes, elements) for a tool-call kind, or the repeated-key lines."""
    if kind == "repeat_tool_calls":
        one = b'"tool_calls":[{}]'
        return _fit(lambda k: b'data: {"choices":[{"delta":{' + b",".join([one] * max(k, 1)) + b'}}]}\n', len(one) + 1, length)
    if kind == "repeat_choices":
        one = b'"choices":[{"delta":{"tool_calls":[{}]}}]'
        return _fit(lambda k: b"data: {" + b",".join([one] * max(k, 1)) + b"}\n", len(one) + 1, length)
    elem = TC_KINDS[kind][0]
    return _fit(lambda k: _tc_line(elem, max(k, 1)), len(elem) + 1, length)


def tc_alloc(kind: str, k: int, legacy: bool = False) -> dict:
    """Elements each engine kind allocates for one line of k elements of a tool-call kind."""
    if kind.startswith("repeat"):
        return {"split": k, "tile": k}
    if legacy and kind in LEGACY_TCS:
        return LEGACY_TCS[kind](k)
    return TC_KINDS[kind][1](k)


def usage_reset_line(length: int):
    """(line of at most length bytes, k): a chunk with k pairs "usage":{},"usage":null and a last "usage":{} (JSON_OK, with a
    usage). Each decoder stores one sse_usage for it; the tile decoder once took a new one for every object after a null."""
    pair = b'"usage":{},"usage":null,'
    return _fit(lambda k: b"data: {" + pair * k + b'"usage":{}}\n', len(pair), length)


def text_line(kind: str, length: int):
    """(line, decoded strings' text bytes, tool-call elements) of a line of at most length bytes whose strings all need the
    text arena: content or arguments of invalid bytes (each becomes U+FFFD, 3 bytes), or ids of one invalid byte each (a 4-byte
    aligned allocation per 13 payload bytes)."""
    if kind == "content":
        head, tail = b'data: {"choices":[{"delta":{"content":"', b'"}}]}\n'
        m = length - len(head) - len(tail)
        return head + b"\xff" * m + tail, r4(3 * m), 0
    if kind == "args":
        head, tail = b'data: {"choices":[{"delta":{"tool_calls":[{"function":{"arguments":"', b'"}}]}}]}\n'
        m = length - len(head) - len(tail)
        return head + b"\xff" * m + tail, r4(3 * m), 1
    line, k = _fit(lambda k: _tc_line(b'{"id":"\xff"}', max(k, 1)), 13, length)
    return line, 4 * k, k


def _load_of_lines(name, arena, mode, line, budget, n_conns, carried: int, *, frames_per=1, recs_per=1, items_per=1,
                   usages_per=0, tcs_per=None, text_per=0, split_only=False) -> Load:
    """n_conns connections, each with as many copies of line as its share of budget holds; the first `carried` of them also
    complete a copy of line held from an earlier batch (all of it but its last byte, the '\\n')."""
    conns, n = [], 0
    for i, per in enumerate(_each(n_conns, budget // n_conns)):
        head = line[-1:] if i < carried else b""
        k = _lines(line, per - len(head))
        conns.append(Conn(mode, head + line * k, line[:-1] if i < carried else b""))
        n += k + (1 if i < carried else 0)
    tcs = {e: v * n for e, v in (tcs_per or {"split": 0, "tile": 0}).items()}
    if not isinstance(usages_per, dict):
        usages_per = {"split": usages_per, "tile": usages_per}
    usages = {e: v * n for e, v in usages_per.items()}
    return Load(name, arena, conns, frames=frames_per * n, recs=recs_per * n, items=items_per * n, usages=usages,
                tcs=tcs, text=text_per * n, split_only=split_only)


def generators(budget: int, n_conns: int, line_max: int, legacy: bool = False) -> list:
    """Every extremal load for a batch of `budget` input bytes on up to n_conns connections whose longest line is line_max
    bytes ('\\n' included). The carried loads use every connection. legacy: the counts of the decoders before a line with a
    type error stopped allocating tool-call elements and before the tile decoder kept one sse_usage slot per line."""
    out = []
    nl = b"\n"
    # frames and runs: one frame per byte, one round per 64 one-byte lines
    out.append(Load("frames.blank_flood", "frames", [Conn(A.MODE_P, nl * (budget & ~15))], frames=budget & ~15))
    half = (budget // 2) & ~15
    out.append(Load("runs.x_lines", "runs", [Conn(A.MODE_P, b"x\n" * (half // 2))], frames=half // 2))
    # runs: a 17-byte tail carried across every window keeps 8,143 lines in each window of 8,160 new bytes: 128 rounds, half a
    # round more than 64 one-byte lines per round would take
    k = max(0, (budget - 8192) // 8160)
    body = nl * 8175 + b"x" * 17 + (nl * 8143 + b"x" * 17) * k
    out.append(Load("runs.partial_rounds", "runs", [Conn(A.MODE_P, body)], frames=8175 + 8143 * k))
    # records and work items: 7-byte lines
    done = b"[DONE]\n"
    n = budget // 7
    out.append(Load("recs.done_lines", "recs", [Conn(R, done * n)], recs=n, items=n))
    out.append(Load("recs.empty_data", "recs", [Conn(PP, b"data: \n" * n)], frames=n, recs=n, items=n))
    u = b'data: {"usage":{}}\n'
    out.append(_load_of_lines("usages.usage_lines", "usages", PP, u, budget, 1, 0, usages_per=1))
    # usages: "usage" objects reopened after null in one line, in the batch and completed from every carry slot
    line, k = usage_reset_line(line_max)
    per = {"split": 1, "tile": k + 1 if legacy else 1}
    out.append(_load_of_lines("usages.reset", "usages", PP, line, budget, 1, 0, usages_per=per))
    out.append(_load_of_lines("usages.reset.carried", "usages", PP, line, budget, n_conns, n_conns, usages_per=per))
    # out bytes: "data: x" reframed to "data: x\n\n" (9 bytes per 8), and a line of the whole slot completing on every connection
    out.append(_load_of_lines("out.reframe", "out", R, b"data: x\n", budget, 1, 0))
    big = b"data: " + b"x" * (line_max - 7) + nl
    out.append(_load_of_lines("out.carried", "out", R, big, budget, n_conns, n_conns))
    # tool-call elements and text, in the batch and completed from every carry slot
    for kind in ("numbers", "objects", "nulls", "repeat_tool_calls", "repeat_choices"):
        line, k = tc_line(kind, line_max)
        per = tc_alloc(kind, k, legacy)
        out.append(_load_of_lines(f"tcs.{kind}", "tcs", PP, line, budget, 1, 0, tcs_per=per))
        out.append(_load_of_lines(f"tcs.{kind}.carried", "tcs", PP, line, budget, n_conns, n_conns, tcs_per=per))
    for kind in ("content", "args", "ids"):
        line, text, k = text_line(kind, line_max)
        per = {"split": k, "tile": k}
        out.append(_load_of_lines(f"text.{kind}", "text", PP, line, budget, 1, 0, tcs_per=per, text_per=text))
        out.append(_load_of_lines(f"text.{kind}.carried", "text", PP, line, budget, n_conns, n_conns, tcs_per=per,
                                  text_per=text))
    return out


def pooled(budget: int, n_conns: int, pool_bytes: int, page_bytes: int, legacy: bool = False) -> list:
    """Lines assembled in the line pool: every connection completes a pooled line of its share of the pool's bytes (whole
    pages), next to in-batch lines of the same kind filling the batch."""
    out = []
    share = (pool_bytes // n_conns) // page_bytes * page_bytes
    if share == 0:
        return out
    for kind in ("numbers", "objects"):
        line, k = tc_line(kind, share)
        small, ks = tc_line(kind, 4096)
        per, sper = tc_alloc(kind, k, legacy), tc_alloc(kind, ks, legacy)
        conns, n_small = [], 0
        for _ in range(n_conns):
            j = _lines(small, (budget // n_conns & ~15) - 1)
            conns.append(Conn(PP, line[-1:] + small * j, line[:-1]))
            n_small += j
        out.append(Load(f"pool.{kind}", "tcs", conns, frames=n_conns + n_small, recs=n_conns + n_small,
                        items=n_conns + n_small, tcs={e: per[e] * n_conns + sper[e] * n_small for e in per}, split_only=True))
    return out


# ------------------------------------------------------------------ demand and bound
def demand(load: Load, engine: str) -> dict:
    """What the batch of `load` asks of every arena on an engine kind ("split": the produce and decode kernels, "tile": the
    single-pass tile kernel): exact frames, records, work items (split only; the tile kernel has none), runs, tool-call
    elements and usages; upper bounds of out bytes and text bytes."""
    runs = out = 0
    for c in load.conns:
        carried = len(c.prefix)
        if engine == "split":
            # a prefix longer than a window went on in the carry slot (it was sent alone, as one segment)
            calls = split_runs_calls(c.prefix, c.body, carried > S.BUF)
        else:
            calls = tile_runs_calls(c.prefix, c.body)
        runs += max(0, calls - 1)
        # every line materialised (mode R: one more '\n' per line), each round's bytes 16-byte aligned, a carried line whole
        out += len(c.body) + (c.body.count(b"\n") if c.mode & A.MODE_R else 0) + 15 * calls + (carried + 2 + 15 if carried else 0)
    return dict(frames=load.frames, recs=load.recs, items=load.items if engine == "split" else 0, runs=runs,
                tcs=load.tcs.get(engine, 0), usages=load.usages.get(engine, 0), out=out, text=load.text)


def bound(cfg) -> dict:
    """The capacity sse_config cfg gives each arena (work items share max_recs)."""
    return dict(frames=cfg.max_frames, recs=cfg.max_recs, items=cfg.max_recs, runs=cfg.max_runs, tcs=cfg.max_tcs,
                usages=cfg.max_usages, out=cfg.out_arena_bytes, text=cfg.text_arena_bytes)


OVF_BIT = dict(frames=A.OVF_OUT, recs=A.OVF_OUT, items=A.OVF_OUT, out=A.OVF_OUT, runs=A.OVF_RUNS, tcs=A.OVF_TCS,
               usages=A.OVF_USAGES, text=A.OVF_TEXT)
