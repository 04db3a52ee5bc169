"""Shared parity harness: drives streams through the GPU path in randomly cut micro-batches and compares
every frame and every side-band record with the CPU oracle (oracle/ is the checker, never the product)."""
from __future__ import annotations

import ctypes as C
import os
from unittest import mock

import numpy as np

from inference_gateway_b200 import _abi as A
from oracle import orc


class ConnOut:
    def __init__(self):
        self.frames = []       # emitted frames (bytes) in order
        self.recs = []         # decoded records (dicts) in order
        self.terminated = False
        self.carry_len = 0
        self.flags = 0
        self.agent = None
        self.tele = None


def rec_to_dict(res, ri: int) -> dict:
    r = res.recs[ri]
    fl = int(r["flags"])
    d = dict(flags=fl, json_ok=bool(fl & A.F_JSON_OK), done=bool(fl & A.F_DONE_LINE),
             done_exact=bool(fl & A.F_DONE_EXACT), terminates=bool(fl & A.F_TERMINATES),
             depth_limit=bool(fl & A.F_DEPTH_LIMIT), too_long=bool(fl & A.F_TOO_LONG), frame=int(r["frame"]), payload_len=int(r["payload_len"]))
    if d["json_ok"]:
        d["n_choices"] = int(r["n_choices"])
        d["finish"] = (fl & A.F_FINISH_MASK) >> A.F_FINISH_SHIFT
        d["usage"] = None
        if fl & A.F_HAS_USAGE:
            u = res.usages[int(r["usage"])]
            d["usage"] = (int(u["prompt"]), int(u["completion"]), int(u["total"]))
        d["content"] = res.span(int(r["content_off"]), int(r["content_len"]), bool(fl & A.F_CONTENT_TEXT))
        d["tc_nonnil"] = bool(fl & A.F_TC_NONNIL)
        d["tc_valid"] = bool(fl & A.F_TC_VALID)
        tcs = []
        t = int(r["tc_first"])
        for _ in range(int(r["tc_count"])):
            assert t != A.NONE, "tool-call chain shorter than tc_count"
            tc = res.tcs[t]
            tf = int(tc["flags"])
            tcs.append(dict(
                index=int(tc["index"]),
                id=res.span(int(tc["id_off"]), int(tc["id_len"]), bool(tf & A.TC_ID_TEXT)) if tf & A.TC_HAS_ID else None,
                type=res.span(int(tc["type_off"]), int(tc["type_len"]), bool(tf & A.TC_TYPE_TEXT)) if tf & A.TC_HAS_TYPE else None,
                function=bool(tf & A.TC_HAS_FUNC),
                name=res.span(int(tc["name_off"]), int(tc["name_len"]), bool(tf & A.TC_NAME_TEXT)),
                args=res.span(int(tc["args_off"]), int(tc["args_len"]), bool(tf & A.TC_ARGS_TEXT))))
            t = int(tc["next"])
        d["tcs"] = tcs
    return d


def chunk_to_dict(ck: orc.ChunkView) -> dict:
    d = dict(json_ok=ck.json_ok)
    if ck.json_ok:
        d.update(n_choices=min(ck.n_choices, 0xFFFF), finish=ck.finish, usage=ck.usage, content=ck.content,
                 tc_nonnil=ck.tool_calls_nonnil, tc_valid=ck.has_valid_tool_call,
                 tcs=[dict(index=t.index, id=t.id, type=t.type, function=t.function, name=t.name, args=t.args)
                      for t in ck.tool_calls])
    return d


def fold_segment(o: ConnOut, res, i: int):
    """Appends segment i of a batch result to its connection's output. A record's frame link becomes the ordinal of the linked
    frame among the connection's frames (A.NONE: no frame; -1: a frame outside the record's own run)."""
    for ff, fc, rf, rc in res.seg_runs(i):
        base = len(o.frames)
        o.frames.extend(res.at(int(f["off"]), int(f["len"])) for f in res.frames[ff:ff + fc])
        for ri in range(rf, rf + rc):
            d = rec_to_dict(res, ri)
            if d["frame"] != A.NONE:
                d["frame"] = base + d["frame"] - ff if 0 <= d["frame"] - ff < fc else -1
            o.recs.append(d)
    sr = res.segs[i]
    o.carry_len = int(sr["carry_len"])
    o.flags |= int(sr["flags"])
    if int(sr["flags"]) & A.SEG_TERMINATED:
        o.terminated = True


# ------------------------------------------------------------------ structural check of every batch result
CHECKED = [0]     # batch results orc_check_result has passed in this process


def line_limit(eng) -> int:
    """The longest line one connection of the engine may hold: the line pool's max_line_bytes, else the carry slot."""
    return int(eng.pool.max_line_bytes) if eng.pool is not None and eng.pool.pool_pages else int(eng.cfg.carry_slot_bytes)


def check_result(eng, res, segs):
    """orc_check_result on one batch result: runs, frame / record ranges, links, chains, spans, flags (oracle/orc_check.c).
    segs: the sse_seg descriptors the batch was submitted with."""
    n, msg = orc.check_result(res.raw, segs[:int(res.raw.n_segs)], int(eng.cfg.flags), line_limit(eng))
    assert n == 0, f"batch result breaks {n} structural rule(s); first: {msg}"
    CHECKED[0] += 1


def process_checked(eng, items):
    """SseEngine.process (acquire, fill, submit, collect) with the structural check of the result. Returns (slot, result); the
    caller releases the slot."""
    slot, arena, segs = eng.acquire()
    try:
        n, nbytes = eng.fill(arena, segs, items)
        eng.submit(slot, n, nbytes)
        res = eng.collect(slot)
        check_result(eng, res, segs[:n].copy())
    except BaseException:
        eng.release(slot)
        raise
    return slot, res


def process_all_checked(eng, items, on_batch=None) -> int:
    """SseEngine.process_all with every batch it submits checked by process_checked."""
    with mock.patch.object(eng, "process", lambda batch: process_checked(eng, batch)):
        return eng.process_all(items, on_batch)


def run_streams(engine, streams, modes, n_batches=1, seed=0, with_folds=False):
    """streams: list of bytes (one upstream body per connection); modes: list of mode bits.
    Feeds every stream in n_batches randomly cut pieces (simulated TCP segmentation), one micro-batch per
    piece index. Returns list[ConnOut]."""
    from inference_gateway_b200.synth import random_cuts
    rng = np.random.default_rng(seed)
    L = engine.L
    n = len(streams)
    outs = [ConnOut() for _ in range(n)]
    engine.reset_all()
    pieces = [random_cuts(rng, s, n_batches) for s in streams]
    if with_folds:
        for o in outs:
            o.agent = L.sse_agent_new()
            o.tele = L.sse_telemetry_new()
    rounds = max(len(p) for p in pieces) if pieces else 0
    for b in range(rounds):
        items, who = [], []
        for c in range(n):
            if b < len(pieces[c]):
                items.append((c, modes[c], pieces[c][b]))
                who.append(c)
        if not items:
            continue
        slot, res = process_checked(engine, items)
        try:
            for i, c in enumerate(who):
                o = outs[c]
                fold_segment(o, res, i)
                if with_folds:
                    A.check(L.sse_agent_feed(o.agent, C.byref(res.raw), i), "sse_agent_feed")
                    A.check(L.sse_telemetry_feed(o.tele, C.byref(res.raw), i), "sse_telemetry_feed")
        finally:
            engine.release(slot)
    return outs


def run_pieces(eng, pieces, modes):
    """Like run_streams, with the pieces of every connection given: pieces[c][b] goes to connection c in batch b (empty pieces
    are submitted as empty segments). Returns list[ConnOut]."""
    outs = [ConnOut() for _ in pieces]
    eng.reset_all()
    for b in range(max(map(len, pieces))):
        who = [c for c in range(len(pieces)) if b < len(pieces[c])]
        slot, res = process_checked(eng, [(c, modes[c], pieces[c][b]) for c in who])
        try:
            for i, c in enumerate(who):
                fold_segment(outs[c], res, i)
        finally:
            eng.release(slot)
    return outs


# ------------------------------------------------------------------ digest parity at scale
def cut_bounds(bodies, n_batches: int, seed: int) -> np.ndarray:
    """Seeded random cut positions: row i holds the n_batches + 1 piece boundaries of bodies[i] (empty pieces included)."""
    n = len(bodies)
    rng = np.random.default_rng(seed)
    lens = np.fromiter((len(b) for b in bodies), dtype=np.int64, count=n)
    cuts = np.sort((rng.random((n, n_batches - 1)) * (lens[:, None] + 1)).astype(np.int64), axis=1) if n_batches > 1 else np.zeros((n, 0), np.int64)
    return np.concatenate([np.zeros((n, 1), np.int64), np.minimum(cuts, lens[:, None]), lens[:, None]], axis=1)


def digest_run(eng, bodies, modes, bounds, providers=None, on_batch=None):
    """Feeds body i in the pieces bounds[i] gives (one micro-batch per piece index, every connection in every batch, empty
    pieces included) and folds every batch result into per-connection digests. modes: one mode for all connections or one per
    connection; providers: the sse_seg.provider hint per connection (default 0). on_batch(batch index, result) sees every
    result before its slot is released. Returns (digests, carry_len, seg_flags)."""
    n = len(bodies)
    n_batches = bounds.shape[1] - 1
    d = orc.new_digests(n)
    carry = np.zeros(n, dtype=np.uint32)
    flags = np.zeros(n, dtype=np.uint32)
    conn = np.arange(n, dtype=np.uint32)
    eng.reset_all()
    for b in range(n_batches):
        plen = bounds[:, b + 1] - bounds[:, b]
        aligned = (plen + 15) & ~15
        offs = np.zeros(n, dtype=np.int64)
        offs[1:] = np.cumsum(aligned)[:-1]
        slot, arena, segs = eng.acquire()
        for i in range(n):
            if plen[i]:
                arena[offs[i]:offs[i] + plen[i]] = np.frombuffer(bodies[i], dtype=np.uint8, count=int(plen[i]), offset=int(bounds[i, b]))
        segs["conn"][:n] = conn
        segs["in_off"][:n] = offs
        segs["in_len"][:n] = plen
        segs["mode"][:n] = modes
        segs["provider"][:n] = 0 if providers is None else providers
        segs["reserved"][:n] = 0
        eng.submit(slot, n, int(offs[-1] + aligned[-1]))
        res = eng.collect(slot)
        try:
            check_result(eng, res, segs[:n])
            assert orc.digest_result(res.raw, conn, d, carry, flags) == n
            if on_batch is not None:
                on_batch(b, res)
        finally:
            eng.release(slot)
    return d, carry, flags


def oracle_digests(bodies, modes):
    """The oracle's digests of whole bodies (modes: one for all or one per body). Returns (digests, terminated, tail_len)."""
    n = len(bodies)
    lens = np.fromiter((len(b) for b in bodies), dtype=np.uint32, count=n)
    offs = np.zeros(n, dtype=np.uint64)
    offs[1:] = np.cumsum(lens.astype(np.uint64))[:-1]
    arena = np.frombuffer(b"".join(bodies) + b"\0", dtype=np.uint8)
    modes = np.ascontiguousarray(np.broadcast_to(np.asarray(modes, dtype=np.uint8), (n,)))
    return orc.digest_streams(arena, offs, lens, modes, max(1, len(os.sched_getaffinity(0))))


def decode_shape(n_items: int, sm_count: int) -> int:
    """Work items a warp of sse_decode_kernel pulls at a time for a batch of n_items decoded lines (csrc/sse_kernel2.cu:823-832).
    The kernel runs one CTA of 32 warps per SM. A batch with fewer items than 32 per warp spreads them over every warp, 8 or 16
    per pull, and then runs the whole warp over any lane left inside a long string (coop_max 32); above 16 per warp the pull
    is 32 items and the warp helps only when at most SSE_COOP (8) lanes are."""
    warps = sm_count * 32
    if n_items >= 32 * warps:
        return 32
    per = -(-n_items // warps)
    return 8 if per <= 8 else (16 if per <= 16 else 32)


def item_class(rel: int, provider: int) -> int:
    """Sort class of a decoded line (csrc/sse_kernel.cu:336-337): its rank among the decoded lines of its produce round (7 and
    up alike; the second line sorts first) and the segment's provider hint. A line longer than the produce window is class 0
    (csrc/sse_common.cuh:683)."""
    o = min(rel, 7)
    return ((0 if o == 1 else (1 if o == 0 else o)) << 2) | (provider & 3)


def item_sort_key(payload_len: int, cls: int) -> int:
    """Bucket of a work item in the decode kernel's item sort (item_bucket, csrc/sse_kernel2.cu:968-971): payload length in
    32-byte steps, longest first, every payload of 4,064 bytes or more in the last one; then the class. Items of one bucket
    keep about the order the produce kernel allocated them in, which follows the segment order."""
    return ((127 - min(payload_len >> 5, 127)) << 5) | cls


def _bytes(b: A.Bytes) -> bytes:
    return C.string_at(b.p, b.n) if b.n else b""


def agent_results(L, fold):
    content = _bytes(L.sse_agent_content(fold))
    has = bool(L.sse_agent_has_tool_calls(fold))
    fin = C.c_int()
    term = bool(L.sse_agent_terminated(fold, C.byref(fin)))
    arr = (A.ToolCall * 64)()
    n = L.sse_agent_tool_calls(fold, arr, 64)
    calls = [dict(id=_bytes(arr[i].id), type=_bytes(arr[i].type), name=_bytes(arr[i].name), args=_bytes(arr[i].arguments))
             for i in range(min(n, 64))]
    return content, has, term, fin.value, calls


def telemetry_results(L, fold):
    u = A.Usage()
    arr = (A.ToolCall * 64)()
    n = C.c_size_t()
    rc = L.sse_telemetry_finish(fold, C.byref(u), arr, 64, C.byref(n))
    calls = [dict(id=_bytes(arr[i].id), type=_bytes(arr[i].type), name=_bytes(arr[i].name), args=_bytes(arr[i].arguments))
             for i in range(min(n.value, 64))]
    return rc, (u.prompt_tokens, u.completion_tokens, u.total_tokens), calls


def _expect(l, frame: int, done: bool, mode_r: bool) -> dict:
    """The record the oracle's line l should give: its decoded fields (none past the nesting limit, DESIGN.md §5 deviation 2),
    the ordinal of its frame among the connection's frames (A.NONE: none), the bytes handed to json.Unmarshal, termination."""
    depth = l.depth_limited
    d = dict(json_ok=False) if depth else chunk_to_dict(l.chunk)
    d.update(done=done, done_exact=False, depth_limit=depth, frame=frame, payload_len=l.payload_len,
             terminates=mode_r and not done and d["json_ok"] and d["n_choices"] > 0 and d["finish"] in (orc.FIN_STOP, orc.FIN_TOOL_CALLS))
    return d


def check_stream(body: bytes, mode: int, o: ConnOut, label=""):
    """Bit-exact comparison of one connection's GPU output with the oracle."""
    if mode & A.MODE_R:
        v = orc.reframe(body)
        exp_frames = [l.out for l in v.lines if l.kind == orc.L_EMITTED]
        exp_recs = []
        n_frames = 0
        for l in v.lines:
            if l.kind == orc.L_EMITTED:
                exp_recs.append(_expect(l, n_frames, False, True))
                n_frames += 1
            elif l.kind == orc.L_DONE:
                exp_recs.append(_expect(l, A.NONE, True, True))
            elif l.kind == orc.L_DONE_EXACT:
                exp_recs.append(dict(json_ok=False, done=True, done_exact=True, depth_limit=False, frame=A.NONE, payload_len=6,
                                     terminates=False))
        assert o.terminated == v.terminated, f"{label}: terminated {o.terminated} != {v.terminated}"
    else:
        v = orc.passthrough(body, parse=bool(mode & A.MODE_PARSE))
        exp_frames = [l.out for l in v.lines]
        exp_recs = [_expect(l, k, False, False) for k, l in enumerate(v.lines) if l.chunk is not None]
        assert b"".join(o.frames) == v.out, f"{label}: passthrough bytes differ"
    assert len(o.frames) == len(exp_frames), f"{label}: {len(o.frames)} frames, oracle {len(exp_frames)}"
    for i, (g, e) in enumerate(zip(o.frames, exp_frames)):
        assert g == e, f"{label}: frame {i} differs:\n gpu={g[:120]!r}\n ref={e[:120]!r}"
    assert len(o.recs) == len(exp_recs), f"{label}: {len(o.recs)} recs, oracle {len(exp_recs)}"
    for i, (g, e) in enumerate(zip(o.recs, exp_recs)):
        assert not g["too_long"], f"{label}: rec {i} was not decoded (SSE_F_TOO_LONG)"
        for k, ev in e.items():
            assert g[k] == ev, f"{label}: rec {i} field {k}: gpu={g[k]!r} ref={ev!r}"
    if not o.terminated and not (o.flags & A.SEG_DEAD):
        assert o.carry_len == v.tail_len, f"{label}: carry {o.carry_len} != tail {v.tail_len}"
    return v
