"""Shared parity harness: drives streams through the GPU path in randomly cut micro-batches and compares
every frame and every side-band record with the CPU oracle (oracle/ is the checker, never the product)."""
from __future__ import annotations

import ctypes as C
import os
import re
from unittest import mock

import numpy as np

from inference_gateway_b200 import _abi as A
from oracle import orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "sse_gpu.h")).read()
GW_HEADER = open(os.path.join(ROOT, "include", "sse_gateway.h")).read()

# the engine variants, by the names of the `engine` fixture (tests/conftest.py): split = produce / sort / decode / finalize
# pipeline, templates = the same with SSE_FLAG_TEMPLATES, copy = SSE_FLAG_COPY_OUT, fused = the single-pass tile kernel
ENGINES = {"split": 0, "templates": A.FLAG_TEMPLATES, "copy": A.FLAG_COPY_OUT, "fused": A.FLAG_KERNEL_FUSED,
           "fused_templates": A.FLAG_KERNEL_FUSED | A.FLAG_TEMPLATES}
# capacities far below what a batch of many streams needs: the produce side's still hold one round (64 lines) of one segment
TINY_PRODUCE = dict(max_frames=128, max_recs=64, out_arena_bytes=32 * 1024, max_runs=16)
TINY_DECODE = dict(max_tcs=8, max_usages=4, text_arena_bytes=512)


def declared_functions(text=None, prefix="sse_"):
    """The functions a C header (default include/sse_gpu.h) declares whose names start with prefix."""
    body = re.sub(r"/\*.*?\*/", "", text or HEADER, flags=re.S)
    return sorted(set(re.findall(r"\b(%s[a-z_0-9]+)\s*\(" % prefix, body)))


class ConnOut:
    def __init__(self):
        self.frames = []       # emitted frames (bytes) in order
        self.recs = []         # decoded records (dicts) in order
        self.terminated = False
        self.carry_len = 0
        self.flags = 0
        self.agent = None
        self.tele = None
        self.fold_rcs = []     # (piece index, sse_agent_feed rc, sse_telemetry_feed rc) of every segment fed to the folds
        self.piece_ends = []   # end offset in the body of every piece submitted, in piece order


def feed_folds(L, o: ConnOut, res, i: int, piece: int, keep_codes: bool):
    """Feeds segment i of a batch result, which holds bytes of piece `piece`, to the connection's folds. keep_codes: their
    return codes go to o.fold_rcs (check_folds judges them); otherwise a code other than SSE_OK raises."""
    rcs = (L.sse_agent_feed(o.agent, C.byref(res.raw), i), L.sse_telemetry_feed(o.tele, C.byref(res.raw), i))
    o.fold_rcs.append((piece, *rcs))
    if not keep_codes:
        A.check(rcs[0], "sse_agent_feed")
        A.check(rcs[1], "sse_telemetry_feed")


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
        count = int(r["tc_count"])
        # tc_count saturates at 0xFFFF: a saturated chain is walked to its end
        while len(tcs) < count or (count == 0xFFFF and t != A.NONE):
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


def one_context_at_a_time(make):
    """Body of a module fixture: yields get(key, **kw), the context make(key, **kw) built for key. Building one closes the one
    before, so that one large context lives at a time; get(None) closes it."""
    live = {}

    def get(key, **kw):
        if key not in live:
            for e in live.values():
                e.close()
            live.clear()
            if key is not None:
                live[key] = make(key, **kw)
        return live.get(key)
    yield get
    get(None)


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


def run_streams(engine, streams, modes, n_batches=1, seed=0, with_folds=False, keep_codes=False):
    """streams: list of bytes (one upstream body per connection); modes: list of mode bits.
    Feeds every stream in n_batches randomly cut pieces (simulated TCP segmentation), one micro-batch per
    piece index, and with_folds, every segment to the connection's agent and telemetry folds (feed_folds: keep_codes keeps
    their return codes for check_folds instead of raising). Returns list[ConnOut]."""
    from inference_gateway_b200.synth import random_cuts
    rng = np.random.default_rng(seed)
    L = engine.L
    n = len(streams)
    outs = [ConnOut() for _ in range(n)]
    engine.reset_all()
    pieces = [random_cuts(rng, s, n_batches) for s in streams]
    for o, p in zip(outs, pieces):
        o.piece_ends = np.cumsum([len(x) for x in p]).tolist()
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
                    feed_folds(L, o, res, i, b, keep_codes)
        finally:
            engine.release(slot)
    return outs


def run_deferred(eng, bodies, modes, n_batches=1, seed=0, with_folds=False, n_folds=None, keep_codes=False):
    """run_streams on an engine with SSE_FLAG_DEFER: every micro-batch of pieces is run to the end with SseEngine.process_all,
    which submits deferred remainders again until every byte was taken. The agent and telemetry folds are fed for the first
    n_folds streams (all by default). Returns (outs, stats)."""
    from inference_gateway_b200.synth import random_cuts
    rng = np.random.default_rng(seed)
    L = eng.L
    outs = [ConnOut() for _ in bodies]
    eng.reset_all()
    pieces = [random_cuts(rng, b, n_batches) for b in bodies]
    for o, p in zip(outs, pieces):
        o.piece_ends = np.cumsum([len(x) for x in p]).tolist()
    if with_folds:
        for o in outs[:n_folds]:
            o.agent, o.tele = L.sse_agent_new(), L.sse_telemetry_new()
    stats = dict(batches=0, deferred=0, overflow=0)
    piece = [0]

    def on_batch(res, conns):
        stats["overflow"] |= res.overflow
        for i, c in enumerate(conns):
            o = outs[c]
            fold_segment(o, res, i)
            stats["deferred"] += bool(int(res.segs[i]["flags"]) & A.SEG_DEFERRED)
            if o.agent is not None:
                feed_folds(L, o, res, i, piece[0], keep_codes)

    for b in range(max(len(p) for p in pieces)):
        piece[0] = b
        items = [(c, modes[c], pieces[c][b]) for c in range(len(bodies)) if b < len(pieces[c])]
        stats["batches"] += process_all_checked(eng, items, on_batch)
    return outs, stats


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


def fill_pieces(arena, segs, bodies, modes, bounds, b, providers=None) -> int:
    """Writes piece b of every body (bounds[i, b]:bounds[i, b + 1]) as segment i for connection i into an acquired slot.
    Returns the batch's input bytes."""
    n = len(bodies)
    plen = bounds[:, b + 1] - bounds[:, b]
    aligned = (plen + 15) & ~15
    offs = np.zeros(n, dtype=np.int64)
    offs[1:] = np.cumsum(aligned)[:-1]
    for i in range(n):
        if plen[i]:
            arena[offs[i]:offs[i] + plen[i]] = np.frombuffer(bodies[i], dtype=np.uint8, count=int(plen[i]), offset=int(bounds[i, b]))
    segs["conn"][:n] = np.arange(n, dtype=np.uint32)
    segs["in_off"][:n] = offs
    segs["in_len"][:n] = plen
    segs["mode"][:n] = modes
    segs["provider"][:n] = 0 if providers is None else providers
    segs["reserved"][:n] = 0
    return int(offs[-1] + aligned[-1])


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
        slot, arena, segs = eng.acquire()
        eng.submit(slot, n, fill_pieces(arena, segs, bodies, modes, bounds, b, providers))
        res = eng.collect(slot)
        try:
            check_result(eng, res, segs[:n])
            assert orc.digest_result(res.raw, conn, d, carry, flags) == n
            if on_batch is not None:
                on_batch(b, res)
        finally:
            eng.release(slot)
    return d, carry, flags


class PipelinedDigests:
    """digest_run with up to `depth` batches in flight: batch b is filled and submitted while up to depth - 1 earlier batches
    are still uncollected. collect_order "fifo" collects the oldest batch once depth are in flight; "lifo" fills every slot and
    then collects the newest first. Whatever order they are collected in, results are folded into the digests in fold_order
    (default: submission order); a collected slot stays unreleased until its turn comes, so fold_order may only move a batch
    by less than depth places. Every collected batch passes check_result.
    between(b) runs after submit b and before the next acquire; on_batch(b, result, slot) sees every result, in fold order,
    before its slot is released. step() submits one batch, so two runs (on two contexts) can be interleaved."""

    def __init__(self, eng, bodies, modes, bounds, depth, collect_order="fifo", providers=None, between=None, on_batch=None,
                 fold_order=None):
        assert collect_order in ("fifo", "lifo") and 1 <= depth <= eng.cfg.n_slots
        self.eng, self.bodies, self.modes, self.bounds, self.providers = eng, bodies, modes, bounds, providers
        self.depth, self.lifo, self.between, self.on_batch = depth, collect_order == "lifo", between, on_batch
        self.n = n = len(bodies)
        self.n_batches = bounds.shape[1] - 1
        self.order = list(range(self.n_batches)) if fold_order is None else list(fold_order)
        assert sorted(self.order) == list(range(self.n_batches))
        self.d = orc.new_digests(n)
        self.carry = np.zeros(n, dtype=np.uint32)
        self.flags = np.zeros(n, dtype=np.uint32)
        self.conn = np.arange(n, dtype=np.uint32)
        self.inflight = []      # (batch, slot, segs) submitted, not collected, oldest first
        self.collected = {}     # batch -> (slot, result) collected, not yet folded
        self.next_batch = 0
        self.folded = 0
        eng.reset_all()

    def _collect(self, k):
        b, slot, segs = self.inflight.pop(k)
        try:
            res = self.eng.collect(slot)
            check_result(self.eng, res, segs)
        except BaseException:
            self.eng.release(slot)
            raise
        self.collected[b] = (slot, res)

    def _fold_ready(self):
        while self.folded < self.n_batches and self.order[self.folded] in self.collected:
            b = self.order[self.folded]
            slot, res = self.collected.pop(b)
            try:
                assert orc.digest_result(res.raw, self.conn, self.d, self.carry, self.flags) == self.n
                if self.on_batch is not None:
                    self.on_batch(b, res, slot)
            finally:
                self.eng.release(slot)
            self.folded += 1

    def _drain(self):
        while self.inflight:
            self._collect(-1 if self.lifo else 0)
        self._fold_ready()

    def step(self) -> bool:
        """Submits the next batch (collecting first where depth batches are held). False once every batch was submitted."""
        if self.next_batch == self.n_batches:
            return False
        while len(self.inflight) + len(self.collected) >= self.depth:
            assert self.inflight, f"fold order {self.order} holds {self.depth} collected batches: it cannot advance"
            if self.lifo:
                self._drain()
            else:
                self._collect(0)
                self._fold_ready()
        b = self.next_batch
        slot, arena, segs = self.eng.acquire()
        try:
            self.eng.submit(slot, self.n, fill_pieces(arena, segs, self.bodies, self.modes, self.bounds, b, self.providers))
        except BaseException:
            self.eng.release(slot)
            raise
        self.inflight.append((b, slot, segs[:self.n].copy()))
        self.next_batch += 1
        if self.between is not None:
            self.between(b)
        return True

    def finish(self):
        """Submits what is left, collects and folds everything. Returns (digests, carry_len, seg_flags) as digest_run does."""
        while self.step():
            pass
        self._drain()
        assert self.folded == self.n_batches and not self.collected
        return self.d, self.carry, self.flags

    def abort(self):
        """Releases every slot the run still holds (after a failure), so that the context stays usable."""
        for _, slot, _ in self.inflight:
            self.eng.release(slot)
        for slot, _ in self.collected.values():
            self.eng.release(slot)
        self.inflight, self.collected = [], {}


def digest_run_pipelined(eng, bodies, modes, bounds, depth, collect_order="fifo", providers=None, between=None, on_batch=None,
                         fold_order=None):
    """digest_run with depth batches in flight (PipelinedDigests). Returns (digests, carry_len, seg_flags)."""
    run = PipelinedDigests(eng, bodies, modes, bounds, depth, collect_order, providers, between, on_batch, fold_order)
    try:
        return run.finish()
    except BaseException:
        run.abort()
        raise


def oracle_digests(bodies, modes):
    """The oracle's digests of whole bodies (modes: one for all or one per body). Returns (digests, terminated, tail_len)."""
    n = len(bodies)
    lens = np.fromiter((len(b) for b in bodies), dtype=np.uint32, count=n)
    offs = np.zeros(n, dtype=np.uint64)
    offs[1:] = np.cumsum(lens.astype(np.uint64))[:-1]
    arena = np.frombuffer(b"".join(bodies) + b"\0", dtype=np.uint8)
    modes = np.ascontiguousarray(np.broadcast_to(np.asarray(modes, dtype=np.uint8), (n,)))
    return orc.digest_streams(arena, offs, lens, modes, max(1, len(os.sched_getaffinity(0))))


# ------------------------------------------------------------------ the digest verdict
DIGEST_FIELDS = ("n_frames", "frame_bytes", "frames_h", "n_recs", "recs_h")
RULES = {
    "digests": "frames or records differ from the oracle's",
    "inexact": "records left undecoded (SSE_F_TOO_LONG) or with a broken tool-call chain",
    "termination": "termination differs from the oracle's",
    "seg_flags": "SSE_SEG_DEAD, SSE_SEG_LINE_TOO_LONG or SSE_SEG_DEFERRED set",
    "finished": "SSE_SEG_FINISHED on a connection that did not terminate",
    "carry": "the carried tail of a live connection differs from the oracle's",
}


def parity_faults(got, oracle, skip=()) -> dict:
    """The rules of RULES that a run's (digests, carry_len, seg_flags) breaks against the oracle's (digests, terminated,
    tail_len): {rule: the connections that break it}, empty when the run is the oracle's. skip: connections left out."""
    gd, carry, flags = got
    od, oterm, otail = oracle
    keep = np.ones(len(gd), dtype=bool)
    keep[list(skip)] = False
    gterm = (flags & A.SEG_TERMINATED) != 0
    broken = {
        "digests": np.any([gd[k] != od[k] for k in DIGEST_FIELDS], axis=0),
        "inexact": gd["inexact"] != 0,
        "termination": gterm != oterm.astype(bool),
        "seg_flags": (flags & (A.SEG_DEAD | A.SEG_LINE_TOO_LONG | A.SEG_DEFERRED)) != 0,
        "finished": ((flags & A.SEG_FINISHED) != 0) & ~gterm,
        "carry": ~gterm & (carry != otail),
    }
    return {rule: np.nonzero(bad & keep)[0] for rule, bad in broken.items() if np.any(bad & keep)}


def parity_message(label, faults, got, oracle) -> str:
    """Each broken rule with its first connections, and what the run and the oracle hold for the first of them."""
    gd, carry, flags = got
    od, oterm, otail = oracle
    out = [f"{label}: the run differs from the oracle"]
    for rule, conns in faults.items():
        c = conns[0]
        out += [f"  {RULES[rule]}: {conns.size} connection(s), first {conns[:8].tolist()}",
                f"    connection {c}: gpu {DIGEST_FIELDS} {gd[list(DIGEST_FIELDS)][c]} inexact {gd['inexact'][c]} seg_flags "
                f"{int(flags[c]):#x} carry {carry[c]}; oracle {od[list(DIGEST_FIELDS)][c]} terminated {bool(oterm[c])} tail {otail[c]}"]
    return "\n".join(out)


def assert_digest_parity(got, bodies, modes, label, *, oracle=None, skip=()):
    """The digest verdict: got, a run's (digests, carry_len, seg_flags), breaks no rule of RULES against the oracle's single
    pass over every whole body (oracle: oracle_digests(bodies, modes) when already computed) on any connection but those in
    skip. Returns the oracle's digests."""
    oracle = oracle if oracle is not None else oracle_digests(bodies, modes)
    faults = parity_faults(got, oracle, skip)
    assert not faults, parity_message(label, faults, got, oracle)
    return oracle[0]


def digest_parity(eng, bodies, modes, bounds, label, *, providers=None, on_batch=None, oracle=None, skip=(), depth=1,
                  **pipelined):
    """Feeds the bodies in the pieces bounds gives (digest_run, or digest_run_pipelined with depth batches in flight and its
    other arguments) and applies assert_digest_parity. When a rule is broken, the same engine runs the same batches again
    and the first connections that break one are compared field by field (check_stream); if they compare equal, the digest
    message is the failure. Returns the run's (digests, carry_len, seg_flags)."""
    modes = np.ascontiguousarray(np.broadcast_to(np.asarray(modes, dtype=np.uint8), (len(bodies),)))
    oracle = oracle if oracle is not None else oracle_digests(bodies, modes)

    def run(hook):
        if depth == 1 and not pipelined:
            return digest_run(eng, bodies, modes, bounds, providers, hook)
        return digest_run_pipelined(eng, bodies, modes, bounds, depth, providers=providers, on_batch=hook, **pipelined)
    got = run(on_batch)
    faults = parity_faults(got, oracle, skip)
    if faults:
        outs = {int(c): ConnOut() for c in np.unique(np.concatenate(list(faults.values())))[:4]}

        def keep(b, res, *slot):
            for c, o in outs.items():
                fold_segment(o, res, c)
        run(keep)
        for c, o in outs.items():
            check_stream(bodies[c], int(modes[c]), o, label=f"{label} connection {c}")
    assert not faults, parity_message(label, faults, got, oracle)
    return got


# ------------------------------------------------------------------ decode launch shapes
# decoded lines per launch, in items per warp of the grid: 10 % or more inside each shape's range (8: up to 8, 16: above 8 up
# to 16, 32: above 16)
TARGET = {8: 6.5, 16: 12.0, 32: 20.0}


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


def shape_check(eng, sm_count, shape, log):
    """digest_run hook: the launch's decoded lines must put it in `shape`, at least 10 % inside that shape's range. A record
    is written for each decoded line and for each exact "data: [DONE]" line, which gets no work item."""
    warps = sm_count * 32
    lo, hi = {8: (0, 8 * warps), 16: (8 * warps, 16 * warps), 32: (16 * warps, None)}[shape]

    def on_batch(b, res):
        n_items = int(res.raw.n_recs) - int(np.count_nonzero(res.recs["flags"] & A.F_DONE_EXACT))
        log.append(int(res.raw.n_recs))
        if eng.cfg.flags & A.FLAG_KERNEL_FUSED:          # the tile kernel has no decode launch
            return
        got = decode_shape(n_items, sm_count)
        assert got == shape, f"batch {b}: {n_items} decoded lines on {sm_count} SMs decode {got} items per warp, not {shape}"
        assert n_items >= 1.1 * lo and (hi is None or n_items <= 0.9 * hi), \
            f"batch {b}: {n_items} decoded lines are within 10 % of a boundary of the {shape}-item shape ({lo}, {hi}]"
    return on_batch


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


def _calls(arr, n):
    return [dict(id=_bytes(arr[i].id), type=_bytes(arr[i].type), name=_bytes(arr[i].name), args=_bytes(arr[i].arguments))
            for i in range(n)]


def agent_results(L, fold):
    """An agent fold's (content, has_tool_calls, terminated, finish, every merged tool call)."""
    content = _bytes(L.sse_agent_content(fold))
    has = bool(L.sse_agent_has_tool_calls(fold))
    fin = C.c_int()
    term = bool(L.sse_agent_terminated(fold, C.byref(fin)))
    n = L.sse_agent_tool_calls(fold, None, 0)
    arr = (A.ToolCall * max(1, n))()
    assert L.sse_agent_tool_calls(fold, arr, n) == n
    return content, has, term, fin.value, _calls(arr, n)


def telemetry_results(L, fold):
    """sse_telemetry_finish: (rc, usage, every tool call). The call array is sized from the count a first call returns; the
    fold closes its open piece once, so the second call sees the same state."""
    u = A.Usage()
    n = C.c_size_t()
    arr = (A.ToolCall * 64)()
    rc = L.sse_telemetry_finish(fold, C.byref(u), arr, 64, C.byref(n))
    if n.value > 64:
        arr = (A.ToolCall * n.value)()
        m = C.c_size_t()
        rc = L.sse_telemetry_finish(fold, C.byref(u), arr, n.value, C.byref(m))
        assert m.value == n.value
    return rc, (u.prompt_tokens, u.completion_tokens, u.total_tokens), _calls(arr, n.value)


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


def check_streams(bodies, modes, outs, label="", L=None):
    """check_stream on every connection (modes: one for all or one per body) and, given the library L, check_folds on every
    connection that has folds. Returns the oracle's views."""
    modes = np.broadcast_to(np.asarray(modes), (len(bodies),))
    views = [check_stream(b, int(m), o, label=f"{label} stream {i} mode {m}") for i, (b, m, o) in enumerate(zip(bodies, modes, outs))]
    for i, (m, o, v) in enumerate(zip(modes, outs, views)):
        if L is not None and o.agent is not None:
            check_folds(L, o, int(m), v, f"{label} stream {i} mode {m}")
    return views


# ------------------------------------------------------------------ the fold verdict
DONE = b"data: [DONE]\n\n"


def check_agent(state, v, label=""):
    """An agent fold's (content, has_tool_calls, terminated, finish, tool calls), as agent_results or Gateway.agent_state
    gives them, against the oracle's reframe of the same body (v, as check_stream returns it in mode R)."""
    content, has, term, fin, calls = state
    assert content == v.acc_content, f"{label}: agent content differs from the oracle's"
    assert (has, term) == (v.has_tool_calls, v.terminated), \
        f"{label}: has_tool_calls, terminated {(has, term)}, oracle {(v.has_tool_calls, v.terminated)}"
    assert not term or fin == v.term_finish, f"{label}: finish {fin}, oracle {v.term_finish}"
    assert calls == orc.parse_tool_calls(v.builder), f"{label}: tool calls differ from the oracle's"


def irregular_telemetry(body: bytes) -> bool:
    """Whether telemetry's "\n\n" pieces of body hold one of several non-blank lines that starts with "data: " (DESIGN.md §5,
    deviation 4): the telemetry fold then finishes with 1 and its usage and tool calls are not the reference's."""
    return any(p.startswith(b"data: ") and sum(1 for x in p.split(b"\n") if x) > 1 for p in body.split(b"\n\n"))


def first_limited_piece(v, piece_ends):
    """The piece that completes the oracle's first line past the nesting limit (v: its view of the body; piece_ends: the end
    offset of every piece), or None when no line is."""
    end = 0
    for l in v.lines:
        end += len(l.line)
        if l.kind != orc.L_UNREAD and l.depth_limited:
            return next(k for k, e in enumerate(piece_ends) if e >= end)
    return None


def check_folds(L, o: ConnOut, mode: int, v, label=""):
    """The agent and telemetry folds run_streams(with_folds=True) fed for one connection, against the oracle (v: what
    check_stream returned).
    - A stream without a line past the nesting limit: every feed returns SSE_OK. Mode R: the agent fold (check_agent), and
      the telemetry over the frames and the [DONE] the agent writes at the end; mode P|PARSE: the telemetry over the frames.
      The telemetry finishes with 1 exactly when those bytes have an irregular piece (irregular_telemetry), and is then not
      compared further; else with 0 and the oracle's usage and tool calls.
    - A stream with one: both feeds return SSE_OK up to the piece that completes the first such line and SSE_ERR_UNDECODED in
      it; the accumulators are short and are not compared.
    Returns the agent fold's state (None outside mode R, or when the stream has a line past the nesting limit)."""
    limited = first_limited_piece(v, o.piece_ends)
    bad = [(p, a, t) for p, a, t in o.fold_rcs if (a, t) != (A.SSE_OK, A.SSE_OK)]
    if limited is not None:
        assert bad and bad[0][0] == limited and bad[0][1:] == (A.SSE_ERR_UNDECODED,) * 2, \
            f"{label}: first failed feeds {bad[:1]}, oracle: a line past the nesting limit in piece {limited}"
        return None
    assert not bad, f"{label}: feeds failed {bad[:4]} (piece, agent rc, telemetry rc) on a stream the decoder can take whole"
    state = None
    if mode & A.MODE_R:
        state = agent_results(L, o.agent)
        check_agent(state, v, label)
        A.check(L.sse_telemetry_feed_bytes(o.tele, DONE, len(DONE)), "sse_telemetry_feed_bytes")
        body = b"".join(o.frames) + DONE
    elif mode & A.MODE_PARSE:
        body = b"".join(o.frames)
    else:
        return None
    rc, usage, calls = telemetry_results(L, o.tele)
    if irregular_telemetry(body):
        assert rc == 1, f"{label}: telemetry finished with {rc} on a body with an irregular piece"
    else:
        assert (rc, usage, calls) == (0, *orc.telemetry(body)), f"{label}: telemetry differs"
    return state


# ------------------------------------------------------------------ SSE_FLAG_COUNTERS
CYCLES = ("c_pull", "c_skip", "c_coop", "c_steps", "c_finish", "c_unquote")


def text_spans(res):
    """(spans flagged SSE_F_CONTENT_TEXT or SSE_TC_*_TEXT, records with at least one, whether any tool-call element has two)"""
    recs, tcs = res.recs, res.tcs
    content = (recs["flags"] & A.F_CONTENT_TEXT) != 0
    per_tc = np.array([bin(int(f) & 0xF0).count("1") for f in tcs["flags"]], dtype=np.int64)
    with_text = content.copy()
    for i in np.nonzero(~content)[0]:
        t = int(recs["tc_first"][i])
        while t != A.NONE and t < len(tcs) and not with_text[i]:
            with_text[i] = per_tc[t] > 0
            t = int(tcs["next"][t])
    return int(content.sum() + per_tc.sum()), int(with_text.sum()), bool((per_tc > 1).any())


def check_batch(k, res, submitted=None, one_job_per_span=True):
    """The identities the counters k of every batch result res satisfy. submitted: the batch's input bytes (their '\\n' are the
    complete lines when no segment stopped early)."""
    raw = res.raw
    assert k["decode_passes"] == (1 if raw.n_segs else 0) or k["decode_passes"] > 1, k
    assert k["p_segments"] == raw.n_segs, (k, raw.n_segs)
    assert k["p_items"] == raw.n_decoded, (k, raw.n_decoded)
    assert k["p_frames_zero_copy"] + k["p_frames_materialised"] == raw.n_frames, (k, raw.n_frames)
    mat = res.frames["off"] < res.in_base
    assert k["p_bytes_materialised"] == int(res.frames["len"][mat].sum()), (k, int(res.frames["len"][mat].sum()))
    if submitted is not None:
        nl = submitted.count(b"\n")
        stopped = int(np.count_nonzero(res.segs["flags"] & (A.SEG_TERMINATED | A.SEG_FINISHED | A.SEG_DEAD | A.SEG_DEFERRED)))
        assert k["p_lines"] == nl if not stopped else k["p_lines"] <= nl, (k, nl, stopped)
    decoded = (res.recs["flags"] & A.F_DONE_EXACT) == 0          # an exact "data: [DONE]" gets a record but no work item
    moved = (k["d_skip_bytes"] + k["d_coop_bytes"] + k["d_plain_steps"] + k["d_actions"] + k["d_abandoned_bytes"]
             + k["d_template_bytes"])
    assert moved == int(res.recs["payload_len"][decoded].sum()), k
    assert k["d_items"] == k["d_lines_finished"] == raw.n_decoded, (k, raw.n_decoded)
    assert k["d_busy_lane_rounds"] <= 32 * k["d_warp_rounds"], k
    assert sum(k[c] for c in CYCLES) <= k["c_total"], k
    if raw.n_decoded:
        assert k["d_items_per_pull"] in (8, 16, 32) and k["d_pulls"] > 0, k
    # every unquote job yields one text span. A lane queues one job at a time (the warp drains the queues every two rounds), so
    # a line's first string to unquote is always a job, and a tool-call element with two such strings, or a line replayed
    # from a template (all its captures at once), unquotes the rest on its lane
    spans, lines, two = text_spans(res)
    assert lines <= k["d_unquote_jobs"] <= spans, (k, lines, spans)
    if one_job_per_span and not two:
        assert k["d_unquote_jobs"] == spans, (k, spans)
