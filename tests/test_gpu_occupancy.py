"""GPU: the adversarial corpora at full decode occupancy, compared with the oracle.

The decode kernel pulls 8, 16 or 32 work items per warp depending on how many items the batch has (tests.util.decode_shape),
and how it finishes long strings depends on that shape too. Small test batches only ever reach the 8-item shape, so here
plain filler lines are added to every micro-batch until the launch lands in the shape under test, and the shape is checked
from the batch's record count. Two mixes per shape:
  * dense: the adversarial lines plus filler with plain content strings: most lanes of a warp are inside strings, so in the
    32-item shape each lane resumes its own skip;
  * sparse: a seeded sample of the adversarial connections, each followed by 8 twins: connections with the same framing,
    payload lengths and cut positions whose payloads are number arrays. A twin's line has its adversarial line's sort bucket,
    class and batch, so each adversarial line shares its pull with about 8 lanes that are busy outside strings, and in the
    32-item shape the warp cooperates on the few lanes still inside a string.
A host-side restatement of the item sort (tests.util.item_sort_key) checks that the mixes are what they claim in the 32-item
shape. Every connection's frames and records are compared with the oracle through per-connection digests; a connection that
differs is shown field by field by check_stream."""
import functools

import numpy as np
import pytest
import torch

from inference_gateway_b200 import SseEngine, _abi as A, synth
from tests.corpus import TRICKY, mutate, string_alignment_docs, template_near_misses
from tests.streams import dealt, filler_payload
from tests.util import ENGINES, TARGET, cut_bounds, digest_parity, item_class, item_sort_key, one_context_at_a_time, shape_check

pytestmark = pytest.mark.gpu
R, PP = A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE
BATCH_BYTES = 96 << 20
MAX_CONNS = 65536
TWINS = 8
SPARSE_ADV_BYTES = (80 << 20) // (TWINS + 1)     # the sampled adversarial bodies and their twins take at most 80 MiB
LONG = 600                  # a payload at least this long holds a string that outlasts a lane's own skip (4 x 16 bytes)
BUF, LT_MAX = 8192, 64      # the produce kernel's line window and lines per round (csrc/sse_common.cuh:15-16)


@pytest.fixture(scope="module")
def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def engines():
    """engines(name): a context with that engine's flags; one context lives at a time."""
    yield from one_context_at_a_time(
        lambda name: SseEngine(device=0, max_conns=MAX_CONNS, bytes_per_batch=BATCH_BYTES, n_slots=1, flags=ENGINES[name]))


# ------------------------------------------------------------------ inputs
@functools.lru_cache(None)
def adversarial():
    """(bodies, modes, lines): one document per connection, so that a terminating chunk in mode R hides nothing; lines[i]
    holds (start of the line, offset of its '\\n', payload offset, payload length) per data line of body i. The
    string-alignment documents follow a line of 0-15 bytes (every payload alignment against the 16-byte windows) and, in mode
    R, 0-3 leading blanks; the other documents alternate between modes R and P|PARSE."""
    bodies, modes, lines = [], [], []

    def add(body, mode, payloads):
        ents, at = [], 0
        for p in payloads:
            ps = body.index(b"data: " + p, at) + 6
            at = ps + len(p)
            ents.append((body.rfind(b"\n", 0, ps) + 1, at, ps, len(p)))
        bodies.append(body); modes.append(mode); lines.append(ents)

    for i, d in enumerate(string_alignment_docs()):
        pre = b":" * (i % 16) + b"\n"
        if (i // 16) % 2:
            add(pre + b"data: " + d + b"\n\n", PP, [d])
        else:
            add(pre + b" " * ((i // 32) % 4) + b"data: " + d + b"\n\n", R, [d])
    for i, d in enumerate(TRICKY):
        d = d.replace(b"\n", b" ")
        add(b"data: " + d + b"\n", R, [d])
        add(b"data: " + d + b"\n", PP, [d])
    rng = np.random.default_rng(1000)
    streams, _ = synth.make_config("C4", n_streams=60)
    docs = [ev[6:] for b, _, _ in streams for ev in b.split(b"\n\n") if ev.startswith(b"data: {")] + TRICKY
    for i in range(3000):
        d = mutate(rng, docs[int(rng.integers(0, len(docs)))])
        add(b"data: " + d + b"\n", (R, PP)[i % 2], [d])
    for pad in range(40):                          # "[DONE]" and near misses at every alignment of the produce scan
        for j, marker in enumerate(("[DONE]", "[DONE", "[D", "[", "[DONEE]", "[done]", "[[DONE]]", "[D[DONE]")):
            a = ('{"choices":[{"delta":{"content":"%s%s tail"}}]}' % ("x" * pad, marker)).encode()
            b = b'{"choices":[{"delta":{"content":"next"}}]}'
            add(b"data: " + a + b"\n\ndata: " + b + b"\n\n", (R, PP)[(pad + j) % 2], [a, b])
    return bodies, np.array(modes, dtype=np.uint8), lines


def twin(body: bytes, ents) -> bytes:
    """body with every data payload replaced by a "nostring" payload of the same length."""
    out, at = [], 0
    for _, _, ps, n in ents:
        out += [body[at:ps], filler_payload("nostring", n)]
        at = ps + n
    return b"".join(out + [body[at:]])


def decoded(lines, bounds, providers, n_batches):
    """Host-side restatement of the produce stage, per batch: the decoded lines in segment order as (sort key, segment, line,
    payload length), with the class from the line's rank in its produce round (a round: at most LT_MAX lines in one BUF-byte
    window) or 0 for a line longer than the window."""
    out = [[] for _ in range(n_batches)]
    for s, (ents, row, prov) in enumerate(zip(lines, bounds, providers)):
        for b in range(n_batches):
            rs, rel = None, 0
            for k, (st, nl, _, n) in enumerate(ents):
                if not row[b] <= nl < row[b + 1]:
                    continue
                if nl + 1 - st > BUF - 16:
                    out[b].append((item_sort_key(n, 0), s, k, n))
                    rs = None
                    continue
                if rs is None or nl + 1 - rs > BUF - 16 or rel >= LT_MAX:
                    rs, rel = st, 0
                out[b].append((item_sort_key(n, item_class(rel, int(prov))), s, k, n))
                rel += 1
    return out


def string_lanes_per_pull(batches, is_string, pull):
    """For every string lane (is_string(segment, payload length)) of every batch: how many string lanes its pull of the
    sorted items holds."""
    got = []
    for items in batches:
        items = sorted(items)
        sl = np.array([is_string(s, n) for _, s, _, n in items], dtype=bool)
        per = np.pad(sl, (0, -len(sl) % pull)).reshape(-1, pull).sum(axis=1)
        got.append(np.repeat(per, pull)[:len(sl)][sl])
    return np.concatenate(got)


def mix(shape: int, kind: str, n_batches: int, sm_count: int):
    """(bodies, modes, bounds, providers, adversarial mask, string lanes per pull) of one run: the adversarial connections
    (sparse: each followed by its twins), cut at seeded positions, then the filler connections (mode R: no filler chunk
    finishes)."""
    bodies, modes, lines = adversarial()
    target = int(TARGET[shape] * sm_count * 32)
    rng = np.random.default_rng(shape * 10 + n_batches)
    if kind == "dense":
        pick, twins = np.arange(len(bodies)), 0
    else:                          # a seeded sample that leaves room: all its lines and their twins could land in one batch
        pick, n_lines, n_bytes, twins = [], 0, 0, TWINS
        for i in rng.permutation(len(bodies)):
            if n_lines + len(lines[i]) > 0.9 * target / (TWINS + 1) or n_bytes + len(bodies[i]) > SPARSE_ADV_BYTES:
                break
            pick.append(i); n_lines += len(lines[i]); n_bytes += len(bodies[i])
        pick = np.sort(pick)
    abounds = cut_bounds([bodies[i] for i in pick], n_batches, seed=77 + n_batches)
    cb, cm, cr, cl, cp, adv = [], [], [], [], [], []
    for i, row in zip(pick, abounds):
        for t in range(twins + 1):
            cb.append(bodies[i] if t == 0 else twin(bodies[i], lines[i]))
            cm.append(modes[i]); cr.append(row); cl.append(lines[i]); adv.append(t == 0)
            cp.append(i % 4 if kind == "dense" else 0)
    n_adv = [len(b) for b in decoded(cl, cr, cp, n_batches)]
    per_batch = []
    for b in range(n_batches):
        n_fill = target - n_adv[b]
        assert n_fill > 0
        if kind == "dense":       # plain strings of lengths spread over the item sort's buckets (the last from 4,064 bytes on)
            per_batch.append([filler_payload("strings", int(n)) for n in np.exp(rng.uniform(np.log(64), np.log(4160), n_fill))])
        else:                     # short lines outside strings: the launch's size only
            per_batch.append([filler_payload("nostring", int(n)) for n in rng.integers(40, 400, n_fill)])
    fb, fbounds, fl = dealt(per_batch)
    bounds = np.concatenate([np.array(cr, dtype=np.int64).reshape(-1, n_batches + 1), fbounds])
    providers = np.array(cp + [0] * len(fb), dtype=np.int64)
    adv = np.array(adv + [False] * len(fb))
    filler_strings = kind == "dense"
    lanes = string_lanes_per_pull(decoded(cl + fl, bounds, providers, n_batches),
                                  lambda s, n: n >= LONG and (adv[s] or (filler_strings and s >= len(cb))), shape)
    return cb + fb, np.concatenate([np.array(cm, dtype=np.uint8), np.full(len(fb), R, dtype=np.uint8)]), bounds, providers, adv, lanes


# ------------------------------------------------------------------ tests
CASES = [(e, s, nb) for e in ENGINES for s in (8, 16, 32) for nb in (1, 3)]


@pytest.mark.parametrize("engine_name,shape,n_batches", CASES, ids=[f"{e}-{s}-{nb}" for e, s, nb in CASES])
def test_adversarial_corpus_in_each_decode_shape(engines, sm_count, engine_name, shape, n_batches):
    eng = engines(engine_name)
    for kind in ("dense", "sparse"):
        bodies, modes, bounds, providers, adv, lanes = mix(shape, kind, n_batches, sm_count)
        assert len(bodies) <= MAX_CONNS and int((bounds[:, 1:] - bounds[:, :-1]).sum(axis=0).max()) + 16 * len(bodies) <= BATCH_BYTES
        if shape == 32:           # below it every warp helps its lanes in strings whatever their number (coop_max 32)
            coop = float(np.mean(lanes <= 8))
            if kind == "dense":
                assert coop < 0.5, f"dense: {coop:.0%} of the long-string lanes share their pull with 8 or fewer"
            else:
                assert coop > 0.9, f"sparse: only {coop:.0%} of the long-string lanes share their pull with 8 or fewer"
        log = []
        gd, _, _ = digest_parity(eng, bodies, modes, bounds, f"{engine_name} {shape}-item shape {kind} x{n_batches}",
                                 providers=providers, on_batch=shape_check(eng, sm_count, shape, log))
        assert len(log) == n_batches
        assert int(gd["n_recs"][adv].sum()) > 0
        print(f"{engine_name} {kind} shape {shape} batches {n_batches}: {int(adv.sum())} adversarial of {len(bodies)} connections, "
              f"{len(lanes)} long-string lanes, {np.mean(lanes <= 8):.0%} of them in pulls with <= 8, n_recs per launch {log}")


@pytest.mark.parametrize("engine_name", ["templates", "fused_templates"])
def test_template_near_misses_after_learning(engines, sm_count, engine_name):
    """Three launches in the 32-item shape on the same connections: canonical chunks teach the template cache; then near-misses
    of them among canonical chunks; then canonical chunks only, replayed from the cache the earlier launches left."""
    eng = engines(engine_name)
    canon, miss = template_near_misses()
    target = int(TARGET[32] * sm_count * 32)
    teach = [canon[i % len(canon)] for i in range(target)]
    mixed = miss + [canon[i % len(canon)] for i in range(target - len(miss))]
    rng = np.random.default_rng(3)
    mixed = [mixed[i] for i in rng.permutation(len(mixed))]
    bodies, bounds, _ = dealt([teach, mixed, teach])
    log = []
    digest_parity(eng, bodies, PP, bounds, f"{engine_name} near-misses", on_batch=shape_check(eng, sm_count, 32, log))
    assert len(log) == 3
    print(f"{engine_name}: {len(canon)} canonical chunks, {len(miss)} near-misses, n_recs per launch {log}")
