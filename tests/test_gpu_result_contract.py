"""GPU: the parts of a batch result that tie its contents together, on inputs the other corpora never reach. Every batch here
goes through orc_check_result (runs, frame and record ranges, record -> frame links, chains, spans, termination and segment
flags), and every connection is compared with the oracle including each record's frame link, payload_len, SSE_F_TERMINATES
and SSE_F_DEPTH_LIMIT (tests/util.py::check_stream, oracle/orc_check.c digests)."""
import numpy as np
import pytest

from inference_gateway_b200 import SseEngine, _abi as A
from tests.corpus import nesting_docs
from tests.streams import chunk
from tests.util import ENGINES, check_stream, check_streams, digest_parity, run_pieces, run_streams

pytestmark = pytest.mark.gpu

R, PP = A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE
MiB = 1 << 20


STOP = chunk(b"bye", '"stop"')
DONE = b"data: [DONE]\n\n"


# ------------------------------------------------------------------ nesting at the 128-level limit
@pytest.mark.parametrize("n_batches", [1, 3])
@pytest.mark.parametrize("mode", [R, PP], ids=["R", "PP"])
def test_nesting_limit_is_flagged_exactly(engine, mode, n_batches):
    """Every document of the nesting corpus (tests/corpus.py::nesting_docs), each after its shallow twin: a record carries
    SSE_F_DEPTH_LIMIT exactly when the oracle's restatement of the limit says so, and is otherwise decoded like any other."""
    docs = nesting_docs()
    bodies = [b"".join(b"data: " + twin + b"\n\ndata: " + d + b"\n\n" for _, d, twin in docs[k:k + 12]) + DONE
              for k in range(0, len(docs), 12)]
    modes = [mode] * len(bodies)
    outs = run_streams(engine, bodies, modes, n_batches=n_batches, seed=n_batches)
    check_streams(bodies, modes, outs, "nesting")
    flagged = sum(r["depth_limit"] for o in outs for r in o.recs)
    assert flagged > 300, flagged


# ------------------------------------------------------------------ record -> frame links across run boundaries
SWALLOWED = [b"data: [DONE]\n\n", b"[DONE]\n\n", b"data: x[DONE]\n\n", b'data: {"choices":[{"delta":{"content":"[DONE]"}}]}\n\n']


def long_segment(n_lines: int, term_at: int | None, seed: int) -> bytes:
    """n_lines chunks, swallowed [DONE] lines at and around the 64-line run edges, comment and blank lines (frames without a
    record in mode P), and a terminating chunk at line term_at."""
    rng = np.random.default_rng(seed)
    parts = []
    for i in range(n_lines):
        if i == term_at:
            parts.append(chunk(b"end %d" % i, '"stop"' if i & 1 else '"tool_calls"'))
        elif i in (62, 63, 65, 127, 128, 129, 191, 192):
            parts.append(SWALLOWED[int(rng.integers(len(SWALLOWED)))])
        elif i % 17 == 5:
            parts.append(b": ping\n\n")
        else:
            parts.append(chunk(b"t%d " % i + b"x" * int(rng.integers(0, 40))))
    return b"".join(parts)


@pytest.mark.parametrize("n_batches", [1, 4])
def test_links_across_runs(engine, n_batches):
    """Segments of 200 lines (several 64-line runs) whose swallowed [DONE] lines sit at run edges, terminating in the first, a
    middle or the last run or not at all, in mode R and P|PARSE."""
    bodies, modes = [], []
    for term_at in (None, 10, 63, 64, 100, 190, 199):
        for seed in range(4):
            body = long_segment(200, term_at, seed) + DONE
            for m in (R, PP):
                bodies.append(body)
                modes.append(m)
    outs = run_streams(engine, bodies, modes, n_batches=n_batches, seed=7 + n_batches)
    check_streams(bodies, modes, outs, "runs")
    assert sum(o.terminated for o in outs) == 4 * 6


def test_terminating_chunk_completed_from_the_carry_slot(engine):
    """The terminating chunk is a line the batch completes from the connection's carry slot: its head came in the previous
    batch, cut at every kind of place (inside "data: ", inside the payload, before the '\\n', before the blank line)."""
    head = long_segment(70, None, 3)
    stop = chunk(b"the end " * 300, '"stop"')
    body = head + stop + chunk(b"never read") + DONE
    cuts = [1, 3, 6, 7, 100, len(stop) - 3, len(stop) - 2, len(stop) - 1]
    pieces = [[body[:len(head) + c], body[len(head) + c:]] for c in cuts]
    pieces += [[body[:len(head) + c], body[len(head) + c:len(head) + c + 1], body[len(head) + c + 1:]] for c in cuts]
    outs = run_pieces(engine, pieces, [R] * len(pieces))
    for i, o in enumerate(outs):
        check_stream(body, R, o, label=f"carry cut {i}")
        assert o.terminated


@pytest.fixture(scope="module", params=["split", "templates", "copy"])
def pooled(request):
    e = SseEngine(device=0, max_conns=64, bytes_per_batch=8 * MiB, carry_slot_bytes=32768, n_slots=2, text_arena_bytes=16 * MiB,
                  flags=ENGINES[request.param], line_pool=dict(pool_pages=64, page_bytes=65536))
    yield e
    e.close()


def test_terminating_chunk_completed_from_the_line_pool(pooled):
    """The terminating chunk is a 200 KB line assembled in line-pool pages over several batches, after 70 lines (two runs)."""
    head = long_segment(70, None, 5)
    stop = chunk(b"0123456789abcdef" * 12800, '"tool_calls"')
    body = head + stop + chunk(b"never read") + DONE
    a = len(head)
    pieces = [[body[:a + 10], body[a + 10:a + 40000], body[a + 40000:a + 150000], body[a + 150000:]],
              [body[:a + 50000], body[a + 50000:a + len(stop) - 1], body[a + len(stop) - 1:]],
              [body[:a + len(stop) - 2], body[a + len(stop) - 2:]]]
    for modes in ([R] * 3, [R, PP, R]):
        outs = run_pieces(pooled, pieces, modes)
        for i, (m, o) in enumerate(zip(modes, outs)):
            check_stream(body, m, o, label=f"pool cut {i} mode {m}")
            assert o.terminated == (m == R)
    assert pooled.pool_stats()[0] == 0


# ------------------------------------------------------------------ aliasing: identical bytes on every connection
@pytest.mark.parametrize("mode", [R, PP], ids=["R", "PP"])
def test_identical_connections_are_not_cross_wired(engine, mode):
    """4,096 connections carry byte-identical bodies of 70 lines, cut identically into 6 batches. A run, frame or span that
    points at another connection's identical bytes gives the same digests; only the structural check can tell."""
    n = 4096
    body = long_segment(70, None, 11) + STOP + DONE
    assert 5200 < len(body) < 6700       # the largest piece, 16-byte aligned, times 4,096 fits the 8 MiB batch
    bodies = [body] * n
    row = np.array([0, 17, 1300, 2600, 3900, 5200, len(body)], dtype=np.int64)
    bounds = np.tile(row, (n, 1))
    digest_parity(engine, bodies, mode, bounds, f"identical connections mode {mode}")
