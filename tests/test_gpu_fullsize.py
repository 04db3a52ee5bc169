"""GPU: BASELINE.json's configurations at their stated stream counts (C2 4,096 / C3 16,384 / C4 65,536 concurrent streams).
Two kinds of checks:
  * oracle parity at full size: every stream is cut at seeded random byte positions into n_batches TCP-like pieces, fed through
    the C ABI batch by batch, and every frame and every side-band record is compared with the oracle's single pass over the
    whole body -- as per-connection 64-bit digests of the canonical byte string both sides produce (oracle/orc_check.c; the
    field list is check_stream's), plus frame / record counts, termination and the held-back tail length;
  * size-independent properties: exact byte identities between input and output, record/frame accounting, idempotence."""
import numpy as np
import pytest

from inference_gateway_b200 import SseEngine, _abi as A, synth
from tests.util import ENGINES, cut_bounds, digest_parity, digest_run, fill_pieces, one_context_at_a_time, oracle_digests

pytestmark = pytest.mark.gpu
N = 65536
R = A.MODE_R | A.MODE_PARSE


@pytest.fixture(scope="module")
def workload():
    streams, _ = synth.make_config("C4", n_streams=N)
    return [b for b, _, _ in streams]


@pytest.fixture(scope="module")
def engines(workload):
    """engines(flags): the full-size context with those engine flags; one context lives at a time."""
    yield from one_context_at_a_time(lambda flags: SseEngine(device=0, max_conns=N, bytes_per_batch=sum(map(len, workload)),
                                                             n_slots=1, carry_slot_bytes=16384, flags=flags))


@pytest.fixture
def eng(engines):
    return engines(0)


# ------------------------------------------------------------------ oracle parity at full size
# the default engine on every case; skeleton templates, COPY_OUT, the tile kernel and the tile kernel with templates on the
# mode R cases (grouped by engine: one context is built per group)
FULLSIZE = [("C2", 4096, A.MODE_P, 4), ("C2", 4096, A.MODE_P | A.MODE_PARSE, 5),
            ("C3", 16384, R, 1), ("C3", 16384, R, 4),
            ("C4", 65536, R, 1), ("C4", 65536, R, 4), ("C4", 65536, A.MODE_P | A.MODE_PARSE, 6)]


@pytest.mark.parametrize("name,n_streams,mode,n_batches,eng_flags", [
    pytest.param(*c, 0, id="-".join(map(str, c))) for c in FULLSIZE] + [
    pytest.param(*c, f, id="-".join(map(str, c)) + "-" + e) for e, f in ENGINES.items() if e != "split" for c in FULLSIZE if c[0] != "C2" and c[2] == R])
def test_oracle_parity_at_full_size(engines, workload, name, n_streams, mode, n_batches, eng_flags):
    eng = engines(eng_flags)
    bodies = workload if name == "C4" else [b for b, _, _ in synth.make_config(name, n_streams=n_streams)[0]]
    assert len(bodies) == n_streams
    gd, _, _ = digest_parity(eng, bodies, mode, cut_bounds(bodies, n_batches, seed=1000 + n_batches),
                             f"{name} x{n_streams} mode {mode} batches {n_batches} flags {eng_flags}")
    assert int(gd["n_recs"].sum()) > 0 or mode == A.MODE_P


def test_digest_checker_sees_a_single_flipped_bit(eng, workload):
    """The digests are only as good as their sensitivity: corrupt one byte of one body on the oracle side only."""
    bodies = list(workload[:2048])
    od, _, _ = oracle_digests(bodies, R)
    k = bodies[777].find(b'"content":"') + 12
    twisted = bodies[777][:k] + bytes([bodies[777][k] ^ 1]) + bodies[777][k + 1:]
    bodies2 = bodies[:777] + [twisted] + bodies[778:]
    od2, _, _ = oracle_digests(bodies2, R)
    diff = np.nonzero((od["frames_h"] != od2["frames_h"]) | (od["recs_h"] != od2["recs_h"]))[0]
    assert list(diff) == [777]
    gd, _, _ = digest_run(eng, bodies, R, cut_bounds(bodies, 3, seed=5))
    assert np.array_equal(gd["frames_h"], od["frames_h"]) and np.array_equal(gd["recs_h"], od["recs_h"])
    assert gd["recs_h"][777] != od2["recs_h"][777]


# ------------------------------------------------------------------ size-independent properties
def _run(eng, bodies, mode):
    eng.reset_all()
    slot, arena, segs = eng.acquire()
    eng.submit(slot, len(bodies), fill_pieces(arena, segs, bodies, mode, cut_bounds(bodies, 1, 0), 0))
    return slot, eng.collect(slot)


def _per_stream(res):
    """Total frame count / record count / emitted bytes per segment, following the extra runs of long segments."""
    ff, fc = res.segs["frame_first"].astype(np.int64), res.segs["frame_count"].astype(np.int64)
    rc = res.segs["rec_count"].astype(np.int64)
    flen = res.frames["len"].astype(np.int64)
    csum = np.concatenate([[0], np.cumsum(flen)])
    nbytes = csum[ff + fc] - csum[ff]
    fcount, rcount = fc.copy(), rc.copy()
    nxt = res.segs["next"]
    for i in np.nonzero(nxt != A.NONE)[0]:
        j = int(nxt[i])
        while j != A.NONE:
            r = res.runs[j]
            f0, fn = int(r["frame_first"]), int(r["frame_count"])
            fcount[i] += fn; rcount[i] += int(r["rec_count"]); nbytes[i] += csum[f0 + fn] - csum[f0]
            j = int(r["next"])
    return fcount, rcount, nbytes


def _joined(res, i):
    return b"".join(res.seg_frames(i))


def test_passthrough_is_the_identity_on_complete_lines(eng, workload):
    """Mode P at full size: per stream, the frames are exactly the '\\n'-terminated lines of the input, in order."""
    slot, res = _run(eng, workload, A.MODE_P)
    try:
        fcount, _, nbytes = _per_stream(res)
        n_lines = np.fromiter((b.count(b"\n") for b in workload), dtype=np.int64, count=N)
        assert np.array_equal(fcount, n_lines)
        expect = np.fromiter((b.rfind(b"\n") + 1 for b in workload), dtype=np.int64, count=N)
        assert np.array_equal(nbytes, expect)                    # unterminated tails are held back, nothing else
        total = np.fromiter((len(b) for b in workload), dtype=np.int64, count=N)
        assert np.array_equal(res.segs["carry_len"].astype(np.int64), total - expect)
        # byte identity on a stride of streams, and a checksum of checksums over them
        cin = cout = 0
        for i in range(0, N, 257):
            got = _joined(res, i)
            assert got == workload[i][:int(expect[i])]
            cin += sum(workload[i][:int(expect[i])]); cout += sum(got)
        assert cin == cout
    finally:
        eng.release(slot)


def test_reframe_accounting_and_idempotence(eng, workload):
    """Mode R at full size: every stream terminates at its finish chunk; frames == the stream's events up to it (canonical
    input: "data: X\\n\\n" re-frames to itself); one JSON_OK record per frame; re-framing the output is the identity."""
    slot, res = _run(eng, workload, R)
    try:
        assert np.all(res.segs["flags"] & A.SEG_TERMINATED)
        fcount, rcount, nbytes = _per_stream(res)
        assert np.array_equal(fcount, rcount)                      # no swallowed [DONE] before the finish chunk
        ends = np.empty(N, dtype=np.int64)                         # end of the terminating event in every input stream
        n_ev = np.empty(N, dtype=np.int64)
        for i, b in enumerate(workload):
            k = b.find(b'"finish_reason":"')
            e = b.index(b"\n\n", k) + 2
            ends[i] = e
            n_ev[i] = b.count(b"\n\n", 0, e)
        assert np.array_equal(fcount, n_ev)
        assert np.array_equal(nbytes, ends)
        sample = list(range(0, N, 129))
        outputs = []
        rflags = res.recs["flags"]
        for i in sample:
            got = _joined(res, i)
            assert got == workload[i][:int(ends[i])]               # canonical "data: X\n\n" re-frames to itself
            outputs.append(got)
            recs = res.seg_recs(i)
            assert all(rflags[r] & A.F_JSON_OK for r in recs)
            assert [bool(rflags[r] & A.F_TERMINATES) for r in recs] == [False] * (len(recs) - 1) + [True]
    finally:
        eng.release(slot)
    # idempotence: the emitted frames are canonical SSE, so feeding them back yields the same bytes
    slot, res2 = _run(eng, outputs, R)
    try:
        for j, body in enumerate(outputs):
            assert _joined(res2, j) == body
    finally:
        eng.release(slot)
