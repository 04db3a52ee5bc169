"""GPU: SSE_FLAG_COUNTERS. The counting kernels return the same results as the default ones (oracle digests, orc_check_result on
every batch), and their counters add up: produce accounting against the batch result, line-pool pages, the decode byte
identity, and the decode quantities that depend only on the lines, which must not change with the launch shape."""
import numpy as np
import pytest
import torch

from inference_gateway_b200 import SseEngine, _abi as A, synth
from inference_gateway_b200.gateway import Gateway
from tests.corpus import documents
from tests.streams import PAGE, chunk, dealt, filler_payload, long_line
from tests.util import (TARGET, check_batch, cut_bounds, decode_shape, digest_parity, digest_run, oracle_digests,
                        process_all_checked, run_pieces, shape_check)

pytestmark = pytest.mark.gpu
R, PP, P = A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE, A.MODE_P
MiB = 1 << 20
LINE_ONLY = ("d_actions", "d_action_redos", "d_unquote_jobs", "d_unquote_bytes")   # depend on the lines alone


def counting(flags=0, **kw):
    """An engine with SSE_FLAG_COUNTERS and one slot (so that an on_batch hook knows the slot: 0)."""
    kw.setdefault("n_slots", 1)
    return SseEngine(device=0, flags=A.FLAG_COUNTERS | flags, **kw)


def counter_hook(eng, bodies, bounds, got, one_job_per_span=True, on_batch=None):
    """digest_run hook: every batch's counters, checked by check_batch, appended to got."""
    def hook(b, res):
        k = eng.counters(0)
        sub = b"".join(bodies[i][bounds[i, b]:bounds[i, b + 1]] for i in range(len(bodies)))
        check_batch(k, res, sub, one_job_per_span)
        got.append(k)
        if on_batch is not None:
            on_batch(b, res)
    return hook


def counted_parity(eng, bodies, modes, bounds, label, one_job_per_span=True, on_batch=None):
    """digest_parity (oracle digests and orc_check_result per batch) collecting every batch's counters, checked by check_batch."""
    got = []
    digest_parity(eng, bodies, modes, bounds, label, on_batch=counter_hook(eng, bodies, bounds, got, one_job_per_span, on_batch))
    return got


def total(ks, name):
    return sum(k[name] for k in ks)


# ------------------------------------------------------------------ results and accounting
@pytest.mark.parametrize("name,n_streams,mode", [("C3", 16384, R), ("C4", 65536, R), ("C4", 65536, PP)])
def test_full_size_results_unchanged_and_counted(name, n_streams, mode):
    bodies = [b for b, _, _ in synth.make_config(name, n_streams=n_streams)[0]]
    nbytes = sum(map(len, bodies))
    oracle = oracle_digests(bodies, mode)
    plain = SseEngine(device=0, max_conns=n_streams, bytes_per_batch=nbytes, n_slots=1, carry_slot_bytes=16384)
    try:
        ref = {nb: digest_run(plain, bodies, mode, cut_bounds(bodies, nb, seed=700 + nb)) for nb in (1, 4)}
    finally:
        plain.close()
    eng = counting(max_conns=n_streams, bytes_per_batch=nbytes, carry_slot_bytes=16384)
    try:
        for nb in (1, 4):
            bounds = cut_bounds(bodies, nb, seed=700 + nb)
            ks = []
            got = digest_parity(eng, bodies, mode, bounds, f"{name} x{nb} counting", oracle=oracle,
                                on_batch=counter_hook(eng, bodies, bounds, ks))
            assert len(ks) == nb
            assert all(np.array_equal(x, y) for x, y in zip(got, ref[nb])), (name, nb)      # the plain engine's results
            if mode == R:                 # valid documents only (mode P|PARSE also decodes the payload of "data: [DONE]")
                assert total(ks, "d_abandoned_bytes") == 0
            assert total(ks, "d_template_lines") == 0 and total(ks, "p_long_lines") == 0
            if mode == PP:
                assert total(ks, "p_lines") == sum(b.count(b"\n") for b in bodies)
            print(f"{name} x{nb}: " + ", ".join(f"{f} {total(ks, f)}" for f in ("p_lines", "d_items", "d_warp_rounds",
                                                                                   "d_unquote_jobs", "c_total")))
    finally:
        eng.close()


@pytest.mark.parametrize("flags", [0, A.FLAG_COPY_OUT])
def test_mode_p_every_line_is_a_frame(flags):
    bodies = [b for b, _, _ in synth.make_config("C4", n_streams=2048)[0]]
    eng = counting(flags, max_conns=len(bodies), bytes_per_batch=sum(map(len, bodies)))
    try:
        ks = counted_parity(eng, bodies, P, cut_bounds(bodies, 3, seed=5), "mode P")
        for k in ks:
            assert k["p_frames_zero_copy"] + k["p_frames_materialised"] == k["p_lines"]
            assert k["d_items"] == 0 and k["p_items"] == 0
            if flags & A.FLAG_COPY_OUT:
                assert k["p_frames_zero_copy"] == 0
    finally:
        eng.close()


def test_copy_out_materialises_every_frame():
    bodies = [b for b, _, _ in synth.make_config("C4", n_streams=2048)[0]]
    eng = counting(A.FLAG_COPY_OUT, max_conns=len(bodies), bytes_per_batch=sum(map(len, bodies)))
    try:
        ks = counted_parity(eng, bodies, R, cut_bounds(bodies, 2, seed=6), "copy-out")
        assert all(k["p_frames_zero_copy"] == 0 for k in ks) and total(ks, "p_frames_materialised") > 0
    finally:
        eng.close()


# ------------------------------------------------------------------ long lines and the pool
def test_long_lines_and_pool_pages():
    """Every line is either at most 1 KiB or at least 64 KiB: p_long_lines counts exactly the long ones, and over a run in
    which every pooled line completes the pool's pages all come back."""
    rng = np.random.default_rng(11)
    bodies, n_long = [], 0
    for i in range(96):
        body = chunk(b"Hello") + chunk(b"x" * int(rng.integers(1, 900)))
        if i % 3 == 0:
            n = int(rng.choice([64 * 1024, 100_000, 300_000, MiB]))
            body += long_line(("content", "toolcall", "crlf")[i % 9 // 3], n, rng) + b"\n"
            n_long += 1
        bodies.append(body + chunk(b"bye") + b"data: [DONE]\n\n")
    modes = [(P, PP)[i % 2] for i in range(len(bodies))]
    eng = counting(max_conns=128, bytes_per_batch=40 * MiB, carry_slot_bytes=32768, text_arena_bytes=40 * MiB,
                   line_pool=dict(pool_pages=1024, page_bytes=PAGE))
    try:
        for nb in (1, 5):
            pieces = [synth.random_cuts(np.random.default_rng(nb * 1000 + i), b, nb) for i, b in enumerate(bodies)]
            ks = []
            orig = eng.collect

            def collect(slot):
                res = orig(slot)
                k = eng.counters(slot)
                check_batch(k, res)
                ks.append(k)
                return res
            eng.collect = collect
            try:
                run_pieces(eng, pieces, modes)
            finally:
                del eng.collect
            assert total(ks, "p_long_lines") == n_long, nb
            assert total(ks, "p_lines") == sum(b.count(b"\n") for b in bodies)
            taken, returned = total(ks, "p_pool_pages_taken"), total(ks, "p_pool_pages_returned")
            assert taken == returned and taken > 0, (taken, returned)
            assert eng.pool_stats()[0] == 0
    finally:
        eng.close()


# ------------------------------------------------------------------ the decode quantities that depend on the lines alone
def test_line_quantities_do_not_depend_on_the_launch_shape():
    """k(docs + fillers) - k(fillers) in the 8-, 16- and 32-item shapes, k(docs) twice, and k(docs) on the copy-out engine
    agree in every LINE_ONLY counter (the counters are sums over lines)."""
    sm_count = torch.cuda.get_device_properties(0).multi_processor_count
    docs = documents() + [b'{"choices":[{"index":0,"delta":{"content":"line %d\\n\\"quoted\\""}}]}' % i for i in range(64)] + [
        b'{"choices":[{"index":0,"delta":{"tool_calls":[{"index":0,"id":"c%d","function":{"arguments":"{\\"n\\":%d}"}}]}}]}' % (i, i)
        for i in range(64)]
    assert decode_shape(len(docs), sm_count) == 8

    def run(eng, payloads, label, shape=None):
        bodies, bounds, _ = dealt([payloads])
        log = []
        hook = shape_check(eng, sm_count, shape, log) if shape else None
        ks = counted_parity(eng, bodies, PP, bounds, label, on_batch=hook)
        assert len(ks) == 1
        return ks[0]

    eng = counting(max_conns=8192, bytes_per_batch=96 << 20)
    try:
        alone = [run(eng, docs, "docs"), run(eng, docs, "docs again")]
        rng = np.random.default_rng(9)
        for shape in (8, 16, 32):
            n_fill = int(TARGET[shape] * sm_count * 32) - len(docs)
            fill = [filler_payload("strings" if i % 2 else "nostring", int(n)) for i, n in enumerate(rng.integers(40, 700, n_fill))]
            with_docs = run(eng, docs + fill, f"docs in the {shape}-item shape", shape)
            fill_only = run(eng, fill, f"fillers of the {shape}-item shape")
            alone.append({f: with_docs[f] - fill_only[f] for f in LINE_ONLY})
    finally:
        eng.close()
    eng = counting(A.FLAG_COPY_OUT, max_conns=8192, bytes_per_batch=96 << 20)
    try:
        alone.append(run(eng, docs, "docs, copy-out"))
    finally:
        eng.close()
    for f in LINE_ONLY:
        assert len({k[f] for k in alone}) == 1, (f, [k[f] for k in alone])
    assert alone[0]["d_actions"] > 0 and alone[0]["d_unquote_jobs"] > 0


def test_invalid_documents_count_their_abandoned_bytes():
    docs = [b'{"choices":[{"delta":{"content":"ok"}}]} trailing', b'{"choices":[' + b"[" * 200 + b"]" * 200 + b"]}",
            b'{"choices":[{"delta":{"content":"a"}}]', b"nope nope nope"]
    bodies, bounds, _ = dealt([docs * 8])
    eng = counting(max_conns=8192, bytes_per_batch=4 * MiB)
    try:
        ks = counted_parity(eng, bodies, PP, bounds, "invalid documents")
        assert total(ks, "d_abandoned_bytes") > 0
    finally:
        eng.close()


# ------------------------------------------------------------------ deferral, templates, the gateway
def test_deferred_decode_pass_is_the_one_counted():
    """The text arena is cut below what one batch needs: the batch is decoded a second time after the arena grew, and the
    decode counters describe that pass."""
    rng = np.random.default_rng(4)
    bodies = [b"".join(chunk(b"line\\n" * int(rng.integers(20, 200))) for _ in range(6)) for _ in range(48)]
    eng = counting(A.FLAG_DEFER, max_conns=64, bytes_per_batch=1 * MiB, text_arena_bytes=4096)
    try:
        passes = []

        def on_batch(res, conns):
            k = eng.counters(0)
            check_batch(k, res)
            passes.append(k["decode_passes"])
        process_all_checked(eng, [(i, R, b) for i, b in enumerate(bodies)], on_batch)
        assert passes[0] == 2, passes
    finally:
        eng.close()


def test_templates_count_their_lines_in_the_byte_identity():
    streams, _ = synth.make_config("C4", n_streams=4096)
    bodies = [b for b, _, _ in streams]
    eng = counting(A.FLAG_TEMPLATES, max_conns=len(bodies), bytes_per_batch=sum(map(len, bodies)))
    try:
        ks = counted_parity(eng, bodies, R, cut_bounds(bodies, 4, seed=8), "templates", one_job_per_span=False)
        assert total(ks, "d_template_lines") > 0 and total(ks, "d_template_bytes") > 0
    finally:
        eng.close()


def test_gateway_sums_the_lines_it_delivered():
    cfg = A.Config()
    A.load().sse_worst_case_config(cfg, 64, 1 << 20)
    cfg.flags = A.FLAG_COUNTERS
    g = Gateway(device=0, config=cfg)
    try:
        bodies = [b for b, _, _ in synth.make_config("C4", n_streams=48)[0]]
        sids = [g.stream_chat_completions(P) for _ in bodies]
        for sid, b in zip(sids, bodies):
            for i in range(0, len(b), 777):
                assert g.upstream_write(sid, b[i:i + 777]) == len(b[i:i + 777])
                g.pump()
            g.upstream_close(sid)
        g.pump()
        delivered = 0
        for sid in sids:
            while True:
                try:
                    fr = g.recv(sid)
                except EOFError:
                    break
                if fr is None:
                    break
                delivered += 1
        k = g.counters()
        assert k["p_lines"] == delivered == sum(b.count(b"\n") for b in bodies)
        assert k["p_segments"] > 0 and k["d_items"] == 0
    finally:
        g.close()
    plain = Gateway(device=0, max_conns=4)
    try:
        with pytest.raises(A.SseError) as e:
            plain.counters()
        assert e.value.status == A.SSE_ERR_ARG
    finally:
        plain.close()


def test_counters_read_states():
    eng = counting(max_conns=4, bytes_per_batch=MiB)
    plain = SseEngine(device=0, max_conns=4, bytes_per_batch=MiB)
    try:
        slot, arena, segs = eng.acquire()
        with pytest.raises(A.SseError) as e:       # nothing collected yet
            eng.counters(slot)
        assert e.value.status == A.SSE_ERR_BUSY
        n, nb = eng.fill(arena, segs, [(0, R, chunk(b"hi"))])
        eng.submit(slot, n, nb)
        with pytest.raises(A.SseError) as e:       # submitted, not collected
            eng.counters(slot)
        assert e.value.status == A.SSE_ERR_BUSY
        res = eng.collect(slot)
        check_batch(eng.counters(slot), res)
        eng.release(slot)
        with pytest.raises(A.SseError) as e:
            eng.counters(slot)
        assert e.value.status == A.SSE_ERR_BUSY
        ps, pres = plain.process([(0, R, chunk(b"hi"))])
        with pytest.raises(A.SseError) as e:       # a context without the flag
            plain.counters(ps)
        assert e.value.status == A.SSE_ERR_ARG
        plain.release(ps)
    finally:
        eng.close()
        plain.close()
