"""SSE_FLAG_DEFER measurements on one GPU (DESIGN.md 4.3). Prints one JSON line.

(a) no_overflow   C4 (65,536 streams) in one device-resident launch per step with the default config, without and with
                  SSE_FLAG_DEFER, when nothing overflows: what the deferral path costs when it is not taken. The two engines
                  alternate, --reps rounds each; CUDA events around --steps steps.
(b) half_produce  C4 with max_frames, max_recs and out_arena_bytes cut to half of what one step needs: a step submits every
                  stream and then the deferred remainders until every byte was taken (host driver included: fill, submit,
                  collect). Reports the batches per step and the step time, next to the same driver on the default config
                  (one batch per step).
(c) regrow        C4 with text_arena_bytes cut to half of what a step needs: the first step of a fresh engine grows the slot's
                  text arena and decodes the batch again; later steps fit. Host clock around launch + download (which ends in
                  a synchronise), per step.

The GPU name and power limit are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import build_workload, fill_slot, time_steps   # noqa: E402
from tools.long_line_bench import gpu_info                # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--drain-steps", type=int, default=5)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("defer_bench.py: no CUDA device")
    from inference_gateway_b200 import SseEngine, _abi as A
    torch.cuda.set_device(0)
    tstream = torch.cuda.Stream()
    torch.cuda.set_stream(tstream)
    stream = tstream.cuda_stream
    out = {"gpu": gpu_info(), "streams": args.streams}

    bodies, mode, _ = build_workload(args.streams, 0, "C4")
    in_payload = sum(map(len, bodies))
    base = dict(device=0, max_conns=len(bodies), bytes_per_batch=in_payload, n_slots=1, carry_slot_bytes=16384)

    # ---- (a) the flag on a batch that fits
    def one_launch_engine(flags, **caps):
        e = SseEngine(flags=flags, **base, **caps)
        sl, arena, segs = e.acquire()
        ns, nb, _ = fill_slot(e, arena, segs, bodies, mode)
        e.upload(sl, ns, nb, stream)

        def step(_i):
            e.reset_all(stream)
            e.launch(sl, ns, stream)
        for i in range(3):
            step(i)
        torch.cuda.synchronize()
        return e, sl, ns, step

    engines = {"off": one_launch_engine(0), "defer": one_launch_engine(A.FLAG_DEFER)}
    ms = {k: [] for k in engines}
    for _ in range(args.reps):
        for k, (_, _, _, step) in engines.items():
            ms[k].append(time_steps(torch, step, args.steps) / args.steps)
    need = {}
    for k, (e, sl, _, _) in engines.items():
        res = e.download(sl, stream)
        need[k] = dict(frames=int(res.raw.n_frames), recs=int(res.raw.n_recs), out=int(res.raw.out_bytes),
                       text=int(res.raw.text_bytes), overflow=res.overflow)
        e.close()
    out["no_overflow"] = {"ms_per_step_off": ms["off"], "ms_per_step_defer": ms["defer"], "results": need,
                          "note": f"one launch per step, {args.reps} alternating rounds of {args.steps} steps"}
    torch.cuda.empty_cache()
    n = need["off"]

    # ---- (b) produce-side capacities at half of one step's need: deferred remainders are submitted until drained
    def drain_step(e):
        data = list(bodies)
        pending = np.arange(len(bodies))
        batches = 0
        while len(pending):
            sl, arena, segs = e.acquire()
            ns, nb, _ = fill_slot(e, arena, segs, [data[c] for c in pending], mode)
            segs["conn"][:ns] = pending.astype(np.uint32)
            e.submit(sl, ns, nb)
            res = e.collect(sl)
            d = np.nonzero(res.segs["flags"] & A.SEG_DEFERRED)[0]
            cons = res.segs["consumed"][d].astype(np.int64)
            e.release(sl)
            for i, k in zip(d, cons):
                data[pending[i]] = data[pending[i]][k:]
            pending = pending[d]
            batches += 1
        return batches

    def drain_run(e):
        e.reset_all()
        drain_step(e)                                             # warm-up
        times, batches = [], []
        for _ in range(args.drain_steps):
            e.reset_all()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            batches.append(drain_step(e))
            times.append((time.perf_counter() - t0) * 1e3)
        return times, batches

    half = dict(max_frames=max(64, n["frames"] // 2), max_recs=max(64, n["recs"] // 2), out_arena_bytes=max(1 << 20, n["out"] // 2))
    runs = {}
    for k, caps in (("default", {}), ("half", half)):
        e = SseEngine(flags=A.FLAG_DEFER, **base, **caps)
        t, b = drain_run(e)
        runs[k] = {"ms_per_step": t, "batches_per_step": b}
        e.close()
        torch.cuda.empty_cache()
    out["half_produce"] = {"caps": half, **runs,
                           "note": "host driver included (fill_slot, sse_submit, sse_collect, remainders); a step ends when every "
                                   "byte of every stream was taken"}

    # ---- (c) one decode-side growth: the second decode pass
    first, steady = [], []
    text_half = max(4096, n["text"] // 2)
    for _ in range(3):
        e = SseEngine(flags=A.FLAG_DEFER, text_arena_bytes=text_half, **base)
        sl, arena, segs = e.acquire()
        ns, nb, _ = fill_slot(e, arena, segs, bodies, mode)
        e.upload(sl, ns, nb, stream)
        ovf = []
        for i in range(4):
            e.reset_all(stream)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            e.launch(sl, ns, stream)
            res = e.download(sl, stream)
            (first if i == 0 else steady).append((time.perf_counter() - t0) * 1e3)
            ovf.append(res.overflow)
        assert ovf[0] & A.OVF_TEXT and not any(ovf[1:]), ovf
        e.close()
        torch.cuda.empty_cache()
    out["regrow"] = {"text_arena_bytes": text_half, "text_needed": n["text"], "ms_first_step": first, "ms_steady_step": steady,
                     "note": "fresh engine per row; the first step grows the text arena (cudaMalloc + cudaHostAlloc) and decodes "
                             "again; launch + download, host clock"}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
