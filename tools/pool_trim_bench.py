"""Trimming a grown line pool on one GPU (DESIGN.md 4.3). Prints one JSON line.

Workload of pool_growth_bench.py: C4 where 1 % of the streams carry one extra 1 MiB single-chunk tool call, every stream cut at
seeded random positions into 8 micro-batches, mode R on an SSE_FLAG_DEFER context whose pool starts at 1/16 of the pages the
burst holds at once and may grow to --max-pages (12,000). Each rep on a fresh context:

  burst   the first --held-parts micro-batches, run to the end: the pool grows, and the 1 MiB lines cut after those
          micro-batches are held, partly received, in pages taken during the growths
  trim    sse_trim to the initial pages: host time of the call (it waits for the device and frees the old arrays), pages held
          (and moved) and capacity before and after, sse_memory_held before and after
  rest    the remaining micro-batches (no stream may fail), then a second trim with nothing held

The repack kernels' device time is read with torch.profiler (CUDA activity timestamps of sse_pool_repack_*) in a separate
rep, so that the tracer does not slow the timed ones. Steady C4 steps (the workload without the long lines) are then timed on
a fresh context and on a trimmed one, alternating. The GPU name and power limit are read in the same run.
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

from bench import build_workload   # noqa: E402
from tools.long_line_bench import PAGE, gpu_info, tool_call_line   # noqa: E402
from tools.pool_growth_bench import fill, run_step   # noqa: E402

MiB = 1 << 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5, help="C4 steps per context in the alternating comparison")
    ap.add_argument("--long-frac", type=float, default=0.01)
    ap.add_argument("--long-bytes", type=int, default=MiB)
    ap.add_argument("--pieces", type=int, default=8)
    ap.add_argument("--held-parts", type=int, default=4)
    ap.add_argument("--max-pages", type=int, default=12000)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("pool_trim_bench.py: no CUDA device")
    from inference_gateway_b200 import SseEngine, _abi as A, synth
    torch.cuda.set_device(0)
    out = {"gpu": gpu_info(), "streams": args.streams}

    bodies, _, _ = build_workload(args.streams, 0, "C4")
    mode = A.MODE_R | A.MODE_PARSE
    rng = np.random.default_rng(0x1F)
    long_idx = np.sort(rng.choice(len(bodies), size=max(1, int(args.long_frac * len(bodies))), replace=False))
    lb = list(bodies)
    for i in long_idx:
        b = lb[i]
        cut = b.find(b"\n\n") + 2
        lb[i] = b[:cut] + tool_call_line(args.long_bytes) + b[cut:]
    pieces = [synth.random_cuts(rng, b, args.pieces) for b in lb]
    parts = [[p[k] if k < len(p) else b"" for p in pieces] for k in range(args.pieces)]
    plain_pieces = [synth.random_cuts(rng, b, args.pieces) for b in bodies]
    plain_parts = [[p[k] if k < len(p) else b"" for p in plain_pieces] for k in range(args.pieces)]
    per_batch = max(sum(map(len, part)) + 16 * len(lb) for part in parts + plain_parts)
    start = max(1, (len(long_idx) * (args.long_bytes // PAGE + 1)) // 16)

    def engine():
        return SseEngine(device=0, max_conns=len(lb), bytes_per_batch=per_batch, n_slots=1, carry_slot_bytes=16384,
                         text_arena_bytes=per_batch, flags=A.FLAG_DEFER,
                         line_pool=dict(pool_pages=start, page_bytes=PAGE, max_line_bytes=2 * MiB, max_pages=args.max_pages))

    def burst_and_trim(e):
        """The burst, a timed trim, the rest, a timed second trim. Returns the rep's record."""
        e.reset_all()
        batches, dead = run_step_parts(e, parts[:args.held_parts])
        held = e.pool_stats()[0]
        cap = e.line_pool_capacity()[0]
        mem0 = e.memory_held()
        t0 = time.perf_counter()
        e.trim(start)
        trim_ms = (time.perf_counter() - t0) * 1e3
        rec = {"pages_before": cap, "pages_held_moved": held, "pages_after": e.line_pool_capacity()[0], "trim_ms": trim_ms,
               "memory_before": mem0, "memory_after": e.memory_held(), "pages_in_use_after": e.pool_stats()[0]}
        b2, d2 = run_step_parts(e, parts[args.held_parts:])
        rec["batches"], rec["dead"] = batches + b2, dead + d2
        held2 = e.pool_stats()[0]
        cap2 = e.line_pool_capacity()[0]
        mem2 = e.memory_held()
        t0 = time.perf_counter()
        e.trim(start)
        rec["second_trim"] = {"pages_before": cap2, "pages_held_moved": held2, "trim_ms": (time.perf_counter() - t0) * 1e3,
                              "memory_before": mem2, "memory_after": e.memory_held()}
        return rec

    def run_step_parts(e, ps):
        """run_step without its reset: the micro-batches ps in order, each run to the end. Returns (batches, dead segments)."""
        batches = dead = 0
        for part in ps:
            pending = list(enumerate(part))
            while pending:
                sl, arena, segs = e.acquire()
                e.submit(sl, *fill(arena, segs, pending, mode))
                res = e.collect(sl)
                flags = res.segs["flags"]
                dead += int(np.count_nonzero(flags & A.SEG_DEAD))
                pending = [(pending[i][0], pending[i][1][res.consumed(int(i)):]) for i in np.nonzero(flags & A.SEG_DEFERRED)[0]]
                e.release(sl)
                batches += 1
        return batches, dead

    reps = []
    for _ in range(args.reps):
        e = engine()
        fresh = e.memory_held()
        rec = burst_and_trim(e)
        rec["memory_fresh"] = fresh
        assert rec["dead"] == 0, rec
        reps.append(rec)
        e.close()
        torch.cuda.empty_cache()
    out["pages_start"], out["max_pages"], out["reps"] = start, args.max_pages, reps

    # the repack kernels' device time, in a rep of its own under the profiler
    from torch.profiler import ProfilerActivity, profile
    e = engine()
    e.reset_all()
    run_step_parts(e, parts[:args.held_parts])
    held, cap = e.pool_stats()[0], e.line_pool_capacity()[0]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.trim(start)
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.events():
        if "sse_pool_repack" in ev.name:
            k = "copy" if "copy" in ev.name else "chains"
            kern[k] = kern.get(k, 0.0) + ev.time_range.elapsed_us() / 1e3
    moved_bytes = held * PAGE
    out["repack"] = {"pages_before": cap, "pages_held_moved": held, "kernel_ms": kern,
                     "copy_bytes_read_and_written": 2 * moved_bytes,
                     "copy_GBps": (2 * moved_bytes / (kern["copy"] * 1e-3) / 1e9) if kern.get("copy") else None}
    e.close()
    torch.cuda.empty_cache()

    # steady C4 steps: a fresh context against a trimmed one, alternating
    fresh_e, trimmed_e = engine(), engine()
    trimmed_e.reset_all()
    run_step_parts(trimmed_e, parts)
    trimmed_e.trim(start)
    for e in (fresh_e, trimmed_e):      # warm-up
        run_step(e, plain_parts, mode, A)
    ms = {"fresh": [], "trimmed": []}
    for _ in range(args.steps):
        for name, e in (("fresh", fresh_e), ("trimmed", trimmed_e)):
            t0 = time.perf_counter()
            _, dead = run_step(e, plain_parts, mode, A)
            ms[name].append((time.perf_counter() - t0) * 1e3)
            assert dead == 0
    out["c4_steps_ms"] = ms
    out["c4_median_ms"] = {k: float(np.median(v)) for k, v in ms.items()}
    out["memory"] = {"fresh": fresh_e.memory_held(), "trimmed": trimmed_e.memory_held()}
    fresh_e.close()
    trimmed_e.close()
    out["note"] = (f"{len(long_idx)} streams with a {args.long_bytes}-byte tool call, {args.pieces} micro-batches per step, the trim "
                   f"after {args.held_parts}; one batch in flight; C4 steps include the host fill")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
