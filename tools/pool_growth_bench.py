"""Line-pool growth on one GPU (DESIGN.md 4.3). Prints one JSON line.

Workload of long_line_bench.py (b): C4 where 1 % of the streams carry one extra 1 MiB single-chunk tool call, every stream cut at
seeded random positions into 8 micro-batches. A step feeds the 8 micro-batches through sse_submit / sse_collect (one batch in
flight) on an SSE_FLAG_DEFER context, submitting every deferred rest again before the next micro-batch, from sse_reset_all.

  sized   a pool sized up front (long_line_bench.py's page count): its page high-water mark H is measured here
  grown   a pool of H / 16 pages that may grow to --max-pages (12,000): a fresh context per repetition, so every repetition
          grows from the small pool in its first step; then the same steps as `sized` on the grown pool

Reported: growth events (pages before and after) and the cost of each: the host time of the sse_collect that grew the pool plus
the wait for the copy it queued (sse_line_pool_stats is ordered after it), less the median of the same two calls for batches
that did not grow; extra batches the deferrals cost in the first step; the first step's time and the steady step time of both
pools (a batch that defers for want of out-arena room also adds a batch, on both pools). The GPU name, power limit and SM clocks are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import build_workload   # noqa: E402
from tools.long_line_bench import PAGE, gpu_info, tool_call_line   # noqa: E402

MiB = 1 << 20


def clocks():
    q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def fill(arena, segs, items, mode):
    """items: [(conn, bytes)] -> one segment each, 16-byte aligned. Returns (n_segs, in_bytes)."""
    n = len(items)
    lens = np.fromiter((len(b) for _, b in items), dtype=np.int64, count=n)
    aligned = (lens + 15) & ~15
    offs = np.zeros(n, dtype=np.int64)
    offs[1:] = np.cumsum(aligned)[:-1]
    for (_, b), o in zip(items, offs):
        if b:
            arena[o:o + len(b)] = np.frombuffer(b, dtype=np.uint8)
    segs["conn"][:n] = np.fromiter((c for c, _ in items), dtype=np.uint32, count=n)
    segs["in_off"][:n] = offs
    segs["in_len"][:n] = lens
    segs["mode"][:n] = mode
    segs["provider"][:n] = segs["conn"][:n] % 4
    segs["reserved"][:n] = 0
    return n, int(offs[-1] + aligned[-1]) if n else 0


def run_step(e, parts, mode, A, growth_log=None, plain_log=None):
    """One step: the micro-batches in order, each run to the end. Returns (batches, dead segments)."""
    e.reset_all()
    batches = dead = 0
    for part in parts:
        pending = [(c, b) for c, b in enumerate(part)]
        while pending:
            sl, arena, segs = e.acquire()
            ns, nb = fill(arena, segs, pending, mode)
            e.submit(sl, ns, nb)
            before = e.line_pool_capacity()[0]
            t0 = time.perf_counter()
            res = e.collect(sl)
            e.pool_stats()          # ordered after the growth the collect queued: its copy is done
            dt = (time.perf_counter() - t0) * 1e3
            after = e.line_pool_capacity()[0]
            if after != before and growth_log is not None:
                growth_log.append({"pages_before": before, "pages_after": after, "collect_ms": dt})
            elif plain_log is not None:
                plain_log.append(dt)
            flags = res.segs["flags"]
            dead += int(np.count_nonzero(flags & A.SEG_DEAD))
            left = []
            for i in np.nonzero(flags & A.SEG_DEFERRED)[0]:
                c, b = pending[i]
                left.append((c, b[res.consumed(int(i)):]))
            e.release(sl)
            pending = left
            batches += 1
    return batches, dead


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--long-frac", type=float, default=0.01)
    ap.add_argument("--long-bytes", type=int, default=MiB)
    ap.add_argument("--pieces", type=int, default=8)
    ap.add_argument("--max-pages", type=int, default=12000)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("pool_growth_bench.py: no CUDA device")
    from inference_gateway_b200 import SseEngine, _abi as A, synth
    torch.cuda.set_device(0)
    out = {"gpu": gpu_info(), "clocks_sm_before": clocks(), "streams": args.streams}

    bodies, mode, _ = build_workload(args.streams, 0, "C4")
    rng = np.random.default_rng(0x1F)
    long_idx = np.sort(rng.choice(len(bodies), size=max(1, int(args.long_frac * len(bodies))), replace=False))
    lb = list(bodies)
    for i in long_idx:
        b = lb[i]
        cut = b.find(b"\n\n") + 2
        lb[i] = b[:cut] + tool_call_line(args.long_bytes) + b[cut:]
    pieces = [synth.random_cuts(rng, b, args.pieces) for b in lb]
    parts = [[p[k] if k < len(p) else b"" for p in pieces] for k in range(args.pieces)]
    per_batch = max(sum(map(len, part)) + 16 * len(lb) for part in parts)
    sized_pages = (len(long_idx) * args.long_bytes + len(long_idx) * (PAGE + 16384)) // PAGE + 64

    def engine(pages, max_pages):
        return SseEngine(device=0, max_conns=len(lb), bytes_per_batch=per_batch, n_slots=1, carry_slot_bytes=16384,
                         text_arena_bytes=per_batch, flags=A.FLAG_DEFER,
                         line_pool=dict(pool_pages=pages, page_bytes=PAGE, max_line_bytes=2 * MiB, max_pages=max_pages))

    def steady(e):
        ms, nbs = [], []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            nb, dead = run_step(e, parts, mode, A)
            ms.append((time.perf_counter() - t0) * 1e3)
            nbs.append(nb)
            assert dead == 0, dead
        return {"ms_per_step": ms, "batches_per_step": nbs}

    # ---- sized: the high-water mark and the steady step
    e = engine(sized_pages, 0)
    t0 = time.perf_counter()
    nb, dead = run_step(e, parts, mode, A)
    sized_first = (time.perf_counter() - t0) * 1e3
    hw = e.pool_stats()[1]
    sized_ms = steady(e)
    e.close()
    torch.cuda.empty_cache()
    out["sized"] = {"pages": sized_pages, "pages_high_water": hw, "first_step_ms": sized_first, "batches": nb, "dead": dead,
                    "steady": sized_ms}

    # ---- grown: from high-water / 16
    start = max(1, hw // 16)
    reps = []
    for r in range(args.reps):
        e = engine(start, args.max_pages)
        grow, plain = [], []
        t0 = time.perf_counter()
        nb, dead = run_step(e, parts, mode, A, grow, plain)
        first = (time.perf_counter() - t0) * 1e3
        med = float(np.median(plain)) if plain else 0.0
        for g in grow:
            g["cost_ms"] = g["collect_ms"] - med
        rep = {"first_step_ms": first, "batches": nb, "extra_batches": nb - out["sized"]["batches"], "dead": dead,
               "growth_events": grow, "median_plain_collect_ms": med, "pages_final": e.line_pool_capacity()[0],
               "pages_high_water": e.pool_stats()[1]}
        if r == 0:
            rep["steady_after_growth"] = steady(e)
        reps.append(rep)
        e.close()
        torch.cuda.empty_cache()
    out["grown"] = {"pages_start": start, "max_pages": args.max_pages, "reps": reps}
    out["clocks_sm_after"] = clocks()
    out["note"] = (f"{len(long_idx)} streams with a {args.long_bytes}-byte tool call, {args.pieces} micro-batches per step, "
                   f"one batch in flight, host fill included in step times")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
