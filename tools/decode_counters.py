#!/usr/bin/env python3
"""Where the produce and decode kernels spend their work (SSE_FLAG_COUNTERS), on the workloads DESIGN.md 4.3 measures:

  c4        C4 (65,536 streams), whole bodies in one launch
  c4x4      C4 cut at seeded random positions into 4 micro-batches (a step = 4 launches)
  c3        C3 (16,384 streams) in one launch
  tick      one steady-state tick: one SSE event per connection (tools/tick_bench.py's batch)
  long      C4 with 1 % of the streams carrying one 1 MiB tool call, 8 micro-batches, line pool (tools/long_line_bench.py's (b))

For each workload: the counters of one step (summed over its launches) as JSON in --out, per-item means on stdout, and the time
of a step on the default engine and on the counting engine, alternating in this run after warm-up (CUDA events), so that the
counting build's overhead is known. The cycle shares come from the counting build: they show how its decode time divides, not
the default kernel's time. The GPU name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import build_workload, fill_slot, time_steps   # noqa: E402
from tools.long_line_bench import PAGE, gpu_info, tool_call_line   # noqa: E402

MiB = 1 << 20
BUCKETS = ("c_pull", "c_skip", "c_coop", "c_steps", "c_finish", "c_unquote")
MECHANISMS = ("d_skip_bytes", "d_coop_bytes", "d_plain_steps", "d_actions", "d_abandoned_bytes", "d_template_bytes")


def workloads(args):
    """name -> (parts, mode, engine keyword arguments): parts[k] is the list of bodies launch k of a step carries."""
    from inference_gateway_b200 import synth
    bodies, mode, _ = build_workload(args.streams, 0, "C4")
    rng = np.random.default_rng(0x5EED)
    out = {"c4": ([bodies], mode, {})}
    pieces = [synth.random_cuts(rng, b, 4) for b in bodies]
    out["c4x4"] = ([[p[k] if k < len(p) else b"" for p in pieces] for k in range(4)], mode, {})
    c3, c3_mode, _ = build_workload(args.streams // 4, 0, "C3")
    out["c3"] = ([c3], c3_mode, {})
    streams, tick_mode = synth.make_config("C4", n_streams=args.streams)
    evs = [[e + b"\n\n" for e in b.split(b"\n\n") if e] for b, _, _ in streams]
    out["tick"] = ([[ev[2] for ev in evs if len(ev) > 2]], tick_mode, {})
    long_idx = np.sort(np.random.default_rng(0x1F).choice(len(bodies), size=max(1, len(bodies) // 100), replace=False))
    lb = list(bodies)
    for i in long_idx:
        cut = lb[i].find(b"\n\n") + 2
        lb[i] = lb[i][:cut] + tool_call_line(MiB) + lb[i][cut:]
    pieces = [synth.random_cuts(rng, b, 8) for b in lb]
    parts = [[p[k] if k < len(p) else b"" for p in pieces] for k in range(8)]
    per_batch = max(sum(map(len, part)) + 16 * len(lb) for part in parts)
    pages = (len(long_idx) * (MiB + PAGE + 16384)) // PAGE + 64
    out["long"] = (parts, mode, dict(text_arena_bytes=per_batch, line_pool=dict(pool_pages=pages, page_bytes=PAGE)))
    return out


def per_item(k: dict) -> dict:
    """Means per decoded item (lane-rounds, bytes per mechanism, actions, unquote jobs) and the cycle shares."""
    items = max(k["d_items"], 1)
    lane_rounds = 32 * k["d_warp_rounds"]
    payload = sum(k[m] for m in MECHANISMS)
    m = {"items": k["d_items"], "payload_bytes_per_item": payload / items,
         "warp_rounds_per_pull": k["d_warp_rounds"] / max(k["d_pulls"], 1),
         "lane_rounds_per_item": lane_rounds / items,
         "busy_lane_share": k["d_busy_lane_rounds"] / max(lane_rounds, 1),
         "actions_per_item": k["d_actions"] / items, "redos_per_item": k["d_action_redos"] / items,
         "unquote_jobs_per_item": k["d_unquote_jobs"] / items, "unquote_bytes_per_item": k["d_unquote_bytes"] / items,
         "coop_strings_per_item": k["d_coop_strings"] / items, "items_per_pull": k["d_items_per_pull"]}
    for name in MECHANISMS:
        m["share_" + name[2:]] = k[name] / max(payload, 1)
    tot = max(k["c_total"], 1)
    for b in BUCKETS:
        m[b + "_share"] = k[b] / tot
    m["c_other_share"] = 1.0 - sum(k[b] for b in BUCKETS) / tot
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", default="", help="comma-separated workload names (default: all)")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "decode_counters"),
                    help="directory for the JSON of each workload and summary.json")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("decode_counters.py: no CUDA device")
    from inference_gateway_b200 import SseEngine, _abi as A
    torch.cuda.set_device(0)
    tstream = torch.cuda.Stream()
    torch.cuda.set_stream(tstream)
    stream = tstream.cuda_stream
    os.makedirs(args.out, exist_ok=True)
    gpu = gpu_info()
    summary = {"gpu": gpu, "steps": args.steps, "reps": args.reps}

    for name, (parts, mode, kw) in workloads(args).items():
        if args.only and name not in args.only.split(","):
            continue
        n_conns = max(len(p) for p in parts)
        per_batch = max(sum(map(len, p)) + 16 * len(p) for p in parts) + 64

        def engine(flags):
            e = SseEngine(device=0, max_conns=n_conns, bytes_per_batch=per_batch, n_slots=len(parts), carry_slot_bytes=16384,
                          flags=flags, **kw)
            meta = []
            for p in parts:
                sl, arena, segs = e.acquire()
                ns, nb, _ = fill_slot(e, arena, segs, p, mode)
                segs["provider"][:ns] = np.arange(ns) % 4
                e.upload(sl, ns, nb, stream)
                meta.append((sl, ns))

            def step(_i):
                e.reset_all(stream)
                for sl, ns in meta:
                    e.launch(sl, ns, stream)
            for i in range(3):
                step(i)
            torch.cuda.synchronize()
            return e, meta, step

        engines = {"default": engine(0), "counting": engine(A.FLAG_COUNTERS)}
        ms = {k: [] for k in engines}
        for _ in range(args.reps):
            for k, (_, _, step) in engines.items():
                ms[k].append(time_steps(torch, step, args.steps) / args.steps)
        # one more step of the counting engine, then its counters, summed over the step's launches
        e, meta, step = engines["counting"]
        step(0)
        total = None
        frames = {}
        for sl, _ in meta:
            res = e.download(sl, stream)
            frames[sl] = int(res.raw.n_frames)
            k = e.counters(sl)
            total = k if total is None else {f: total[f] + k[f] for f in k}
        total["d_items_per_pull"] = k["d_items_per_pull"]       # the last launch's choice, not a sum
        d, dmeta, dstep = engines["default"]
        dstep(0)
        same = all(int(d.download(sl, stream).raw.n_frames) == frames[sl] for sl, _ in dmeta)
        for eng, _, _ in engines.values():
            eng.close()
        torch.cuda.empty_cache()
        rec = {"workload": name, "gpu": gpu, "launches_per_step": len(parts), "streams": n_conns,
               "ms_per_step_default": ms["default"], "ms_per_step_counting": ms["counting"],
               "counting_overhead": min(ms["counting"]) / min(ms["default"]) - 1.0, "frames_match": same,
               "counters": total, "per_item": per_item(total)}
        with open(os.path.join(args.out, name + ".json"), "w") as f:
            json.dump(rec, f, indent=1)
        summary[name] = {"ms_default": min(ms["default"]), "ms_counting": min(ms["counting"]),
                         "overhead": rec["counting_overhead"], "per_item": rec["per_item"]}
        pi = rec["per_item"]
        print(f"[{name}] {gpu}: default {min(ms['default']):.3f} ms, counting {min(ms['counting']):.3f} ms "
              f"({rec['counting_overhead']:+.0%}); {pi['items']} items, {pi['payload_bytes_per_item']:.0f} B/item, "
              f"{pi['lane_rounds_per_item']:.1f} lane-rounds/item, busy {pi['busy_lane_share']:.0%}; bytes: "
              + ", ".join(f"{m[2:]} {pi['share_' + m[2:]]:.0%}" for m in MECHANISMS)
              + f"; {pi['actions_per_item']:.1f} actions, {pi['unquote_jobs_per_item']:.2f} unquote jobs/item; cycles: "
              + ", ".join(f"{b[2:]} {pi[b + '_share']:.0%}" for b in BUCKETS) + f", other {pi['c_other_share']:.0%}",
              flush=True)
    with open(os.path.join(args.out, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
