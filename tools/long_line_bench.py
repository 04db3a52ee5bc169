"""Line-pool measurements on one GPU (DESIGN.md 4.3). Prints one JSON line.

(a) pool_cost   C4 (65,536 streams) in one device-resident launch per step, without a line pool and with a pool that no line
                uses: what enabling the pool costs. The two engines alternate, --reps rounds each.
(b) long_lines  C4 where 1 % of the streams carry one extra 1 MiB single-chunk tool call, every stream cut at seeded random
                positions into 8 micro-batches (a step = 8 launches): ms per step, pooled bytes per second (bytes of the
                long lines over step time) and the pool's page high-water mark.

The GPU name and power limit are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import build_workload, fill_slot, time_steps   # noqa: E402

MiB = 1 << 20
PAGE = 65536


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def tool_call_line(n: int) -> bytes:
    pre = b'data: {"choices":[{"index":0,"delta":{"tool_calls":[{"index":0,"id":"call_w","type":"function","function":{"name":"write_file","arguments":"'
    post = b'"}}]},"finish_reason":null}]}\n\n'
    unit = b"line of the file\\n"
    k = n - len(pre) - len(post)
    return pre + (unit * (k // len(unit) + 1))[:k] + post


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--long-frac", type=float, default=0.01)
    ap.add_argument("--long-bytes", type=int, default=MiB)
    ap.add_argument("--pieces", type=int, default=8)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("long_line_bench.py: no CUDA device")
    from inference_gateway_b200 import SseEngine, _abi as A, synth
    torch.cuda.set_device(0)
    tstream = torch.cuda.Stream()
    torch.cuda.set_stream(tstream)
    stream = tstream.cuda_stream
    out = {"gpu": gpu_info(), "streams": args.streams}

    bodies, mode, _ = build_workload(args.streams, 0, "C4")
    in_payload = sum(map(len, bodies))

    # ---- (a) pool off vs. pool on and unused
    def one_launch_engine(pool):
        e = SseEngine(device=0, max_conns=len(bodies), bytes_per_batch=in_payload, n_slots=1, carry_slot_bytes=16384, line_pool=pool)
        sl, arena, segs = e.acquire()
        ns, nb, _ = fill_slot(e, arena, segs, bodies, mode)
        e.upload(sl, ns, nb, stream)

        def step(_i):
            e.reset_all(stream)
            e.launch(sl, ns, stream)
        for i in range(3):
            step(i)
        torch.cuda.synchronize()
        return e, sl, step

    engines = {"off": one_launch_engine(None), "on_unused": one_launch_engine(dict(pool_pages=1024, page_bytes=PAGE))}
    ms = {k: [] for k in engines}
    for _ in range(args.reps):
        for k, (_, _, step) in engines.items():
            ms[k].append(time_steps(torch, step, args.steps) / args.steps)
    for k, (e, sl, _) in engines.items():
        res = e.download(sl, stream)
        ms[k + "_frames"] = int(res.raw.n_frames)
        if k == "on_unused":
            ms["pages_high_water"] = e.pool_stats()[1]
        e.close()
    out["pool_cost"] = {"ms_per_step_off": ms["off"], "ms_per_step_on_unused": ms["on_unused"],
                        "frames_off": ms["off_frames"], "frames_on_unused": ms["on_unused_frames"],
                        "pages_high_water": ms["pages_high_water"],
                        "note": f"one launch per step, {args.reps} alternating rounds of {args.steps} steps; pool 1024 x 64 KiB"}
    del engines
    torch.cuda.empty_cache()

    # ---- (b) 1 % of the streams carry one long single-chunk tool call, 8 micro-batches
    rng = np.random.default_rng(0x1F)
    long_idx = np.sort(rng.choice(len(bodies), size=max(1, int(args.long_frac * len(bodies))), replace=False))
    lb = list(bodies)
    for i in long_idx:
        b = lb[i]
        cut = b.find(b"\n\n") + 2
        lb[i] = b[:cut] + tool_call_line(args.long_bytes) + b[cut:]
    pooled_bytes = len(long_idx) * args.long_bytes
    pieces = [synth.random_cuts(rng, b, args.pieces) for b in lb]
    parts = [[p[k] if k < len(p) else b"" for p in pieces] for k in range(args.pieces)]
    per_batch = max(sum(map(len, part)) + 16 * len(lb) for part in parts)
    pages = (pooled_bytes + len(long_idx) * (PAGE + 16384)) // PAGE + 64

    def long_lines(run_mode):
        # nearly every long line ends in the last piece, so one batch decodes all of their arguments: the default text arena
        # (a quarter of the input) is sized for realistic traffic, not for this; one text byte per input byte covers it
        e = SseEngine(device=0, max_conns=len(lb), bytes_per_batch=per_batch, n_slots=args.pieces, carry_slot_bytes=16384,
                      text_arena_bytes=per_batch, line_pool=dict(pool_pages=pages, page_bytes=PAGE))
        meta = []
        for k in range(args.pieces):
            sl, arena, segs = e.acquire()
            ns, nb, _ = fill_slot(e, arena, segs, parts[k], run_mode)
            e.upload(sl, ns, nb, stream)
            meta.append((sl, ns))
        torch.cuda.synchronize()

        def seg_step(_i):
            e.reset_all(stream)
            for sl, ns in meta:
                e.launch(sl, ns, stream)

        for i in range(3):
            seg_step(i)
        torch.cuda.synchronize()
        dead = 0
        for sl, _ in meta:    # the last warm-up step: no stream may have failed
            res = e.download(sl, stream)
            dead += int(np.count_nonzero(res.segs["flags"] & A.SEG_DEAD))
        hw = e.pool_stats()[1]
        # per launch: which piece (micro-batch) takes the time
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in meta]
        e.reset_all(stream)
        for (a, b), (sl, ns) in zip(evs, meta):
            a.record(); e.launch(sl, ns, stream); b.record()
        torch.cuda.synchronize()
        per_piece = [a.elapsed_time(b) for a, b in evs]
        step_ms = [time_steps(torch, seg_step, args.steps) / args.steps for _ in range(args.reps)]
        e.close()
        torch.cuda.empty_cache()
        return {"mode": run_mode, "ms_per_step": step_ms, "ms_per_piece": per_piece,
                "pooled_bytes_per_s": pooled_bytes / (min(step_ms) / 1e3), "pages_high_water": hw, "dead_streams": dead}

    out["long_lines"] = {"long_streams": int(len(long_idx)), "long_line_bytes": args.long_bytes, "pieces": args.pieces,
                         "pool_pages": pages, "runs": [long_lines(mode), long_lines(0)],
                         "note": "a step = reset + one launch per piece; pooled_bytes_per_s = long-line bytes / fastest step; "
                                 "the second run is mode P (no decode stage) on the same bytes"}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
