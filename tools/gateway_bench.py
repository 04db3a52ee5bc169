"""Ticks per second and delivered chunks per second through the gateway mirror (include/sse_gateway.h), from upstream write to
recv: C3- and C4-shaped streams, each body cut into seeded pieces and written one piece per stream and tick, at depth 1 and at
n_slots, on one context and on two contexts on device 0. Every tick is split into its three host phases: upstream writes,
ssegw_pump (fill, submit, collect, fan-out), receives. Prints one JSON line per case, with the card it ran on.

--tap measures what the telemetry tap (ssegw_stream_with_telemetry) adds to the pump, where the folds run: on one context at
depth 1 and at n_slots, the same streams as plain P, P|PARSE, P|PARSE with a fold per stream, R, and R with a fold per stream,
alternating.

    python tools/gateway_bench.py [--streams 4096] [--pieces 32] [--reps 3] [--tap] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from inference_gateway_b200 import _abi as A, synth  # noqa: E402
from inference_gateway_b200.gateway import Gateway, Telemetry  # noqa: E402

N_SLOTS = 4


def gpu_info() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def one_pass(g, bodies, mode, pieces, tap=False):
    """Opens every stream (tap: each with a telemetry fold of its own), writes piece t of every body at tick t, closes each
    upstream after its last piece, pumps until every channel is closed. Returns the counts and the seconds spent in each
    phase."""
    n = len(bodies)
    taps = [Telemetry() if tap else None for _ in range(n)]
    sids = [g.stream_chat_completions(mode, telemetry=t) for t in taps]
    cur = [0] * n
    left = [b""] * n
    eof = [False] * n
    closed = [False] * n
    st = dict(ticks=0, chunks=0, write_s=0.0, pump_s=0.0, recv_s=0.0)
    recv = g.recv
    t_start = time.perf_counter()
    while not all(eof):
        t0 = time.perf_counter()
        for i, sid in enumerate(sids):
            if not left[i] and cur[i] < len(pieces[i]):
                left[i] = pieces[i][cur[i]]
                cur[i] += 1
            if left[i]:
                left[i] = left[i][g.upstream_write(sid, left[i]):]
            elif not closed[i] and cur[i] == len(pieces[i]):
                g.upstream_close(sid)
                closed[i] = True
        t1 = time.perf_counter()
        g.pump()
        t2 = time.perf_counter()
        for i, sid in enumerate(sids):
            if eof[i]:
                continue
            try:
                while recv(sid) is not None:
                    st["chunks"] += 1
            except EOFError:
                eof[i] = True
        t3 = time.perf_counter()
        st["ticks"] += 1
        st["write_s"] += t1 - t0
        st["pump_s"] += t2 - t1
        st["recv_s"] += t3 - t2
    st["wall_s"] = time.perf_counter() - t_start
    g.flush()
    for sid in sids:
        g.release(sid)
    for t in taps:
        if t is not None:
            t.finish()
            t.close()
    return st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=4096)
    ap.add_argument("--pieces", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--tap", action="store_true", help="pump time with and without a telemetry fold on every stream")
    a = ap.parse_args()
    info = gpu_info()
    L = A.load()
    rows = []
    for name in ("C3", "C4"):
        streams, mode = synth.make_config(name, n_streams=a.streams)
        bodies = [b for b, _, _ in streams]
        rng = np.random.default_rng(11)
        pieces = [synth.random_cuts(rng, b, a.pieces) for b in bodies]
        cfg = A.Config()
        L.sse_default_config(C.byref(cfg), a.streams, max(1 << 16, sum(map(len, bodies)) // a.pieces * 2))
        cfg.n_slots = N_SLOTS
        if a.tap:
            PP = A.MODE_P | A.MODE_PARSE
            arms = [(A.MODE_P, False), (PP, False), (PP, True), (A.MODE_R | A.MODE_PARSE, False), (A.MODE_R | A.MODE_PARSE, True)]
            cases = [((0,), depth) for depth in (1, N_SLOTS)]
        else:
            arms = [(mode, False)]
            cases = [(devs, depth) for devs in ((0,), (0, 0)) for depth in (1, N_SLOTS)]
        gws = {c: Gateway(config=cfg, devices=list(c[0]), depth=c[1]) for c in cases}
        try:
            for c in cases:                                        # warm-up: first launches, pinned pages, allocator
                for m, tap in arms:
                    one_pass(gws[c], bodies, m, pieces, tap)
            runs = {(c, arm): [] for c in cases for arm in arms}
            for _ in range(a.reps):                                # the cases alternate, so that drift hits them alike
                for c in cases:
                    for arm in arms:
                        runs[(c, arm)].append(one_pass(gws[c], bodies, arm[0], pieces, arm[1]))
        finally:
            for g in gws.values():
                g.close()
        for ((devs, depth), (m, tap)), rs in runs.items():
            best = min(rs, key=lambda r: r["wall_s"])
            row = dict(workload=name, streams=a.streams, bytes=sum(map(len, bodies)), pieces=a.pieces, contexts=len(devs),
                       depth=depth, mode=m, tap=tap, ticks=best["ticks"], chunks=best["chunks"],
                       ticks_per_s=round(best["ticks"] / best["wall_s"], 1), chunks_per_s=round(best["chunks"] / best["wall_s"]),
                       wall_ms=[round(r["wall_s"] * 1e3, 1) for r in rs],
                       tick_ms=dict(write=round(best["write_s"] / best["ticks"] * 1e3, 3),
                                    pump=round(best["pump_s"] / best["ticks"] * 1e3, 3),
                                    recv=round(best["recv_s"] / best["ticks"] * 1e3, 3)),
                       pump_ms_per_tick=[round(r["pump_s"] / r["ticks"] * 1e3, 3) for r in rs],
                       gpu=info)
            rows.append(row)
            print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
