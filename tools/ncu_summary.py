#!/usr/bin/env python3
"""Writes profiles/<tag>_{produce,decode}_ncu.txt, <tag>_launches.{csv,txt} and profiles/traffic.json from the captures
tools/profile_round.sh leaves in gpurun_out/ (produce.ncu-rep, decode.ncu-rep, launches.csv, traffic.csv)."""
import csv
import json
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
tag = sys.argv[1]
G = os.path.join(ROOT, "gpurun_out")
Pdir = os.path.join(ROOT, "profiles")
WANT = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "smsp__inst_executed.sum",
        "sm__inst_executed.avg.per_cycle_elapsed", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "smsp__thread_inst_executed_per_inst_executed.ratio",
        "smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio",
        "lts__t_sector_hit_rate.pct", "launch__grid_size", "launch__block_size"]
HEAD = {"produce": "stage 1 of the split pipeline: sse_stream_kernel (stage, split, classify, frame table, work items; "
                   "zero-copy frames are not serialized)",
        "decode": "stage 3 of the split pipeline: sse_decode_kernel (table-driven automaton, one lane per line, items sorted by "
                  "(length, shape))"}
CMD = "python bench.py --steps 2 --warmup 3 --no-e2e --no-cpu-baseline --no-strong --segments 0"


def raw(rep):
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    return dict(zip(rows[0], zip(rows[1], rows[-1])))


for k in ("produce", "decode"):
    rep = os.path.join(G, k + ".ncu-rep")
    if not os.path.exists(rep):
        continue
    m = raw(rep)
    lines = [f"ncu --set full --clock-control none --import-source on, {HEAD[k]}",
             f"workload C4: 65536 streams, 332.8 MB input, 714214 SSE events; {CMD}", ""]
    for w in WANT:
        if w in m:
            unit, val = m[w]
            lines.append(f"{w:<90s} {val:>18s} {unit}")
    lines += ["", "source lines ranked by executed warp instructions (tools/ncu_lines.py):"]
    lines.append(subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ncu_lines.py"), rep, "45"],
                                capture_output=True, text=True).stdout)
    open(os.path.join(Pdir, f"{tag}_{k}_ncu.txt"), "w").write("\n".join(lines))

lc = os.path.join(G, "launches.csv")
if os.path.exists(lc):
    shutil.copy(lc, os.path.join(Pdir, f"{tag}_launches.csv"))
    rows = [r for r in csv.reader(open(lc)) if len(r) > 5 and r[0].isdigit()]
    per = {}
    for r in rows[-12:]:         # the two timed steps (6 launches each)
        name = r[4].split("(")[0].replace("void ", "").replace("<unnamed>::", "")
        per.setdefault(name, []).append(float(r[-1]))
    tot = sum(sum(v) / len(v) for v in per.values())
    txt = [f"ncu --metrics gpu__time_duration.sum --clock-control none; {CMD}; two steps of the run, per launch (ns, serialised, cold):"]
    for n, v in per.items():
        a = sum(v) / len(v)
        txt.append(f"  {n:<45s} {a:>12.0f} ns   {100 * a / tot:5.1f} % of the step")
    txt.append(f"  {'sum':<45s} {tot:>12.0f} ns")
    open(os.path.join(Pdir, f"{tag}_launches.txt"), "w").write("\n".join(txt) + "\n")

tc = os.path.join(G, "traffic.csv")
if os.path.exists(tc):
    rows = [r for r in csv.reader(open(tc)) if len(r) > 5 and r[0].isdigit()]
    per = {}
    for r in rows:
        if r[-3].startswith("dram__bytes"):
            name = r[4].split("(")[0].replace("void ", "").replace("<unnamed>::", "")
            per[name] = per.get(name, 0) + int(float(r[-1]))
    json.dump({"workload": "C4", "streams": 65536, "dram_bytes_per_launch": sum(per.values()), "per_kernel": per,
               "note": "dram__bytes_read.sum + dram__bytes_write.sum of the six launches of one step (ncu, tools/profile_round.sh)"},
              open(os.path.join(Pdir, "traffic.json"), "w"), indent=1)
print("ok")
