"""Long-line decode sweep on one GPU (DESIGN.md 4.3): how the decode of one long line costs against its payload size and kind, for the
library it runs (SSE_LIB selects a prebuilt variant, e.g. one built with -DSSE_LONG_LINE=0 by tools/build_variants.sh). Prints one
JSON line.

Kinds:  args    a tool call whose arguments are an escaped file (a "\\n" every 18 bytes, as tools/long_line_bench.py)
        ascii   a content string of plain ASCII
        cjk     a content string of CJK characters and emoji (3- and 4-byte UTF-8)
        struct  a tool_calls array of small elements (structure, keys and short strings)
Counts: one line alone in the batch (latency), and as many lines as make about --batch-bytes (throughput).
Sizes:  payload bytes, 16 KiB .. 4 MiB; 16 KiB lies below the default threshold, the rest at or above it.

A step is one launch over the uploaded batch (reset, produce, sort, decode, finalize); every line is complete in its segment, so
the pool assembles it in the same launch. The GPU name and power limit are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import fill_slot, time_steps                      # noqa: E402
from tools.long_line_bench import gpu_info, tool_call_line   # noqa: E402

KiB, MiB = 1 << 10, 1 << 20
SIZES = [16 * KiB, 32 * KiB, 64 * KiB, 256 * KiB, MiB, 4 * MiB]


def line_of(kind: str, n: int) -> bytes:
    """A data line ('\\n\\n' included) whose payload is about n bytes."""
    if kind == "args":
        return tool_call_line(n + 8)
    head, tail = b'data: {"choices":[{"index":0,"delta":{"content":"', b'"},"finish_reason":null}]}\n\n'
    k = n - (len(head) - 6) - (len(tail) - 2)
    if kind == "ascii":
        return head + (b"The quick brown fox jumps over the lazy dog. " * (k // 45 + 1))[:k] + tail
    if kind == "cjk":
        unit = "长行解码😀".encode()
        return head + unit * (k // len(unit)) + b"x" * (k % len(unit)) + tail
    el = b'{"index":%d,"id":"c","type":"function","function":{"name":"f","arguments":"{}"}}'
    parts, size, i = [], 0, 0
    while size < n - 80:
        parts.append(el % i)
        size += len(parts[-1]) + 1
        i += 1
    return b'data: {"choices":[{"index":0,"delta":{"tool_calls":[' + b",".join(parts) + b']},"finish_reason":null}]}\n\n'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--batch-bytes", type=int, default=64 * MiB)
    ap.add_argument("--kinds", default="args,ascii,cjk,struct")
    ap.add_argument("--sizes", default=",".join(str(s) for s in SIZES))
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("long_decode_bench.py: no CUDA device")
    from inference_gateway_b200 import SseEngine, _abi as A
    torch.cuda.set_device(0)
    tstream = torch.cuda.Stream()
    torch.cuda.set_stream(tstream)
    stream = tstream.cuda_stream
    sm_count = torch.cuda.get_device_properties(0).multi_processor_count
    out = {"gpu": gpu_info(), "lib": os.path.basename(os.environ.get("SSE_LIB", "libssegpu.so")), "runs": []}
    mode = A.MODE_R | A.MODE_PARSE
    for kind in args.kinds.split(","):
        for size in (int(s) for s in args.sizes.split(",")):
            line = line_of(kind, size)
            for count in (1, max(1, min(8 * sm_count * 4, args.batch_bytes // len(line)))):
                bodies = [line] * count
                nbytes = sum(map(len, bodies))
                e = SseEngine(device=0, max_conns=count, bytes_per_batch=nbytes, n_slots=1, carry_slot_bytes=16384,
                              text_arena_bytes=2 * nbytes + MiB, line_pool=dict(pool_pages=count * (len(line) // 65536 + 2) + 64))
                sl, arena, segs = e.acquire()
                ns, nb, _ = fill_slot(e, arena, segs, bodies, mode)
                e.upload(sl, ns, nb, stream)

                def step(_i):
                    e.reset_all(stream)
                    e.launch(sl, ns, stream)
                for i in range(2):
                    step(i)
                torch.cuda.synchronize()
                res = e.download(sl, stream)
                ok = int(A.F_JSON_OK)
                decoded = int(((res.recs["flags"] & ok) != 0).sum())
                ms = time_steps(torch, step, args.steps) / args.steps
                run = {"kind": kind, "payload_bytes": len(line) - 8, "lines": count, "ms_per_step": round(ms, 4),
                       "mb_per_s": round(nbytes / (ms / 1e3) / 1e6, 1), "json_ok": decoded}
                out["runs"].append(run)
                print("#", json.dumps(run), file=sys.stderr, flush=True)
                e.close()
                torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
