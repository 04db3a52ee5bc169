"""GPU: contexts are independent. One context per engine variant (and one more per extra visible device) is created and driven
on its own thread, all released together, in a fresh process so that every context's first launch is the first in its process;
each one's digests match the oracle's. And a context holds exactly what its engine uses: SSE_FLAG_TEMPLATES adds the template
cache and nothing else."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from inference_gateway_b200 import SseEngine, _abi as A, synth
from tests.util import ENGINES, ROOT, assert_digest_parity, oracle_digests

pytestmark = pytest.mark.gpu

N_STREAMS, N_PIECES, SEED = 512, 3, 41

# Runs in the fresh process: argv = output directory, contexts as JSON [[label, flags, device], ...]. Each thread waits at the
# barrier, then creates its context and feeds every stream in N_PIECES batches; ctypes drops the GIL in sse_init_ex and sse_submit,
# so the threads' calls overlap. Writes <label>.npz (digests, carry_len, seg_flags) per context.
CHILD = f"""
import json, os, sys, threading, traceback
import numpy as np
from inference_gateway_b200 import SseEngine, _abi as A, synth
from oracle import orc
from tests.util import cut_bounds, digest_run

out, contexts = sys.argv[1], json.loads(sys.argv[2])
streams, mode = synth.make_config("C3", n_streams={N_STREAMS})
bodies = [b for b, _, _ in streams]
modes = np.full(len(bodies), mode, dtype=np.uint8)
bounds = cut_bounds(bodies, {N_PIECES}, seed={SEED})
A.load()
orc.lib()   # both libraries are loaded before the threads start
barrier = threading.Barrier(len(contexts))
failed = []

def run(label, flags, device):
    try:
        barrier.wait()
        eng = SseEngine(device=device, max_conns=len(bodies), bytes_per_batch=sum(map(len, bodies)), flags=flags)
        try:
            d, carry, seg_flags = digest_run(eng, bodies, modes, bounds)
        finally:
            eng.close()
        np.savez(os.path.join(out, label + ".npz"), d=d, carry=carry, seg_flags=seg_flags)
    except BaseException:
        failed.append(label + ": " + traceback.format_exc())

threads = [threading.Thread(target=run, args=c) for c in contexts]
for t in threads:
    t.start()
for t in threads:
    t.join()
if failed:
    sys.exit("\\n".join(failed))
"""


def test_contexts_on_threads_at_once_match_the_oracle(tmp_path):
    contexts = [[name, flags, 0] for name, flags in ENGINES.items()]
    names = list(ENGINES)
    contexts += [[f"{names[(dev - 1) % len(names)]}@{dev}", ENGINES[names[(dev - 1) % len(names)]], dev]
                 for dev in range(1, torch.cuda.device_count())]
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(p for p in (ROOT, os.environ.get("PYTHONPATH")) if p))
    flags = ["-s"] if sys.flags.no_user_site else []
    p = subprocess.run([sys.executable, *flags, "-c", CHILD, str(tmp_path), json.dumps(contexts)], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-4000:]
    streams, mode = synth.make_config("C3", n_streams=N_STREAMS)
    bodies = [b for b, _, _ in streams]
    oracle = oracle_digests(bodies, mode)
    for label, _, _ in contexts:
        z = np.load(tmp_path / f"{label}.npz")
        assert_digest_parity((z["d"], z["carry"], z["seg_flags"]), bodies, mode, f"context {label} on its own thread", oracle=oracle)


@pytest.mark.parametrize("engine", ["split", "fused"])
def test_templates_hold_exactly_the_template_cache(engine):
    def held(flags):
        eng = SseEngine(device=0, max_conns=1024, bytes_per_batch=1 << 20, flags=ENGINES[engine] | flags)
        try:
            return eng.memory_held()
        finally:
            eng.close()
    dev, pinned = held(0)
    assert held(A.FLAG_TEMPLATES) == (dev + 8192 * 4, pinned)
