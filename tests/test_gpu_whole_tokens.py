"""GPU: member keys, string values and digit runs that the decode automaton takes a window at a time, against the oracle.

The decode kernel skips the plain bytes of key and value strings and of digit runs, and resolves a key (and a finish_reason
value) at its end from its bytes through the name table (csrc/sse_tables.h). These documents put those tokens at every window
alignment and every case the name match distinguishes: schema keys in mixed case and in the wrong struct, near misses, long keys,
keys that hash to a known name's slot, escaped and Unicode-folded keys, the case-sensitive google map, finish_reason values, and
numbers of 1-40 digits. Every engine decodes them alone (field-by-field parity, per connection) and among filler lines that put
the launch in each of the 8-, 16- and 32-item decode shapes (digest parity)."""
import numpy as np
import pytest
import torch

from inference_gateway_b200 import SseEngine, _abi as A
from tests.corpus import documents
from tests.streams import dealt, filler_payload
from tests.util import ENGINES, TARGET, check_streams, digest_parity, run_streams, shape_check

pytestmark = pytest.mark.gpu
R, PP = A.MODE_R | A.MODE_PARSE, A.MODE_P | A.MODE_PARSE


def bodies_of(docs):
    return [b"data: " + d + b"\n\n" for d in docs], np.array([(R, PP)[i % 2] for i in range(len(docs))], dtype=np.uint8)


@pytest.mark.parametrize("engine_name", list(ENGINES))
def test_whole_tokens_field_by_field(engine_name):
    bodies, modes = bodies_of(documents())
    eng = SseEngine(device=0, max_conns=len(bodies) + 16, bytes_per_batch=8 << 20, flags=ENGINES[engine_name])
    try:
        for nb in (1, 3):
            outs = run_streams(eng, bodies, list(modes), n_batches=nb, seed=nb)
            check_streams(bodies, modes, outs, f"{engine_name} x{nb}")
    finally:
        eng.close()


@pytest.mark.parametrize("engine_name", list(ENGINES))
@pytest.mark.parametrize("shape", [8, 16, 32])
def test_whole_tokens_in_each_decode_shape(engine_name, shape):
    sm_count = torch.cuda.get_device_properties(0).multi_processor_count
    docs = documents()
    target = int(TARGET[shape] * sm_count * 32)
    rng = np.random.default_rng(shape)
    assert len(docs) < target
    fill = [filler_payload("strings" if i % 2 else "nostring", int(n)) for i, n in enumerate(rng.integers(40, 700, target - len(docs)))]
    per = docs + fill
    per = [per[i] for i in rng.permutation(len(per))]
    bodies, bounds, _ = dealt([per])
    eng = SseEngine(device=0, max_conns=len(bodies) + 16, bytes_per_batch=96 << 20, n_slots=1, flags=ENGINES[engine_name])
    try:
        log = []
        digest_parity(eng, bodies, PP, bounds, f"{engine_name} {shape}-item shape", on_batch=shape_check(eng, sm_count, shape, log))
        assert len(log) == 1
    finally:
        eng.close()
