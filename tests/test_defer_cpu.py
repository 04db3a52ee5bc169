"""CPU: the SSE_FLAG_DEFER surface of include/sse_gpu.h / sse_gateway.h is present, and sse_init / ssegw_new_cfg check it before
any device is touched."""
import ctypes as C
import os

from inference_gateway_b200 import _abi as A
from inference_gateway_b200.engine import SEGRES_DT, make_line_pool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(flags=0, conns=1024, batch=1 << 20):
    cfg = A.Config()
    A.load().sse_default_config(C.byref(cfg), conns, batch)
    cfg.flags = flags
    return cfg


def _init(cfg, pool=None):
    ctx = C.c_void_p()
    return A.load().sse_init_ex(0, C.byref(cfg), C.byref(pool) if pool is not None else None, C.byref(ctx))


def _no_gpu():
    import torch
    return not torch.cuda.is_available()


def test_defer_symbols_in_header_and_abi():
    h = open(os.path.join(ROOT, "include", "sse_gpu.h")).read()
    assert "#define SSE_FLAG_DEFER 64u" in h and "#define SSE_SEG_DEFERRED     0x10u" in h
    assert "uint32_t consumed;" in h and "uint32_t reserved;\n} sse_seg_result" not in h
    assert "ssegw_new_cfg(int device, const sse_config *cfg, const sse_line_pool *pool, int *status)" in \
        open(os.path.join(ROOT, "include", "sse_gateway.h")).read()
    assert A.FLAG_DEFER == 0x40 and A.SEG_DEFERRED == 0x10
    assert (A.OVF_OUT, A.OVF_TCS, A.OVF_USAGES, A.OVF_TEXT, A.OVF_RUNS) == (1, 2, 4, 8, 16)
    assert [n for n, _ in A.SegResult._fields_][-1] == "consumed" and C.sizeof(A.SegResult) == 32
    assert SEGRES_DT.names[-1] == "consumed" and SEGRES_DT.fields["consumed"][1] == 28
    assert hasattr(A.load(), "ssegw_new_cfg")


def test_defer_flag_passes_argument_checks():
    if not _no_gpu():
        return
    assert _init(_cfg(A.FLAG_DEFER)) == A.SSE_ERR_NO_DEVICE
    assert _init(_cfg(A.FLAG_DEFER | A.FLAG_TEMPLATES | A.FLAG_COPY_OUT)) == A.SSE_ERR_NO_DEVICE
    assert _init(_cfg(A.FLAG_DEFER), make_line_pool(64, max_line_bytes=1 << 20)) == A.SSE_ERR_NO_DEVICE
    # a pooled line must fit the (pool-grown) out arena of an empty batch: 16 MiB lines do not fit 1 MiB batches with 4 MiB of pool
    assert _init(_cfg(A.FLAG_DEFER), make_line_pool(64)) == A.SSE_ERR_ARG


def test_defer_with_the_tile_kernel_is_refused():
    assert _init(_cfg(A.FLAG_DEFER | A.FLAG_KERNEL_FUSED)) == A.SSE_ERR_ARG


def test_defer_refuses_capacities_below_one_round_or_one_line():
    """With SSE_FLAG_DEFER a segment alone in a batch must always get somewhere."""
    for field, value in (("max_frames", 63), ("max_recs", 63), ("out_arena_bytes", 8192)):
        cfg = _cfg(A.FLAG_DEFER)
        setattr(cfg, field, value)
        assert _init(cfg) == A.SSE_ERR_ARG, field
    cfg = _cfg(A.FLAG_DEFER)
    cfg.out_arena_bytes = cfg.carry_slot_bytes + 32           # the longest line held in the slot would never fit
    assert _init(cfg) == A.SSE_ERR_ARG
    if _no_gpu():                                             # the same capacities without the flag are a matter for the caller
        cfg.flags = 0
        assert _init(cfg) == A.SSE_ERR_NO_DEVICE


def test_unknown_flag_bits_stay_refused():
    for bit in (1, 2, 32, 128, 1 << 31):
        assert _init(_cfg(bit)) == A.SSE_ERR_ARG, bit


def test_gateway_new_cfg_refuses_bad_configs_before_a_device():
    L = A.load()
    L.ssegw_new_cfg.argtypes = [C.c_int, C.POINTER(A.Config), C.POINTER(A.LinePool), C.POINTER(C.c_int)]
    L.ssegw_new_cfg.restype = C.c_void_p
    st = C.c_int(1)
    assert not L.ssegw_new_cfg(0, None, None, C.byref(st)) and st.value == A.SSE_ERR_ARG
    bad = _cfg(A.FLAG_DEFER)
    bad.struct_size = 4
    st.value = 1
    assert not L.ssegw_new_cfg(0, C.byref(bad), None, C.byref(st)) and st.value == A.SSE_ERR_ARG
    fused = _cfg(A.FLAG_DEFER | A.FLAG_KERNEL_FUSED)
    st.value = 1
    assert not L.ssegw_new_cfg(0, C.byref(fused), None, C.byref(st)) and st.value == A.SSE_ERR_ARG
    if _no_gpu():
        st.value = 1
        assert not L.ssegw_new_cfg(0, C.byref(_cfg(A.FLAG_DEFER)), None, C.byref(st)) and st.value == A.SSE_ERR_NO_DEVICE
