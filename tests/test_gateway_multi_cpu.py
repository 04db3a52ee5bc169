"""CPU: the entry points of batches in flight (sse_poll) and of a gateway over several contexts (ssegw_new_multi,
ssegw_flush) are declared, exported and refuse bad arguments before any device is touched."""
import ctypes as C
import os

import pytest

from inference_gateway_b200 import _abi as A
from inference_gateway_b200.gateway import Gateway
from tests.util import GW_HEADER, HEADER, declared_functions


def _cfg(n_slots=4, conns=16):
    cfg = A.Config()
    A.load().sse_default_config(C.byref(cfg), conns, 1 << 16)
    cfg.n_slots = n_slots
    return cfg


def _multi(devices, cfg, depth, pool=None):
    L = A.load()
    L.ssegw_new_multi.argtypes = [C.POINTER(C.c_int), C.c_uint32, C.POINTER(A.Config), C.POINTER(A.LinePool), C.c_uint32,
                                  C.POINTER(C.c_int)]
    L.ssegw_new_multi.restype = C.c_void_p
    st = C.c_int(1)
    arr = (C.c_int * max(1, len(devices)))(*devices)
    g = L.ssegw_new_multi(arr, len(devices), C.byref(cfg) if cfg is not None else None, pool, depth, C.byref(st))
    return g, st.value


def _no_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")


def test_new_symbols_are_declared_and_exported():
    L = A.load()
    assert "sse_poll" in declared_functions() and "sse_poll" in A.EXPORTS and hasattr(L, "sse_poll")
    gw = declared_functions(GW_HEADER, "ssegw_")
    for n in ("ssegw_new_multi", "ssegw_flush"):
        assert n in gw and hasattr(L, n)
    assert L.sse_abi_version() == 2
    assert "#define SSE_ABI_VERSION 2" in HEADER


def test_go_binding_polls():
    go = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "integration", "go", "ssegpu.go")).read()
    assert "C.sse_poll(" in go


def test_poll_refuses_a_null_context():
    L = A.load()
    for slot in (0, -1, 7):
        assert L.sse_poll(None, slot) == A.SSE_ERR_ARG


@pytest.mark.parametrize("devices,depth,why", [
    ([], 1, "no device"),
    ([0] * 65, 1, "more than 64 contexts"),
    ([0], 0, "depth 0"),
    ([0, 0], 5, "depth above n_slots"),
])
def test_new_multi_refuses_bad_arguments(devices, depth, why):
    g, st = _multi(devices, _cfg(n_slots=4), depth)
    assert not g and st == A.SSE_ERR_ARG, why


def test_new_multi_refuses_bad_configs():
    bad = _cfg()
    bad.struct_size = 0
    assert _multi([0], bad, 1) == (None, A.SSE_ERR_ARG)
    assert _multi([0], None, 1) == (None, A.SSE_ERR_ARG)
    odd = _cfg()
    odd.flags = 1 << 31          # what sse_init_ex refuses, before a device is touched
    assert _multi([0, 0], odd, 1) == (None, A.SSE_ERR_ARG)
    pool = A.LinePool(struct_size=C.sizeof(A.LinePool), page_bytes=100, pool_pages=4, max_line_bytes=1 << 20)
    assert _multi([0], _cfg(), 1, C.byref(pool)) == (None, A.SSE_ERR_ARG)   # page size not a multiple of 16


@pytest.mark.parametrize("devices,depth", [([0], 1), ([0, 0], 2), ([0, 0, 0], 4)])
def test_new_multi_without_a_device_is_an_error_not_a_fallback(devices, depth):
    _no_gpu()
    assert _multi(devices, _cfg(n_slots=4), depth) == (None, A.SSE_ERR_NO_DEVICE)


def test_python_gateway_needs_a_config_for_devices_and_depth():
    with pytest.raises(ValueError):
        Gateway(devices=[0, 0])
    with pytest.raises(ValueError):
        Gateway(depth=2)
    _no_gpu()
    with pytest.raises(A.SseError) as e:
        Gateway(devices=[0, 0], config=_cfg(), depth=2)
    assert e.value.status == A.SSE_ERR_NO_DEVICE
    with pytest.raises(A.SseError) as e:
        Gateway(devices=[0], config=_cfg(n_slots=2), depth=3)
    assert e.value.status == A.SSE_ERR_ARG
