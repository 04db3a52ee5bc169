"""CPU: sse_trim, sse_memory_held and ssegw_trim are declared, exported and bound; NULL arguments are refused with SSE_ERR_ARG
before a device is touched, and a refused call writes nothing."""
import ctypes as C
import inspect

from inference_gateway_b200 import SseEngine, _abi as A
from inference_gateway_b200.gateway import Gateway
from tests.util import GW_HEADER, declared_functions

SENTINEL = 0x5EED5EED5EED5EED


def test_declared_exported_and_listed():
    L = A.load()
    for name in ("sse_trim", "sse_memory_held"):
        assert name in declared_functions() and name in A.EXPORTS and hasattr(L, name)
    assert "ssegw_trim" in declared_functions(GW_HEADER, "ssegw_") and hasattr(L, "ssegw_trim")


def test_null_arguments_are_refused_and_nothing_is_written():
    L = A.load()
    assert L.sse_trim(None, 8) == A.SSE_ERR_ARG
    assert L.sse_trim(None, A.NONE) == A.SSE_ERR_ARG
    dev, pin = C.c_uint64(SENTINEL), C.c_uint64(SENTINEL)
    assert L.sse_memory_held(None, C.byref(dev), C.byref(pin)) == A.SSE_ERR_ARG
    assert L.sse_memory_held(None, None, C.byref(pin)) == A.SSE_ERR_ARG
    assert L.sse_memory_held(None, C.byref(dev), None) == A.SSE_ERR_ARG
    assert (dev.value, pin.value) == (SENTINEL, SENTINEL)
    L.ssegw_trim.argtypes = [C.c_void_p, C.c_uint32]
    assert L.ssegw_trim(None, 0) == A.SSE_ERR_ARG


def test_engine_and_gateway_expose_the_methods():
    for cls in (SseEngine, Gateway):
        sig = inspect.signature(cls.trim)
        assert list(sig.parameters) == ["self", "min_pool_pages"] and sig.parameters["min_pool_pages"].default is None
    assert list(inspect.signature(SseEngine.memory_held).parameters) == ["self"]
