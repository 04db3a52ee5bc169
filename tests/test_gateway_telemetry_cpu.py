"""CPU: the gateway's telemetry tap (ssegw_stream_with_telemetry) is declared, exported and bound in Python and Go, refuses
bad arguments before a device is touched, and leaves the ABI version alone."""
import ctypes as C
import os

from inference_gateway_b200 import _abi as A
from inference_gateway_b200.gateway import Gateway, Telemetry
from tests.util import GW_HEADER, HEADER, declared_functions

GO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "integration", "go")


def test_tap_is_declared_and_exported():
    L = A.load()
    assert "ssegw_stream_with_telemetry" in declared_functions(GW_HEADER, "ssegw_")
    assert hasattr(L, "ssegw_stream_with_telemetry")
    assert L.sse_abi_version() == 2 and "#define SSE_ABI_VERSION 2" in HEADER


def test_python_binds_the_tap():
    import inspect
    src = inspect.getsource(Gateway)
    assert "ssegw_stream_with_telemetry" in src
    for fn in (Gateway.stream_chat_completions, Gateway.proxy_stream):
        assert "telemetry" in inspect.signature(fn).parameters


def test_tap_refuses_a_null_gateway_or_fold_without_a_device():
    L = A.load()
    L.ssegw_stream_with_telemetry.argtypes = [C.c_void_p, C.c_uint8, C.c_void_p]
    t = Telemetry()
    try:
        assert L.ssegw_stream_with_telemetry(None, A.MODE_P | A.MODE_PARSE, t.f) == A.SSE_ERR_ARG
        assert L.ssegw_stream_with_telemetry(None, A.MODE_R, None) == A.SSE_ERR_ARG
        t.feed_bytes(b"data: [DONE]\n\n")
        assert t.finish() == (0, (0, 0, 0), [])
    finally:
        t.close()


def test_go_binding_feeds_the_tap():
    src = {f: open(os.path.join(GO, f)).read() for f in ("ssegpu.go", "gpu_provider.go")}
    assert "C.sse_telemetry_feed(" in src["ssegpu.go"]
    for fn in ("sse_telemetry_new", "sse_telemetry_feed_bytes", "sse_telemetry_finish", "sse_telemetry_free"):
        assert f"C.{fn}(" in src["ssegpu.go"]
