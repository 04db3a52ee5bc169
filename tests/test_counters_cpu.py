"""CPU: the SSE_FLAG_COUNTERS ABI (include/sse_gpu.h sse_counters, sse_counters_read, ssegw_counters) without a device."""
import ctypes as C
import re

from inference_gateway_b200 import _abi as A
from tests.test_abi import GW_HEADER, HEADER, declared_functions


def header_counter_fields():
    body = re.search(r"typedef struct \{([^}]*)\} sse_counters;", re.sub(r"/\*.*?\*/", "", HEADER, flags=re.S), re.S).group(1)
    return re.findall(r"(uint32_t|uint64_t)\s+(\w+);", body)


def test_layout_matches_header():
    fields = header_counter_fields()
    assert fields[:2] == [("uint32_t", "struct_size"), ("uint32_t", "decode_passes")]
    assert all(t == "uint64_t" for t, _ in fields[2:])
    assert tuple(n for _, n in fields[2:]) == A.COUNTER_FIELDS
    assert [n for n, _ in A.Counters._fields_] == [n for _, n in fields]
    assert C.sizeof(A.Counters) == 8 + 8 * len(A.COUNTER_FIELDS) == 336
    assert A.Counters.p_segments.offset == 8 and A.Counters.c_unquote.offset == C.sizeof(A.Counters) - 8
    assert re.search(r"#define SSE_FLAG_COUNTERS 256u", HEADER) and A.FLAG_COUNTERS == 256


def test_counters_with_the_tile_kernel_are_refused():
    L = A.load()
    ctx = C.c_void_p()
    cfg = A.Config()
    L.sse_default_config(C.byref(cfg), 1024, 1 << 20)
    cfg.flags = A.FLAG_COUNTERS | A.FLAG_KERNEL_FUSED
    assert L.sse_init(0, C.byref(cfg), C.byref(ctx)) == A.SSE_ERR_ARG


def test_counters_read_argument_checks():
    L = A.load()
    k = A.Counters()
    k.struct_size = C.sizeof(A.Counters)
    assert L.sse_counters_read(None, 0, C.byref(k)) == A.SSE_ERR_ARG
    assert L.sse_counters_read(None, 0, None) == A.SSE_ERR_ARG
    k.struct_size = C.sizeof(A.Counters) - 8
    assert L.sse_counters_read(None, 0, C.byref(k)) == A.SSE_ERR_ARG
    L.ssegw_counters.argtypes = [C.c_void_p, C.POINTER(A.Counters)]
    k.struct_size = C.sizeof(A.Counters)
    assert L.ssegw_counters(None, C.byref(k)) == A.SSE_ERR_ARG


def test_new_symbols_are_exported():
    L = A.load()
    assert "sse_counters_read" in declared_functions() and "sse_counters_read" in A.EXPORTS
    assert "ssegw_counters" in declared_functions(GW_HEADER, "ssegw_")
    assert hasattr(L, "sse_counters_read") and hasattr(L, "ssegw_counters")
