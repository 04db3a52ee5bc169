"""CPU: the line-pool growth entry points (sse_line_pool_set_growth, sse_line_pool_capacity, ssegw_line_pool_growth) are
declared and exported, SSE_OVF_POOL agrees between the header and _abi.py, and the entry points refuse a NULL context or NULL
outputs with SSE_ERR_ARG without touching a device."""
import ctypes as C
import re

from inference_gateway_b200 import _abi as A
from tests.util import GW_HEADER, HEADER, declared_functions

NEW = ("sse_line_pool_set_growth", "sse_line_pool_capacity")


def test_growth_symbols_declared_and_exported():
    L = A.load()
    for n in NEW:
        assert n in declared_functions() and n in A.EXPORTS and hasattr(L, n), n
    assert "ssegw_line_pool_growth" in declared_functions(GW_HEADER, "ssegw_") and hasattr(L, "ssegw_line_pool_growth")


def test_ovf_pool_matches_the_header():
    m = re.search(r"#define\s+SSE_OVF_POOL\s+(0x[0-9a-fA-F]+)u", HEADER)
    assert m and int(m.group(1), 16) == A.OVF_POOL == 0x20
    bits = [A.OVF_OUT, A.OVF_TCS, A.OVF_USAGES, A.OVF_TEXT, A.OVF_RUNS, A.OVF_POOL]
    assert len(set(bits)) == len(bits) and all(b & (b - 1) == 0 for b in bits)     # one distinct bit each


def test_null_context_and_outputs_are_refused_without_a_device():
    L = A.load()
    L.ssegw_line_pool_growth.argtypes = [C.c_void_p, C.c_uint32]
    pages, limit = C.c_uint32(7), C.c_uint32(7)
    for max_pages in (0, 1, 1 << 20):
        assert L.sse_line_pool_set_growth(None, max_pages) == A.SSE_ERR_ARG
        assert L.ssegw_line_pool_growth(None, max_pages) == A.SSE_ERR_ARG
    assert L.sse_line_pool_capacity(None, C.byref(pages), C.byref(limit)) == A.SSE_ERR_ARG
    assert L.sse_line_pool_capacity(None, None, C.byref(limit)) == A.SSE_ERR_ARG
    assert L.sse_line_pool_capacity(None, C.byref(pages), None) == A.SSE_ERR_ARG
    assert (pages.value, limit.value) == (7, 7)          # nothing written on a refusal


def test_engine_keeps_the_growth_limit_out_of_the_pool_struct():
    """max_pages is not a field of sse_line_pool (whose size tests/test_line_pool_cpu.py pins): SseEngine and Gateway take it
    from the line_pool dict and set it after init."""
    assert [n for n, _ in A.LinePool._fields_] == ["struct_size", "page_bytes", "pool_pages", "max_line_bytes"]
    assert C.sizeof(A.LinePool) == 16
