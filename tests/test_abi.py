"""CPU: the C-ABI library loads, exports exactly the symbols include/sse_gpu.h and include/sse_gateway.h declare, has the documented struct
layouts, and fails loudly without a CUDA device (no CPU fallback). No compute calls here."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from inference_gateway_b200 import _abi as A
from tests.util import GW_HEADER, declared_functions


def test_exports_every_declared_symbol():
    L = A.load()
    names = declared_functions()
    assert len(names) >= 25
    for n in names:
        assert hasattr(L, n), f"{n} is declared in include/sse_gpu.h but not exported by libssegpu.so"
    assert set(names) == set(A.EXPORTS)
    assert L.sse_abi_version() == 2
    gw = declared_functions(GW_HEADER, "ssegw_")
    assert len(gw) >= 12
    for n in gw:
        assert hasattr(L, n), f"{n} is declared in include/sse_gateway.h but not exported"
    # and nothing else: every sse_* / ssegw_* symbol the library exports is declared by one of the two headers
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm not available")
    out = subprocess.run([nm, "-D", "--defined-only", A.lib_path()], capture_output=True, text=True, check=True).stdout
    exported = {f[-1] for f in map(str.split, out.splitlines()) if f and re.match(r"sse(gw)?_", f[-1])}
    assert exported == set(names) | set(gw)


def test_struct_layouts_match_header():
    assert C.sizeof(A.Seg) == 16 and C.sizeof(A.Frame) == 8 and C.sizeof(A.Rec) == 32 and C.sizeof(A.Tc) == 48
    assert C.sizeof(A.Usage) == 24 and C.sizeof(A.Run) == 20 and C.sizeof(A.SegResult) == 32
    assert C.sizeof(A.Config) == 14 * 4
    cfg = A.Config()
    A.load().sse_default_config(C.byref(cfg), 1024, 1 << 20)
    assert cfg.struct_size == C.sizeof(A.Config) and cfg.max_conns == 1024 and cfg.in_arena_bytes % 16 == 0


def test_strerror_and_argument_checks():
    L = A.load()
    assert b"no CPU fallback" in L.sse_strerror(A.SSE_ERR_NO_DEVICE)
    assert L.sse_strerror(0) == b"ok"
    ctx = C.c_void_p()
    bad = A.Config()
    assert L.sse_init(0, C.byref(bad), C.byref(ctx)) == A.SSE_ERR_ARG        # struct_size mismatch
    # arena offsets are 31-bit (out arena + input arena share one address space, include/sse_gpu.h sse_at): a batch that
    # cannot be addressed is refused up front, before any device is touched
    big = A.Config()
    L.sse_default_config(C.byref(big), 1024, 1 << 20)
    big.in_arena_bytes = 1 << 30
    big.out_arena_bytes = (1 << 30) + (1 << 29)
    assert L.sse_init(0, C.byref(big), C.byref(ctx)) == A.SSE_ERR_ARG
    # unknown engine flags are refused (bit 0 was the first-generation kernel, bit 1 an earlier fused design: both removed)
    for fl in (1, 2, 32, 1 << 31):
        odd = A.Config()
        L.sse_default_config(C.byref(odd), 1024, 1 << 20)
        odd.flags = fl
        assert L.sse_init(0, C.byref(odd), C.byref(ctx)) == A.SSE_ERR_ARG
    # sse_worst_case_config: capacities that no batch of that many input bytes can overflow (one record per 4 bytes at most:
    # "data: x\n" is 8 bytes, "\n" alone yields a frame but no record)
    wc = A.Config()
    L.sse_worst_case_config(C.byref(wc), 64, 1 << 20)
    assert wc.struct_size == C.sizeof(A.Config) and wc.max_frames >= (1 << 20) and wc.max_recs >= (1 << 20) // 8
    # sse_at resolves both halves of the offset space
    res = A.Result()
    ob = (C.c_uint8 * 8)(*b"OUTARENA"); ib = (C.c_uint8 * 8)(*b"INPUTBUF")
    res.out = C.cast(ob, C.POINTER(C.c_uint8)); res.in_ = C.cast(ib, C.POINTER(C.c_uint8)); res.in_base = 4096
    assert L.sse_at(C.byref(res), 3)[0] == ord("A") and L.sse_at(C.byref(res), 4096 + 5)[0] == ord("B")


def test_no_device_is_an_error_not_a_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    from inference_gateway_b200 import SseEngine
    with pytest.raises(A.SseError) as e:
        SseEngine(device=0, max_conns=16, bytes_per_batch=1 << 16)
    assert e.value.status == A.SSE_ERR_NO_DEVICE


def test_sass_is_sm90a():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-lelf", A.lib_path()], capture_output=True, text=True).stdout
    assert "sm_90a" in out
