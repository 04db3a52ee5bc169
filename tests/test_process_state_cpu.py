"""CPU: libssegpu.so keeps no process-wide state of its own. Contexts are created and driven on several threads at once, often
on different devices, so what their launches need (kernel attributes, occupancy, decode tables, launch counts) belongs to each
context. Among the data symbols the library defines, none comes from csrc/ except the two listed here."""
import shutil
import subprocess

import pytest

from inference_gateway_b200 import _abi as A

# each thread's text for sse_last_cuda_error, and the host shadow of the schema kept in constant memory (read-only)
ALLOWED = {"(anonymous namespace)::g_cuda_err", "(anonymous namespace)::c_schema"}


def from_toolchain(name: str) -> bool:
    """nvcc's module registration (__fatDeviceText, __cudaFatCubinHandle), the static CUDA runtime and what the linker and the
    C runtime add (_DYNAMIC, __dso_handle, completed.0, DW.ref.*): reserved identifiers, names no C++ source can declare, and
    the runtime's prefix."""
    return name.startswith(("_", "libcudart_static_")) or "." in name


def test_no_process_wide_data():
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm not available")
    A.load()
    out = subprocess.run([nm, "-C", "--defined-only", A.lib_path()], capture_output=True, text=True, check=True).stdout
    data = {f[2] for f in (line.split(None, 2) for line in out.splitlines()) if len(f) == 3 and f[1] in ("b", "B", "d", "D")}
    ours = {n for n in data if not from_toolchain(n)}
    assert ours <= ALLOWED, f"process-wide data outside a context: {sorted(ours - ALLOWED)}"
    assert "(anonymous namespace)::g_cuda_err" in ours   # the filter keeps what the sources define
