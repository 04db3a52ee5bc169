"""CPU: the line-pool entry points of include/sse_gpu.h are exported, sse_init_ex refuses bad pool arguments before any
device is touched, and sse_line_pool_config grows the per-batch capacities by the documented rule."""
import ctypes as C

from inference_gateway_b200 import _abi as A
from inference_gateway_b200.engine import make_line_pool as line_pool

GROWN = ("out_arena_bytes", "max_frames", "max_recs", "max_tcs", "max_usages", "text_arena_bytes", "max_runs")
CAP = 0xF0000000


def _cfg(worst=False, conns=1024, batch=1 << 20):
    L = A.load()
    cfg = A.Config()
    (L.sse_worst_case_config if worst else L.sse_default_config)(C.byref(cfg), conns, batch)
    return cfg


def _init_ex(cfg, pool):
    ctx = C.c_void_p()
    return A.load().sse_init_ex(0, C.byref(cfg), C.byref(pool) if pool is not None else None, C.byref(ctx))


def test_line_pool_symbols_exported():
    L = A.load()
    for n in ("sse_init_ex", "sse_line_pool_config", "sse_line_pool_stats", "ssegw_new_ex"):
        assert hasattr(L, n), n
    assert {"sse_init_ex", "sse_line_pool_config", "sse_line_pool_stats"} <= set(A.EXPORTS)
    assert C.sizeof(A.LinePool) == 16 and A.MAX_LINE_BYTES == (1 << 24) - 1


def test_init_ex_refuses_bad_pools_without_a_device():
    cfg = _cfg()
    bad = line_pool(64)
    bad.struct_size = 12
    assert _init_ex(cfg, bad) == A.SSE_ERR_ARG                                   # struct_size mismatch
    assert _init_ex(cfg, line_pool(64, page_bytes=65536 + 8)) == A.SSE_ERR_ARG    # page size not a multiple of 16
    assert _init_ex(cfg, line_pool(64, max_line_bytes=A.MAX_LINE_BYTES + 1)) == A.SSE_ERR_ARG   # 24-bit work-item length
    assert _init_ex(cfg, line_pool(64, max_line_bytes=cfg.carry_slot_bytes - 16)) == A.SSE_ERR_ARG   # below the carry slot
    fused = _cfg()
    fused.flags = A.FLAG_KERNEL_FUSED
    assert _init_ex(fused, line_pool(64)) == A.SSE_ERR_ARG                      # the tile kernel has no pool
    assert _init_ex(fused, line_pool(0)) == A.SSE_ERR_ARG
    # the grown out arena must keep arena offsets 31-bit: 1 MiB of input per batch, a 16 GiB pool
    assert _init_ex(cfg, line_pool(1 << 18)) == A.SSE_ERR_ARG
    bad_cfg = A.Config()                                                          # config checks still come first
    assert _init_ex(bad_cfg, line_pool(64)) == A.SSE_ERR_ARG


def test_init_ex_without_pool_or_with_good_pool_needs_a_device():
    import torch
    if torch.cuda.is_available():
        return
    assert _init_ex(_cfg(), None) == A.SSE_ERR_NO_DEVICE
    assert _init_ex(_cfg(), line_pool(64)) == A.SSE_ERR_NO_DEVICE
    assert _init_ex(_cfg(), line_pool(0, max_line_bytes=16384)) == A.SSE_ERR_NO_DEVICE


def _grown(cfg, pool):
    L = A.load()
    out = A.Config()
    C.memmove(C.byref(out), C.byref(cfg), C.sizeof(A.Config))
    L.sse_line_pool_config(C.byref(out), C.byref(pool) if pool is not None else None)
    return out


def test_pool_config_grows_every_capacity_at_the_config_ratio():
    for worst in (False, True):
        for pages, page in ((16, 0), (100, 4096), (7, 65536 + 16)):
            cfg = _cfg(worst)
            g = _grown(cfg, line_pool(pages, page_bytes=page))
            extra = pages * (page or 65536)
            ib = cfg.in_arena_bytes
            for name in GROWN:
                x = getattr(cfg, name)
                want = min(x + -(-x * extra // ib), CAP)
                assert getattr(g, name) == want, (worst, pages, page, name)
            for name, _ in A.Config._fields_:
                if name not in GROWN:
                    assert getattr(g, name) == getattr(cfg, name), name


def test_pool_config_null_or_empty_pool_leaves_the_config_unchanged():
    cfg = _cfg(True)
    raw = bytes(memoryview(cfg))
    assert bytes(memoryview(_grown(cfg, None))) == raw
    assert bytes(memoryview(_grown(cfg, line_pool(0)))) == raw
    assert bytes(memoryview(_grown(cfg, line_pool(0, page_bytes=4096)))) == raw


def test_worst_case_config_with_a_pool_still_covers_every_pooled_byte():
    """sse_worst_case_config admits one frame per input byte; with a pool it admits one per input or pooled byte."""
    cfg = _cfg(True, conns=64, batch=1 << 20)
    pool = line_pool(32)
    g = _grown(cfg, pool)
    assert g.max_frames >= cfg.in_arena_bytes + 32 * 65536
    assert g.out_arena_bytes >= cfg.out_arena_bytes + 32 * 65536
