"""ctypes mirror of include/sse_gpu.h (the C ABI of libssegpu.so)."""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

SSE_OK, SSE_ERR_NO_DEVICE, SSE_ERR_CUDA, SSE_ERR_ARG, SSE_ERR_BUSY, SSE_ERR_OVERFLOW, SSE_ERR_NOMEM, SSE_ERR_UNDECODED = 0, -1, -2, -3, -4, -5, -6, -7
MODE_P, MODE_R, MODE_PARSE = 0, 1, 2
FLAG_KERNEL_FUSED, FLAG_COPY_OUT, FLAG_TEMPLATES, FLAG_DEFER, FLAG_COUNTERS = 4, 8, 16, 64, 256
NONE = 0xFFFFFFFF
MAX_LINE_BYTES = 16777215   # SSE_MAX_LINE_BYTES: decode work items carry a 24-bit payload length

F_JSON_OK, F_HAS_USAGE, F_TC_NONNIL, F_TC_VALID, F_CONTENT_TEXT = 0x1, 0x2, 0x4, 0x8, 0x10
F_DONE_LINE, F_DONE_EXACT, F_TERMINATES, F_DEPTH_LIMIT, F_TOO_LONG = 0x20, 0x40, 0x80, 0x100, 0x200
F_FINISH_SHIFT, F_FINISH_MASK = 12, 0x7000
TC_HAS_ID, TC_HAS_TYPE, TC_HAS_FUNC = 0x1, 0x2, 0x4
TC_ID_TEXT, TC_TYPE_TEXT, TC_NAME_TEXT, TC_ARGS_TEXT = 0x10, 0x20, 0x40, 0x80
SEG_TERMINATED, SEG_FINISHED, SEG_LINE_TOO_LONG, SEG_DEAD, SEG_DEFERRED = 0x1, 0x2, 0x4, 0x8, 0x10
OVF_OUT, OVF_TCS, OVF_USAGES, OVF_TEXT, OVF_RUNS, OVF_POOL = 0x1, 0x2, 0x4, 0x8, 0x10, 0x20


class Config(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in (
        "struct_size", "max_conns", "max_segs", "in_arena_bytes", "out_arena_bytes", "max_frames", "max_recs",
        "max_tcs", "max_usages", "text_arena_bytes", "max_runs", "carry_slot_bytes", "n_slots", "flags")]


class LinePool(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("struct_size", "page_bytes", "pool_pages", "max_line_bytes")]


class Seg(C.Structure):
    _fields_ = [("conn", C.c_uint32), ("in_off", C.c_uint32), ("in_len", C.c_uint32),
                ("mode", C.c_uint8), ("provider", C.c_uint8), ("reserved", C.c_uint16)]


class Frame(C.Structure):
    _fields_ = [("off", C.c_uint32), ("len", C.c_uint32)]


class Rec(C.Structure):
    _fields_ = [("frame", C.c_uint32), ("flags", C.c_uint32), ("content_off", C.c_uint32),
                ("content_len", C.c_uint32), ("tc_first", C.c_uint32), ("tc_count", C.c_uint16),
                ("n_choices", C.c_uint16), ("usage", C.c_uint32), ("payload_len", C.c_uint32)]


class Tc(C.Structure):
    _fields_ = [("index", C.c_int64), ("flags", C.c_uint32), ("next", C.c_uint32),
                ("id_off", C.c_uint32), ("id_len", C.c_uint32), ("type_off", C.c_uint32), ("type_len", C.c_uint32),
                ("name_off", C.c_uint32), ("name_len", C.c_uint32), ("args_off", C.c_uint32), ("args_len", C.c_uint32)]


class Usage(C.Structure):
    _fields_ = [("prompt_tokens", C.c_int64), ("completion_tokens", C.c_int64), ("total_tokens", C.c_int64)]


class Run(C.Structure):
    _fields_ = [("frame_first", C.c_uint32), ("frame_count", C.c_uint32), ("rec_first", C.c_uint32),
                ("rec_count", C.c_uint32), ("next", C.c_uint32)]


class SegResult(C.Structure):
    _fields_ = [("run", Run), ("carry_len", C.c_uint32), ("flags", C.c_uint32), ("consumed", C.c_uint32)]


class Result(C.Structure):
    _fields_ = [("status", C.c_int32), ("n_segs", C.c_uint32), ("n_frames", C.c_uint32), ("n_recs", C.c_uint32),
                ("n_tcs", C.c_uint32), ("n_usages", C.c_uint32), ("n_runs", C.c_uint32),
                ("out_bytes", C.c_uint32), ("text_bytes", C.c_uint32),
                ("out", C.POINTER(C.c_uint8)), ("frames", C.POINTER(Frame)), ("recs", C.POINTER(Rec)),
                ("tcs", C.POINTER(Tc)), ("usages", C.POINTER(Usage)), ("text", C.POINTER(C.c_uint8)),
                ("runs", C.POINTER(Run)), ("segs", C.POINTER(SegResult)),
                ("n_decoded", C.c_uint32), ("n_derived", C.c_uint32), ("overflow", C.c_uint32),
                ("in_base", C.c_uint32), ("in_", C.POINTER(C.c_uint8))]


class Batch(C.Structure):
    _fields_ = [("in_arena", C.POINTER(C.c_uint8)), ("segs", C.POINTER(Seg)),
                ("in_arena_bytes", C.c_uint32), ("max_segs", C.c_uint32)]


class Bytes(C.Structure):
    _fields_ = [("p", C.POINTER(C.c_uint8)), ("n", C.c_size_t)]


class ToolCall(C.Structure):
    _fields_ = [("id", Bytes), ("type", Bytes), ("name", Bytes), ("arguments", Bytes)]


# sse_counters (SSE_FLAG_COUNTERS): the uint64_t fields in header order
COUNTER_FIELDS = (
    "p_segments", "p_segments_skipped", "p_windows", "p_window_bytes", "p_rounds", "p_lines", "p_frames_zero_copy",
    "p_frames_materialised", "p_bytes_materialised", "p_items", "p_long_lines", "p_pool_pages_taken", "p_pool_pages_returned",
    "p_deferred_rounds",
    "d_items", "d_pulls", "d_items_per_pull", "d_warp_rounds", "d_busy_lane_rounds", "d_skip_windows", "d_skip_bytes",
    "d_coop_strings", "d_coop_steps", "d_coop_bytes", "d_plain_steps", "d_actions", "d_action_redos", "d_abandoned_bytes",
    "d_template_lines", "d_template_bytes", "d_template_misses", "d_unquote_jobs", "d_unquote_bytes", "d_lines_finished",
    "c_total", "c_pull", "c_skip", "c_coop", "c_steps", "c_finish", "c_unquote")


class Counters(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("decode_passes", C.c_uint32)] + [(n, C.c_uint64) for n in COUNTER_FIELDS]


def counters_dict(k: Counters) -> dict:
    d = {n: int(getattr(k, n)) for n in COUNTER_FIELDS}
    d["decode_passes"] = int(k.decode_passes)
    return d


assert C.sizeof(Seg) == 16 and C.sizeof(Rec) == 32 and C.sizeof(Tc) == 48 and C.sizeof(SegResult) == 32

EXPORTS = [
    "sse_init", "sse_init_ex", "sse_line_pool_config", "sse_line_pool_stats", "sse_line_pool_set_growth", "sse_line_pool_capacity",
    "sse_trim", "sse_memory_held",
    "sse_destroy", "sse_strerror", "sse_last_cuda_error", "sse_abi_version", "sse_default_config", "sse_worst_case_config",
    "sse_acquire", "sse_submit", "sse_poll", "sse_collect", "sse_release", "sse_reset_conn", "sse_reset_all",
    "sse_upload", "sse_launch", "sse_download", "sse_launch_count", "sse_at", "sse_counters_read",
    "sse_agent_new", "sse_agent_free", "sse_agent_reset", "sse_agent_feed", "sse_agent_content",
    "sse_agent_has_tool_calls", "sse_agent_terminated", "sse_agent_tool_calls",
    "sse_telemetry_new", "sse_telemetry_free", "sse_telemetry_reset", "sse_telemetry_feed", "sse_telemetry_feed_bytes", "sse_telemetry_finish",
]

_lib = None


def lib_path() -> str:
    return _build.LIB


def load(build_if_missing: bool = True):
    """Loads libssegpu.so. There is no fallback: a missing library is an error."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path) or (build_if_missing and _build.needs_build()):
        if not build_if_missing:
            raise RuntimeError(f"{path} is missing: build it with `python -m inference_gateway_b200.build`")
        _build.build()
    L = C.CDLL(path)
    vp, u32, i32 = C.c_void_p, C.c_uint32, C.c_int
    L.sse_init.argtypes = [i32, C.POINTER(Config), C.POINTER(vp)]
    L.sse_init_ex.argtypes = [i32, C.POINTER(Config), C.POINTER(LinePool), C.POINTER(vp)]
    L.sse_line_pool_config.argtypes = [C.POINTER(Config), C.POINTER(LinePool)]
    L.sse_line_pool_config.restype = None
    L.sse_line_pool_stats.argtypes = [vp, C.POINTER(u32), C.POINTER(u32)]
    L.sse_line_pool_set_growth.argtypes = [vp, u32]
    L.sse_line_pool_capacity.argtypes = [vp, C.POINTER(u32), C.POINTER(u32)]
    L.sse_trim.argtypes = [vp, u32]
    L.sse_memory_held.argtypes = [vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.sse_destroy.argtypes = [vp]
    L.sse_destroy.restype = None
    L.sse_strerror.argtypes = [i32]
    L.sse_strerror.restype = C.c_char_p
    L.sse_last_cuda_error.restype = C.c_char_p
    L.sse_default_config.argtypes = [C.POINTER(Config), u32, u32]
    L.sse_default_config.restype = None
    L.sse_worst_case_config.argtypes = [C.POINTER(Config), u32, u32]
    L.sse_worst_case_config.restype = None
    L.sse_acquire.argtypes = [vp, C.POINTER(i32), C.POINTER(Batch)]
    L.sse_submit.argtypes = [vp, i32, u32, u32]
    L.sse_poll.argtypes = [vp, i32]
    L.sse_collect.argtypes = [vp, i32, C.POINTER(Result)]
    L.sse_release.argtypes = [vp, i32]
    L.sse_reset_conn.argtypes = [vp, u32]
    L.sse_reset_all.argtypes = [vp, vp]
    L.sse_upload.argtypes = [vp, i32, u32, u32, vp]
    L.sse_launch.argtypes = [vp, i32, u32, vp]
    L.sse_download.argtypes = [vp, i32, C.POINTER(Result), vp]
    L.sse_launch_count.argtypes = [vp, C.POINTER(C.c_uint64)]
    L.sse_counters_read.argtypes = [vp, i32, C.POINTER(Counters)]
    L.sse_at.argtypes = [C.POINTER(Result), u32]
    L.sse_at.restype = C.POINTER(C.c_uint8)
    if hasattr(L, "ssegw_mcp_writer_step"):
        L.ssegw_mcp_writer_step.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_int)]
        L.ssegw_mcp_writer_step.restype = C.c_int
    L.sse_agent_new.restype = vp
    L.sse_agent_free.argtypes = [vp]
    L.sse_agent_free.restype = None
    L.sse_agent_reset.argtypes = [vp]
    L.sse_agent_reset.restype = None
    L.sse_agent_feed.argtypes = [vp, C.POINTER(Result), u32]
    L.sse_agent_content.argtypes = [vp]
    L.sse_agent_content.restype = Bytes
    L.sse_agent_has_tool_calls.argtypes = [vp]
    L.sse_agent_terminated.argtypes = [vp, C.POINTER(i32)]
    L.sse_agent_tool_calls.argtypes = [vp, C.POINTER(ToolCall), C.c_size_t]
    L.sse_agent_tool_calls.restype = C.c_size_t
    L.sse_telemetry_new.restype = vp
    L.sse_telemetry_free.argtypes = [vp]
    L.sse_telemetry_free.restype = None
    L.sse_telemetry_reset.argtypes = [vp]
    L.sse_telemetry_reset.restype = None
    L.sse_telemetry_feed.argtypes = [vp, C.POINTER(Result), u32]
    L.sse_telemetry_feed_bytes.argtypes = [vp, C.c_char_p, C.c_size_t]
    L.sse_telemetry_finish.argtypes = [vp, C.POINTER(Usage), C.POINTER(ToolCall), C.c_size_t, C.POINTER(C.c_size_t)]
    _lib = L
    return L


class SseError(RuntimeError):
    def __init__(self, status: int, where: str):
        L = load()
        msg = L.sse_strerror(status).decode()
        if status == SSE_ERR_CUDA:
            msg += ": " + L.sse_last_cuda_error().decode()
        super().__init__(f"{where}: {msg} ({status})")
        self.status = status


def check(status: int, where: str) -> None:
    if status != SSE_OK:
        raise SseError(status, where)
