"""ctypes binding of the CPU oracle (oracle/sse_oracle.c).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs -- never by the product package.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass, field

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "liborc.so")


def build(force: bool = False) -> str:
    srcs = [os.path.join(_HERE, f) for f in ("sse_oracle.c", "sse_oracle.h", "orc_bench.c", "orc_check.c", "Makefile")]
    if force or not os.path.exists(_LIB_PATH) or any(
            os.path.getmtime(s) > os.path.getmtime(_LIB_PATH) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-s", "-B"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


class Span(C.Structure):
    _fields_ = [("off", C.c_uint32), ("len", C.c_uint32)]


class Tc(C.Structure):
    _fields_ = [("index", C.c_int64), ("has_id", C.c_uint32), ("has_type", C.c_uint32),
                ("has_function", C.c_uint32), ("pad", C.c_uint32),
                ("id", Span), ("type", Span), ("name", Span), ("args", Span)]


class Chunk(C.Structure):
    _fields_ = [("json_ok", C.c_uint32), ("n_choices", C.c_uint32), ("finish", C.c_uint32),
                ("has_usage", C.c_uint32), ("prompt", C.c_int64), ("completion", C.c_int64),
                ("total", C.c_int64), ("content", Span), ("tool_calls_nonnil", C.c_uint32),
                ("tc_first", C.c_uint32), ("tc_count", C.c_uint32), ("has_valid_tool_call", C.c_uint32)]


class Line(C.Structure):
    _fields_ = [("line_off", C.c_uint32), ("line_len", C.c_uint32), ("out_off", C.c_uint32),
                ("out_len", C.c_uint32), ("kind", C.c_uint32), ("chunk", C.c_uint32), ("pay_off", C.c_uint32),
                ("pay_len", C.c_uint32)]


class Result(C.Structure):
    _fields_ = [("out", C.POINTER(C.c_uint8)), ("out_len", C.c_size_t), ("out_cap", C.c_size_t),
                ("text", C.POINTER(C.c_uint8)), ("text_len", C.c_size_t), ("text_cap", C.c_size_t),
                ("lines", C.POINTER(Line)), ("n_lines", C.c_size_t), ("cap_lines", C.c_size_t),
                ("chunks", C.POINTER(Chunk)), ("n_chunks", C.c_size_t), ("cap_chunks", C.c_size_t),
                ("tcs", C.POINTER(Tc)), ("n_tcs", C.c_size_t), ("cap_tcs", C.c_size_t),
                ("acc_content", Span), ("has_tool_calls", C.c_uint32), ("terminated", C.c_uint32),
                ("term_finish", C.c_uint32), ("tail_len", C.c_size_t)]


class Call(C.Structure):
    _fields_ = [("id", Span), ("type", Span), ("name", Span), ("args", Span)]


class Usage(C.Structure):
    _fields_ = [("prompt", C.c_int64), ("completion", C.c_int64), ("total", C.c_int64)]


L_DROPPED, L_EMITTED, L_DONE, L_UNREAD, L_DONE_EXACT = 0, 1, 2, 3, 4
JSON_OK, JSON_SYNTAX, JSON_DEPTH = 0, 1, 2
DEPTH_LIMIT = 128
FIN_NONE, FIN_STOP, FIN_TOOL_CALLS, FIN_LENGTH, FIN_CONTENT_FILTER, FIN_FUNCTION_CALL, FIN_OTHER = 0, 1, 2, 3, 4, 5, 7

_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.orc_result_new.restype = C.POINTER(Result)
        _lib.orc_result_free.argtypes = [C.POINTER(Result)]
        _lib.orc_result_clear.argtypes = [C.POINTER(Result)]
        _lib.orc_trim_space.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
        _lib.orc_json_valid.argtypes = [C.c_char_p, C.c_size_t]
        _lib.orc_json_valid.restype = C.c_int
        _lib.orc_json_scan.argtypes = [C.c_char_p, C.c_size_t, C.c_int]
        _lib.orc_json_scan.restype = C.c_int
        _lib.orc_unmarshal_chunk.argtypes = [C.POINTER(Result), C.c_char_p, C.c_size_t]
        _lib.orc_unmarshal_chunk.restype = C.c_uint32
        _lib.orc_passthrough.argtypes = [C.POINTER(Result), C.c_char_p, C.c_size_t, C.c_int]
        _lib.orc_reframe_stream.argtypes = [C.POINTER(Result), C.c_char_p, C.c_size_t, C.c_int]
        _lib.orc_parse_tool_calls.argtypes = [C.POINTER(Result), C.c_char_p, C.c_size_t, C.POINTER(Call), C.c_size_t]
        _lib.orc_parse_tool_calls.restype = C.c_size_t
        _lib.orc_telemetry.argtypes = [C.POINTER(Result), C.c_char_p, C.c_size_t, C.POINTER(Usage),
                                       C.POINTER(Call), C.c_size_t]
        _lib.orc_telemetry.restype = C.c_size_t
        _lib.orc_last_builder.argtypes = [C.POINTER(Result), C.POINTER(C.c_size_t)]
        _lib.orc_last_builder.restype = C.POINTER(C.c_uint8)
        _lib.orc_bench_run.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int,
                                       C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        _lib.orc_bench_run.restype = C.c_double
        _lib.orc_digest_init.argtypes = [C.c_void_p, C.c_size_t]
        _lib.orc_digest_init.restype = None
        _lib.orc_digest_streams.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int,
                                            C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.orc_digest_streams.restype = None
        _lib.orc_digest_result.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.orc_digest_result.restype = C.c_uint32
        _lib.orc_check_result.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_char_p, C.c_size_t]
        _lib.orc_check_result.restype = C.c_uint32
    return _lib


# ---------------------------------------------------------------- pythonic views
@dataclass
class ToolCallChunk:
    index: int
    id: bytes | None
    type: bytes | None
    function: bool
    name: bytes
    args: bytes


@dataclass
class ChunkView:
    json_ok: bool
    n_choices: int = 0
    finish: int = 0
    usage: tuple | None = None
    content: bytes = b""
    tool_calls_nonnil: bool = False
    tool_calls: list = field(default_factory=list)
    has_valid_tool_call: bool = False


@dataclass
class LineView:
    line: bytes
    kind: int
    out: bytes
    chunk: ChunkView | None
    payload: bytes = b""        # what the line handed to json.Unmarshal (the "[DONE]" a DONE_EXACT line did not decode)

    @property
    def payload_len(self) -> int:
        return len(self.payload)

    @property
    def depth_limited(self) -> bool:
        """The payload hits the product's documented nesting limit (DESIGN.md §5, deviation 2)."""
        return self.chunk is not None and json_scan(self.payload, DEPTH_LIMIT) == JSON_DEPTH


@dataclass
class StreamView:
    out: bytes
    lines: list
    acc_content: bytes = b""
    has_tool_calls: bool = False
    terminated: bool = False
    term_finish: int = 0
    tail_len: int = 0
    builder: bytes = b""


def _txt(r, sp):
    return bytes(C.string_at(r.text, r.text_len)[sp.off:sp.off + sp.len]) if sp.len else b""


def _chunk_view(r, ci) -> ChunkView:
    ck = r.chunks[ci]
    if not ck.json_ok:
        return ChunkView(False)
    text = C.string_at(r.text, r.text_len) if r.text_len else b""
    g = lambda sp: text[sp.off:sp.off + sp.len]
    tcs = []
    for i in range(ck.tc_count):
        t = r.tcs[ck.tc_first + i]
        tcs.append(ToolCallChunk(t.index, g(t.id) if t.has_id else None, g(t.type) if t.has_type else None,
                                 bool(t.has_function), g(t.name), g(t.args)))
    return ChunkView(True, ck.n_choices, ck.finish,
                     (ck.prompt, ck.completion, ck.total) if ck.has_usage else None,
                     g(ck.content), bool(ck.tool_calls_nonnil), tcs, bool(ck.has_valid_tool_call))


def unmarshal(payload: bytes) -> ChunkView:
    L = lib()
    rp = L.orc_result_new()
    try:
        ci = L.orc_unmarshal_chunk(rp, payload, len(payload))
        return _chunk_view(rp.contents, ci)
    finally:
        L.orc_result_free(rp)


def json_valid(payload: bytes) -> bool:
    return bool(lib().orc_json_valid(payload, len(payload)))


def json_scan(payload: bytes, max_depth: int = 10000) -> int:
    """checkValid with a nesting limit: JSON_OK, JSON_SYNTAX, or JSON_DEPTH when a container opens while max_depth are open
    before the first syntax error."""
    return lib().orc_json_scan(payload, len(payload), max_depth)


def trim_space(s: bytes) -> bytes:
    a, b = C.c_size_t(), C.c_size_t()
    lib().orc_trim_space(s, len(s), C.byref(a), C.byref(b))
    return s[a.value:b.value]


def _stream_view(L, rp, data: bytes, with_builder: bool) -> StreamView:
    r = rp.contents
    out = C.string_at(r.out, r.out_len) if r.out_len else b""
    lines = []
    for i in range(r.n_lines):
        ln = r.lines[i]
        lines.append(LineView(data[ln.line_off:ln.line_off + ln.line_len], ln.kind,
                              out[ln.out_off:ln.out_off + ln.out_len],
                              _chunk_view(r, ln.chunk) if ln.chunk != 0xFFFFFFFF else None,
                              data[ln.pay_off:ln.pay_off + ln.pay_len]))
    b = b""
    if with_builder:
        n = C.c_size_t()
        p = L.orc_last_builder(rp, C.byref(n))
        b = C.string_at(p, n.value) if n.value else b""
    return StreamView(out, lines, _txt(r, r.acc_content), bool(r.has_tool_calls), bool(r.terminated),
                      r.term_finish, r.tail_len, b)


def passthrough(data: bytes, parse: bool = False) -> StreamView:
    L = lib()
    rp = L.orc_result_new()
    try:
        L.orc_passthrough(rp, data, len(data), int(parse))
        return _stream_view(L, rp, data, False)
    finally:
        L.orc_result_free(rp)


def reframe(data: bytes, append_done: bool = False) -> StreamView:
    L = lib()
    rp = L.orc_result_new()
    try:
        L.orc_reframe_stream(rp, data, len(data), int(append_done))
        return _stream_view(L, rp, data, True)
    finally:
        L.orc_result_free(rp)


def _calls(r, arr, n):
    text = C.string_at(r.text, r.text_len) if r.text_len else b""
    g = lambda sp: text[sp.off:sp.off + sp.len]
    return [dict(id=g(arr[i].id), type=g(arr[i].type), name=g(arr[i].name), args=g(arr[i].args)) for i in range(n)]


def parse_tool_calls(body: bytes, cap: int = 256):
    L = lib()
    rp = L.orc_result_new()
    try:
        arr = (Call * cap)()
        n = L.orc_parse_tool_calls(rp, body, len(body), arr, cap)
        return _calls(rp.contents, arr, min(n, cap))
    finally:
        L.orc_result_free(rp)


def telemetry(body: bytes, cap: int = 256):
    L = lib()
    rp = L.orc_result_new()
    try:
        arr = (Call * cap)()
        u = Usage()
        n = L.orc_telemetry(rp, body, len(body), C.byref(u), arr, cap)
        return (u.prompt, u.completion, u.total), _calls(rp.contents, arr, min(n, cap))
    finally:
        L.orc_result_free(rp)


def bench_run(arena, off, length, mode, n_threads: int, passes: int = 1):
    """arena: np.uint8 array; off: np.uint64; length: np.uint32; mode: np.uint8 (bit0 R, bit1 parse).
    One pool of n_threads threads runs `passes` passes over the streams. Returns (seconds, out_bytes, frames, chunks_ok),
    totals over all passes."""
    L = lib()
    ob, fr, ok = C.c_uint64(), C.c_uint64(), C.c_uint64()
    secs = L.orc_bench_run(arena.ctypes.data, off.ctypes.data, length.ctypes.data, mode.ctypes.data,
                           len(off), n_threads, passes, C.byref(ob), C.byref(fr), C.byref(ok))
    return secs, ob.value, fr.value, ok.value


# ---------------------------------------------------------------- full-size parity digests (orc_check.c)
def _digest_dtype():
    import numpy as np
    return np.dtype([("frames_h", "<u8"), ("recs_h", "<u8"), ("n_frames", "<u8"), ("n_recs", "<u8"), ("frame_bytes", "<u8"),
                     ("inexact", "<u4"), ("pad", "<u4")])


def new_digests(n: int):
    import numpy as np
    d = np.zeros(n, dtype=_digest_dtype())
    lib().orc_digest_init(d.ctypes.data, n)
    return d


def digest_streams(arena, off, length, mode, n_threads: int):
    """Oracle digests of whole bodies: arena uint8[], off uint64[], length uint32[], mode uint8[] (bit0 R, bit1 parse).
    Returns (digests, terminated uint8[], tail_len uint32[])."""
    import numpy as np
    n = len(off)
    d = new_digests(n)
    term = np.zeros(n, dtype=np.uint8)
    tail = np.zeros(n, dtype=np.uint32)
    lib().orc_digest_streams(arena.ctypes.data, off.ctypes.data, length.ctypes.data, mode.ctypes.data, n, n_threads,
                             d.ctypes.data, term.ctypes.data, tail.ctypes.data)
    return d, term, tail


def digest_result(raw_result, conn, digests, carry_len, seg_flags) -> int:
    """Folds one sse_result (ctypes struct of the product's C ABI, passed by reference) into per-connection digests."""
    return lib().orc_digest_result(C.addressof(raw_result), conn.ctypes.data, digests.ctypes.data, carry_len.ctypes.data,
                                   seg_flags.ctypes.data)


def check_result(raw_result, segs, flags: int, max_line: int) -> tuple[int, str]:
    """Structural check of one sse_result (ctypes struct, by reference) against the submitted sse_seg descriptors (a numpy
    array of sse_seg records, at least n_segs long) of an engine with sse_config.flags `flags` whose longest line is max_line.
    Returns (number of violations, description of the first)."""
    import numpy as np
    segs = np.ascontiguousarray(segs)
    msg = C.create_string_buffer(512)
    n = lib().orc_check_result(C.addressof(raw_result), segs.ctypes.data, flags, max_line, msg, len(msg))
    return n, msg.value.decode()
