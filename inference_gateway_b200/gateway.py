"""ctypes view of the host-side mirror (include/sse_gateway.h): a provider whose StreamChatCompletions returns a
channel of lines, the batcher tick, and the MCP agent's per-iteration view. Plumbing only."""
from __future__ import annotations

import ctypes as C

from . import _abi as A


def _bytes(b: A.Bytes) -> bytes:
    return C.string_at(b.p, b.n) if b.n else b""


class Telemetry:
    """One telemetry fold (sse_telemetry_*): api/middlewares/telemetry.go:190-277 over one client response. Attach it to the
    upstream streams that make up the response (Gateway.stream_chat_completions / proxy_stream, one open at a time) and
    feed what the handler writes itself (the agent's final [DONE], error frames) with feed_bytes."""

    def __init__(self):
        self.L = A.load()
        self.f = self.L.sse_telemetry_new()
        if not self.f:
            raise MemoryError("sse_telemetry_new")

    def feed_bytes(self, b: bytes):
        A.check(self.L.sse_telemetry_feed_bytes(self.f, b, len(b)), "sse_telemetry_feed_bytes")

    def finish(self):
        """(rc, (prompt, completion, total), tool calls): rc 1 when a piece of the body was irregular (DESIGN.md §5,
        deviation 4), else 0. Feed nothing after it."""
        u, n = A.Usage(), C.c_size_t()
        rc = self.L.sse_telemetry_finish(self.f, C.byref(u), None, 0, C.byref(n))
        arr = (A.ToolCall * max(1, n.value))()
        if n.value:
            rc = self.L.sse_telemetry_finish(self.f, C.byref(u), arr, n.value, C.byref(n))
        if rc < 0:
            raise A.SseError(rc, "sse_telemetry_finish")
        calls = [dict(id=_bytes(c.id), type=_bytes(c.type), name=_bytes(c.name), args=_bytes(c.arguments)) for c in arr[:n.value]]
        return rc, (u.prompt_tokens, u.completion_tokens, u.total_tokens), calls

    def close(self):
        """Frees the fold: only once no open stream of a gateway feeds it."""
        if self.f:
            self.L.sse_telemetry_free(self.f)
            self.f = None


class Gateway:
    def __init__(self, device: int = 0, max_conns: int = 256, bytes_per_batch: int = 1 << 20, line_pool: dict | None = None,
                 config: A.Config | None = None, devices: list[int] | None = None, depth: int = 1):
        """line_pool: keyword arguments of engine.make_line_pool() (pool_pages, page_bytes, max_line_bytes): lines longer than the
        64 KiB carry slot continue in a shared device page pool instead of failing their stream. max_pages in it
        (ssegw_line_pool_growth; a config with FLAG_DEFER) lets every context's pool grow on demand up to that many pages.
        config: an sse_config to run on (ssegw_new_cfg; max_conns and bytes_per_batch are then ignored), e.g. default capacities
        with FLAG_DEFER; None: the worst-case config.
        devices, depth: one context per entry of devices (a device may repeat), each with up to depth (1 .. config.n_slots)
        batches in flight (ssegw_new_multi; needs config). Stream id = context index * config.max_conns + connection. With depth
        above 1 a pump delivers what earlier pumps submitted; flush() collects the rest. depth alone runs on [device]."""
        from .engine import make_line_pool
        self.L = L = A.load()
        vp, i32 = C.c_void_p, C.c_int
        L.ssegw_new.argtypes = [i32, C.c_uint32, C.c_uint32, C.POINTER(i32)]
        L.ssegw_new.restype = vp
        L.ssegw_new_ex.argtypes = [i32, C.c_uint32, C.c_uint32, C.POINTER(A.LinePool), C.POINTER(i32)]
        L.ssegw_new_ex.restype = vp
        L.ssegw_new_cfg.argtypes = [i32, C.POINTER(A.Config), C.POINTER(A.LinePool), C.POINTER(i32)]
        L.ssegw_new_cfg.restype = vp
        L.ssegw_new_multi.argtypes = [C.POINTER(i32), C.c_uint32, C.POINTER(A.Config), C.POINTER(A.LinePool), C.c_uint32,
                                      C.POINTER(i32)]
        L.ssegw_new_multi.restype = vp
        L.ssegw_flush.argtypes = [vp]
        L.ssegw_free.argtypes = [vp]
        L.ssegw_free.restype = None
        L.ssegw_stream_chat_completions.argtypes = [vp, C.c_uint8]
        L.ssegw_stream_with_telemetry.argtypes = [vp, C.c_uint8, vp]
        L.ssegw_upstream_write.argtypes = [vp, i32, C.c_char_p, C.c_size_t]
        L.ssegw_upstream_write.restype = C.c_size_t
        L.ssegw_upstream_close.argtypes = [vp, i32]
        L.ssegw_upstream_close.restype = None
        L.ssegw_pump.argtypes = [vp]
        L.ssegw_recv.argtypes = [vp, i32, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.ssegw_agent_recv.argtypes = [vp, i32, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.ssegw_proxy_stream.argtypes = [vp]
        L.ssegw_proxy_step.argtypes = [vp, i32, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.ssegw_release_stream.argtypes = [vp, i32]
        L.ssegw_release_stream.restype = None
        L.ssegw_agent_content.argtypes = [vp, i32]
        L.ssegw_agent_content.restype = A.Bytes
        L.ssegw_agent_has_tool_calls.argtypes = [vp, i32]
        L.ssegw_agent_terminated.argtypes = [vp, i32, C.POINTER(i32)]
        L.ssegw_agent_tool_calls.argtypes = [vp, i32, C.POINTER(A.ToolCall), C.c_size_t]
        L.ssegw_agent_tool_calls.restype = C.c_size_t
        L.ssegw_counters.argtypes = [vp, C.POINTER(A.Counters)]
        L.ssegw_line_pool_growth.argtypes = [vp, C.c_uint32]
        L.ssegw_trim.argtypes = [vp, C.c_uint32]
        st = i32()
        line_pool = dict(line_pool) if line_pool is not None else None
        max_pages = line_pool.pop("max_pages", 0) if line_pool is not None else 0
        self._pool = make_line_pool(**line_pool) if line_pool is not None else None
        if devices is not None or depth != 1:
            if config is None:
                raise ValueError("devices / depth need an sse_config (config=)")
            devs = list(devices) if devices is not None else [device]
            arr = (i32 * max(1, len(devs)))(*devs)
            self.g = L.ssegw_new_multi(arr, len(devs), C.byref(config), C.byref(self._pool) if self._pool is not None else None,
                                       depth, C.byref(st))
        elif config is not None:
            self.g = L.ssegw_new_cfg(device, C.byref(config), C.byref(self._pool) if self._pool is not None else None, C.byref(st))
        elif line_pool is None:
            self.g = L.ssegw_new(device, max_conns, bytes_per_batch, C.byref(st))
        else:
            self.g = L.ssegw_new_ex(device, max_conns, bytes_per_batch, C.byref(self._pool), C.byref(st))
        if not self.g:
            raise A.SseError(st.value, "ssegw_new")
        if max_pages:
            rc = L.ssegw_line_pool_growth(self.g, max_pages)
            if rc != A.SSE_OK:
                L.ssegw_free(self.g)
                self.g = None
                raise A.SseError(rc, "ssegw_line_pool_growth")
        self._buf = C.create_string_buffer(1 << 20)
        self._taps = {}          # stream id -> the Telemetry it feeds, kept alive until the stream is released

    def close(self):
        if self.g:
            self.L.ssegw_free(self.g)
            self.g = None
            self._taps.clear()

    def _open(self, mode: int, telemetry: Telemetry | None) -> int:
        if telemetry is None:
            sid = self.L.ssegw_stream_chat_completions(self.g, mode)
        else:
            sid = self.L.ssegw_stream_with_telemetry(self.g, mode, telemetry.f)
            if sid < -1:
                raise A.SseError(sid, "ssegw_stream_with_telemetry")
        if sid < 0:
            raise RuntimeError("no free connection slot")
        if telemetry is not None:
            self._taps[sid] = telemetry
        return sid

    def stream_chat_completions(self, mode: int, telemetry: Telemetry | None = None) -> int:
        """telemetry: the response's fold, fed from this stream's records (mode must have MODE_PARSE or MODE_R; a fold
        feeds one open stream at a time: SseError SSE_ERR_BUSY otherwise)."""
        return self._open(mode, telemetry)

    def upstream_write(self, sid: int, data: bytes) -> int:
        return self.L.ssegw_upstream_write(self.g, sid, data, len(data))

    def upstream_close(self, sid: int):
        self.L.ssegw_upstream_close(self.g, sid)

    def pump(self) -> int:
        rc = self.L.ssegw_pump(self.g)
        if rc < 0:
            raise A.SseError(rc, "ssegw_pump")
        return rc

    def flush(self) -> int:
        """ssegw_flush: collects every batch still in flight; returns the frames delivered."""
        rc = self.L.ssegw_flush(self.g)
        if rc < 0:
            raise A.SseError(rc, "ssegw_flush")
        return rc

    def _recv(self, fn, sid):
        n = C.c_size_t()
        rc = fn(self.g, sid, self._buf, len(self._buf), C.byref(n))
        if rc == A.SSE_ERR_ARG and n.value > len(self._buf):   # an element longer than the buffer (a pooled line): grow, retry
            self._buf = C.create_string_buffer(n.value)
            rc = fn(self.g, sid, self._buf, len(self._buf), C.byref(n))
        if rc == 1:
            return self._buf.raw[:n.value]
        if rc == 0:
            return None
        if rc == -1:
            raise EOFError
        raise A.SseError(rc, "recv")

    def recv(self, sid: int):
        """One channel element, None if nothing is available yet; raises EOFError when the channel is closed."""
        return self._recv(self.L.ssegw_recv, sid)

    def proxy_stream(self, telemetry: Telemetry | None = None) -> int:
        """handleStreamingRequest (api/routes.go:129-232): the raw /proxy stream. With telemetry, a MODE_P | MODE_PARSE
        stream (same frames) whose records feed the fold."""
        if telemetry is not None:
            return self._open(A.MODE_P | A.MODE_PARSE, telemetry)
        sid = self.L.ssegw_proxy_stream(self.g)
        if sid < 0:
            raise RuntimeError("no free connection slot")
        return sid

    def proxy_step(self, sid: int):
        """One turn of the c.Stream callback: the line to write, None if none has arrived, EOFError when the loop ends."""
        return self._recv(self.L.ssegw_proxy_step, sid)

    def agent_recv(self, sid: int):
        return self._recv(self.L.ssegw_agent_recv, sid)

    def agent_state(self, sid: int):
        b = self.L.ssegw_agent_content(self.g, sid)
        content = C.string_at(b.p, b.n) if b.n else b""
        fin = C.c_int()
        term = bool(self.L.ssegw_agent_terminated(self.g, sid, C.byref(fin)))
        n = self.L.ssegw_agent_tool_calls(self.g, sid, None, 0)
        arr = (A.ToolCall * max(1, n))()
        n = min(n, self.L.ssegw_agent_tool_calls(self.g, sid, arr, n))
        g = _bytes
        calls = [dict(id=g(arr[i].id), type=g(arr[i].type), name=g(arr[i].name), args=g(arr[i].arguments)) for i in range(n)]
        return content, bool(self.L.ssegw_agent_has_tool_calls(self.g, sid)), term, fin.value, calls

    def counters(self) -> dict:
        """ssegw_counters: the sse_counters of every batch collected so far, added up (the gateway's config must have
        FLAG_COUNTERS), as {field: int} plus decode_passes."""
        k = A.Counters()
        k.struct_size = C.sizeof(A.Counters)
        A.check(self.L.ssegw_counters(self.g, C.byref(k)), "ssegw_counters")
        return A.counters_dict(k)

    def trim(self, min_pool_pages: int | None = None):
        """ssegw_trim: sse_trim on every context (the config must have FLAG_DEFER); min_pool_pages defaults to the pages of the
        line pool the gateway was created with."""
        if min_pool_pages is None:
            min_pool_pages = self._pool.pool_pages if self._pool is not None else 0
        A.check(self.L.ssegw_trim(self.g, min_pool_pages), "ssegw_trim")

    def release(self, sid: int):
        self.L.ssegw_release_stream(self.g, sid)
        self._taps.pop(sid, None)

    def mcp_write_loop(self, sid: int):
        """handleMCPStreamingRequest's writer (api/middlewares/mcp.go:253-299) over the agent channel of one stream:
        returns (bytes written to the client so far, status_503, ended). Call after pump() until ended."""
        out = bytearray()
        status_503 = False
        while True:
            try:
                fr = self.agent_recv(sid)
            except EOFError:                     # channel closed without the terminal frame (mcp.go:256-259)
                return bytes(out), status_503, True
            if fr is None:
                return bytes(out), status_503, False
            flag = C.c_int(0)
            stop = self.L.ssegw_mcp_writer_step(fr, len(fr), C.byref(flag))
            status_503 = status_503 or bool(flag.value)
            out += fr
            if stop:
                return bytes(out), status_503, True
