"""Thin Python driver over the C ABI (one context = one GPU).

Plumbing only: it fills the pinned staging buffers the library lends out, submits, collects and turns the
result arrays into numpy views. All work happens in libssegpu.so; nothing here parses or splits bytes.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _abi as A


def _np_view(ptr, count, dtype):
    if count == 0:
        return np.zeros(0, dtype=dtype)
    nbytes = count * np.dtype(dtype).itemsize
    buf = (C.c_uint8 * nbytes).from_address(C.addressof(ptr.contents))
    return np.frombuffer(buf, dtype=dtype, count=count)


FRAME_DT = np.dtype([("off", "<u4"), ("len", "<u4")])
REC_DT = np.dtype([("frame", "<u4"), ("flags", "<u4"), ("content_off", "<u4"), ("content_len", "<u4"),
                   ("tc_first", "<u4"), ("tc_count", "<u2"), ("n_choices", "<u2"), ("usage", "<u4"),
                   ("payload_len", "<u4")])
TC_DT = np.dtype([("index", "<i8"), ("flags", "<u4"), ("next", "<u4"), ("id_off", "<u4"), ("id_len", "<u4"),
                  ("type_off", "<u4"), ("type_len", "<u4"), ("name_off", "<u4"), ("name_len", "<u4"),
                  ("args_off", "<u4"), ("args_len", "<u4")])
USAGE_DT = np.dtype([("prompt", "<i8"), ("completion", "<i8"), ("total", "<i8")])
RUN_DT = np.dtype([("frame_first", "<u4"), ("frame_count", "<u4"), ("rec_first", "<u4"), ("rec_count", "<u4"),
                   ("next", "<u4")])
SEGRES_DT = np.dtype([("frame_first", "<u4"), ("frame_count", "<u4"), ("rec_first", "<u4"), ("rec_count", "<u4"),
                      ("next", "<u4"), ("carry_len", "<u4"), ("flags", "<u4"), ("consumed", "<u4")])
SEG_DT = np.dtype([("conn", "<u4"), ("in_off", "<u4"), ("in_len", "<u4"), ("mode", "u1"), ("provider", "u1"),
                   ("reserved", "<u2")])
assert FRAME_DT.itemsize == 8 and REC_DT.itemsize == 32 and TC_DT.itemsize == 48 and SEGRES_DT.itemsize == 32
assert SEG_DT.itemsize == 16 and RUN_DT.itemsize == 20


@dataclass
class BatchResult:
    """Views into the library's pinned result buffers (valid until the slot is released)."""
    raw: A.Result
    out: np.ndarray
    frames: np.ndarray
    recs: np.ndarray
    tcs: np.ndarray
    usages: np.ndarray
    text: np.ndarray
    runs: np.ndarray
    segs: np.ndarray
    in_arena: np.ndarray = None     # the batch's input arena; arena offsets >= in_base index it (zero-copy frames)
    in_base: int = 0xFFFFFFFF

    def at(self, off: int, length: int) -> bytes:
        """sse_at(): resolve an arena offset."""
        if off >= self.in_base:
            o = off - self.in_base
            return self.in_arena[o:o + length].tobytes()
        return self.out[off:off + length].tobytes()

    def seg_runs(self, i: int):
        s = self.segs[i]
        run = (int(s["frame_first"]), int(s["frame_count"]), int(s["rec_first"]), int(s["rec_count"]))
        nxt = int(s["next"])
        yield run
        while nxt != A.NONE:
            r = self.runs[nxt]
            yield (int(r["frame_first"]), int(r["frame_count"]), int(r["rec_first"]), int(r["rec_count"]))
            nxt = int(r["next"])

    def seg_frames(self, i: int) -> list:
        out = []
        for ff, fc, _, _ in self.seg_runs(i):
            for k in range(ff, ff + fc):
                f = self.frames[k]
                out.append(self.at(int(f["off"]), int(f["len"])))
        return out

    def seg_recs(self, i: int) -> list:
        out = []
        for _, _, rf, rc in self.seg_runs(i):
            out.extend(range(rf, rf + rc))
        return out

    def span(self, off: int, length: int, in_text: bool) -> bytes:
        return self.text[off:off + length].tobytes() if in_text else self.at(off, length)

    def consumed(self, i: int) -> int:
        """Input bytes of segment i the batch took: its whole length unless it was deferred (SSE_FLAG_DEFER, SEG_DEFERRED)."""
        return int(self.segs[i]["consumed"])

    @property
    def overflow(self) -> int:
        """SSE_OVF_* bits of what this batch deferred or grew (SSE_FLAG_DEFER); 0 when everything fit."""
        return int(self.raw.overflow)


def make_line_pool(pool_pages: int, page_bytes: int = 0, max_line_bytes: int = A.MAX_LINE_BYTES) -> A.LinePool:
    """sse_line_pool: pool_pages pages of page_bytes (0: 64 KiB) shared by all connections for lines longer than the carry slot;
    one connection's line may grow to max_line_bytes."""
    return A.LinePool(C.sizeof(A.LinePool), page_bytes, pool_pages, max_line_bytes)


class SseEngine:
    def __init__(self, device: int = 0, max_conns: int = 1024, bytes_per_batch: int = 1 << 20, line_pool: dict | None = None,
                 **overrides):
        """line_pool: keyword arguments of make_line_pool() (pool_pages, page_bytes, max_line_bytes), and optionally max_pages
        (sse_line_pool_set_growth: with flags=FLAG_DEFER the pool grows on demand up to that many pages instead of failing
        a line that finds no free page), or None for no pool: a line longer than carry_slot_bytes then fails its connection."""
        self.L = A.load()
        cfg = A.Config()
        self.L.sse_default_config(C.byref(cfg), max_conns, bytes_per_batch)
        for k, v in overrides.items():
            setattr(cfg, k, v)
        self._ctx = C.c_void_p()
        line_pool = dict(line_pool) if line_pool is not None else None
        max_pages = line_pool.pop("max_pages", 0) if line_pool is not None else 0
        self.pool = make_line_pool(**line_pool) if line_pool is not None else None
        pp = C.byref(self.pool) if self.pool is not None else None
        A.check(self.L.sse_init_ex(device, C.byref(cfg), pp, C.byref(self._ctx)), "sse_init_ex")
        if pp is not None:
            self.L.sse_line_pool_config(C.byref(cfg), pp)   # the capacities the context allocated
        self.cfg = cfg
        self.device = device
        if max_pages:
            self.line_pool_growth(max_pages)

    def line_pool_growth(self, max_pages: int):
        """sse_line_pool_set_growth: the pool may grow up to max_pages pages (0: never), ordered after the batches submitted."""
        A.check(self.L.sse_line_pool_set_growth(self._ctx, max_pages), "sse_line_pool_set_growth")

    def line_pool_capacity(self):
        """(pages, growth limit) of the line pool: its pages after the growths of the batches collected so far; limit 0: none."""
        pages, limit = C.c_uint32(), C.c_uint32()
        A.check(self.L.sse_line_pool_capacity(self._ctx, C.byref(pages), C.byref(limit)), "sse_line_pool_capacity")
        return pages.value, limit.value

    def pool_stats(self):
        """(pages in use, high-water mark) of the line pool, after every batch submitted so far."""
        used, hw = C.c_uint32(), C.c_uint32()
        A.check(self.L.sse_line_pool_stats(self._ctx, C.byref(used), C.byref(hw)), "sse_line_pool_stats")
        return used.value, hw.value

    def trim(self, min_pool_pages: int | None = None):
        """sse_trim: gives back what on-demand growth took (FLAG_DEFER). A pool with a growth limit shrinks to
        max(min_pool_pages, pages held, 1) pages (default: the pages the engine was created with) when that is below its capacity;
        every slot's decode arenas go back to the config's capacities, a slot that holds a batch at its release."""
        if min_pool_pages is None:
            min_pool_pages = self.pool.pool_pages if self.pool is not None else 0
        A.check(self.L.sse_trim(self._ctx, min_pool_pages), "sse_trim")

    def memory_held(self):
        """sse_memory_held: (device bytes, pinned host bytes) the context holds now."""
        dev, pin = C.c_uint64(), C.c_uint64()
        A.check(self.L.sse_memory_held(self._ctx, C.byref(dev), C.byref(pin)), "sse_memory_held")
        return dev.value, pin.value

    def close(self):
        if self._ctx:
            self.L.sse_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- slot level ------------------------------------------------------------------------------
    def acquire(self):
        slot = C.c_int()
        b = A.Batch()
        A.check(self.L.sse_acquire(self._ctx, C.byref(slot), C.byref(b)), "sse_acquire")
        arena = _np_view(b.in_arena, b.in_arena_bytes, np.uint8)
        segs = _np_view(C.cast(b.segs, C.POINTER(C.c_uint8)), b.max_segs * 16, np.uint8).view(SEG_DT)
        return slot.value, arena, segs

    def fill(self, arena, segs, items):
        """items: iterable of (conn, mode, bytes). Returns (n_segs, in_bytes)."""
        off = 0
        n = 0
        for conn, mode, data in items:
            ln = len(data)
            if ln:
                arena[off:off + ln] = np.frombuffer(data, dtype=np.uint8)
            segs[n] = (conn, off, ln, mode, 0, 0)
            off = (off + ln + 15) & ~15
            n += 1
        return n, off

    def submit(self, slot, n_segs, in_bytes):
        A.check(self.L.sse_submit(self._ctx, slot, n_segs, in_bytes), "sse_submit")

    def _wrap(self, res: A.Result) -> BatchResult:
        return BatchResult(
            res,
            _np_view(res.out, res.out_bytes, np.uint8),
            _np_view(C.cast(res.frames, C.POINTER(C.c_uint8)), res.n_frames * 8, np.uint8).view(FRAME_DT),
            _np_view(C.cast(res.recs, C.POINTER(C.c_uint8)), res.n_recs * 32, np.uint8).view(REC_DT),
            _np_view(C.cast(res.tcs, C.POINTER(C.c_uint8)), res.n_tcs * 48, np.uint8).view(TC_DT),
            _np_view(C.cast(res.usages, C.POINTER(C.c_uint8)), res.n_usages * 24, np.uint8).view(USAGE_DT),
            _np_view(res.text, res.text_bytes, np.uint8),
            _np_view(C.cast(res.runs, C.POINTER(C.c_uint8)), res.n_runs * 20, np.uint8).view(RUN_DT),
            _np_view(C.cast(res.segs, C.POINTER(C.c_uint8)), res.n_segs * 32, np.uint8).view(SEGRES_DT),
            _np_view(res.in_, self.cfg.in_arena_bytes, np.uint8), int(res.in_base),
        )

    def collect(self, slot) -> BatchResult:
        res = A.Result()
        rc = self.L.sse_collect(self._ctx, slot, C.byref(res))
        if rc == A.SSE_ERR_OVERFLOW:
            raise A.SseError(rc, f"sse_collect (overflow mask 0x{res.overflow:x}: 1 out/frames/recs, 2 tcs, 4 usages, 8 text, 16 runs)")
        A.check(rc, "sse_collect")
        return self._wrap(res)

    def release(self, slot):
        A.check(self.L.sse_release(self._ctx, slot), "sse_release")

    def reset_conn(self, conn: int):
        A.check(self.L.sse_reset_conn(self._ctx, conn), "sse_reset_conn")

    def reset_all(self, stream: int = 0):
        A.check(self.L.sse_reset_all(self._ctx, C.c_void_p(stream)), "sse_reset_all")

    # -- device-resident stages (bench) ------------------------------------------------------------
    def upload(self, slot, n_segs, in_bytes, stream: int = 0):
        A.check(self.L.sse_upload(self._ctx, slot, n_segs, in_bytes, C.c_void_p(stream)), "sse_upload")

    def launch(self, slot, n_segs, stream: int = 0):
        A.check(self.L.sse_launch(self._ctx, slot, n_segs, C.c_void_p(stream)), "sse_launch")

    def download(self, slot, stream: int = 0) -> BatchResult:
        res = A.Result()
        rc = self.L.sse_download(self._ctx, slot, C.byref(res), C.c_void_p(stream))
        if rc == A.SSE_ERR_OVERFLOW:
            raise A.SseError(rc, f"sse_download (overflow mask 0x{res.overflow:x}: 1 out/frames/recs, 2 tcs, 4 usages, 8 text, 16 runs)")
        A.check(rc, "sse_download")
        return self._wrap(res)

    def counters(self, slot) -> dict:
        """sse_counters_read (engine made with flags=FLAG_COUNTERS): what the kernels did for the batch collected or downloaded in
        slot, as {field: int} with the field names of sse_counters, plus decode_passes. Valid until the slot is released."""
        k = A.Counters()
        k.struct_size = C.sizeof(A.Counters)
        A.check(self.L.sse_counters_read(self._ctx, slot, C.byref(k)), "sse_counters_read")
        return A.counters_dict(k)

    def launch_count(self) -> int:
        n = C.c_uint64()
        A.check(self.L.sse_launch_count(self._ctx, C.byref(n)), "sse_launch_count")
        return n.value

    # -- convenience: one synchronous batch ---------------------------------------------------------
    def process(self, items):
        """items: list of (conn, mode, bytes). Returns a BatchResult; caller must release(result_slot)."""
        slot, arena, segs = self.acquire()
        n, nbytes = self.fill(arena, segs, items)
        self.submit(slot, n, nbytes)
        r = self.collect(slot)
        return slot, r

    def process_all(self, items, on_batch=None) -> int:
        """items: list of (conn, mode, bytes), at most one per connection, run to the end on an engine with SSE_FLAG_DEFER: the
        part of a segment a batch deferred is submitted again, from its first byte not taken, in the next batch, until every
        byte was taken. on_batch(result, conns) sees every batch before its slot is released (conns[i]: the connection of
        segment i). A batch in which no segment got anywhere (segments competing for arenas that fit each of them alone) is
        followed by one that carries only the first remaining segment, which always fits an empty batch. Returns the number
        of batches."""
        pending = [(c, m, bytes(d)) for c, m, d in items]
        n_batches = 0
        alone = False
        while pending:
            batch = pending[:1] if alone else pending
            slot, res = self.process(batch)
            try:
                if on_batch is not None:
                    on_batch(res, [c for c, _, _ in batch])
                left, progress = [], False
                for i, (conn, mode, data) in enumerate(batch):
                    took = res.consumed(i)
                    if int(res.segs[i]["flags"]) & A.SEG_DEFERRED:
                        left.append((conn, mode, data[took:]))
                    progress = progress or took > 0 or not int(res.segs[i]["flags"]) & A.SEG_DEFERRED
            finally:
                self.release(slot)
            if alone and not progress:
                raise RuntimeError("a segment alone in a batch was deferred without progress: capacities below one round")
            pending = left + pending[len(batch):]
            alone = not progress
            n_batches += 1
        return n_batches
