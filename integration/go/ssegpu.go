// Package ssegpu binds libssegpu.so (include/sse_gpu.h) through cgo.
//
// NOT COMPILED IN THIS REPOSITORY'S CI: the build image has no Go toolchain (SURVEY.md section 8c). This file is the
// binding a maintainer adds to the gateway; it is written against the C ABI only and keeps no Go pointer on the C
// side (all buffers are cudaHostAlloc'd by the library and viewed with unsafe.Slice).
package ssegpu

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../inference_gateway_b200 -lssegpu -Wl,-rpath,${SRCDIR}/../../inference_gateway_b200
#include "sse_gpu.h"
*/
import "C"

import (
	"errors"
	"fmt"
	"os"
	"runtime"
	"strconv"
	"sync"
	"unsafe"
)

const (
	ModeP     = uint8(C.SSE_MODE_P)
	ModeR     = uint8(C.SSE_MODE_R)
	ModeParse = uint8(C.SSE_MODE_PARSE)
)

// Context is one GPU. It must be driven from ONE goroutine locked to its OS thread (the per-GPU batcher).
type Context struct{ c *C.sse_ctx }

func statusErr(where string, rc C.int) error {
	if rc == C.SSE_OK {
		return nil
	}
	msg := C.GoString(C.sse_strerror(rc))
	if rc == C.SSE_ERR_CUDA {
		msg += ": " + C.GoString(C.sse_last_cuda_error())
	}
	return fmt.Errorf("%s: %s (%d)", where, msg, int(rc))
}

func envUint32(name string) uint32 {
	v, err := strconv.ParseUint(os.Getenv(name), 10, 32)
	if err != nil {
		return 0
	}
	return uint32(v)
}

// NewContext fails when no CUDA device is present: there is no CPU fallback.
//
// GPU_LINE_POOL_PAGES > 0 gives the context a line pool of that many pages (GPU_LINE_POOL_PAGE_BYTES each, default 64 KiB),
// shared by all connections: a line longer than the carry slot continues there instead of failing its stream, up to
// GPU_LINE_POOL_MAX_LINE bytes per connection (default and ceiling SSE_MAX_LINE_BYTES, 16 MiB - 1).
// GPU_LINE_POOL_MAX_PAGES > GPU_LINE_POOL_PAGES lets the pool grow on demand up to that many pages
// (sse_line_pool_set_growth): a line that finds no free page waits as a deferred rest while the pool grows, instead of
// failing its stream. It requires GPU_DEFER=1.
//
// GPU_COUNTERS=1 sets SSE_FLAG_COUNTERS: the counting kernels run and Counters(slot) reports what they did for each batch
// (INTEGRATION.md section 2 maps the fields to metric names).
//
// GPU_DEFER=1 sets SSE_FLAG_DEFER: a batch whose results do not fit the default capacities no longer fails (which would close
// every stream in it); what does not fit waits for the next batch. The batcher must then keep the unconsumed tail of a
// deferred segment (data[res.Consumed(i):], see Result.Deferred) at the head of that connection's queue and submit it before
// any newer bytes of the connection.
//
// nSlots (1..8) is how many batches the context can hold at once: the batcher keeps up to that many in flight
// (GPU_BATCH_DEPTH).
func NewContext(device int, maxConns, bytesPerBatch, nSlots uint32) (*Context, error) {
	runtime.LockOSThread()
	var cfg C.sse_config
	C.sse_default_config(&cfg, C.uint32_t(maxConns), C.uint32_t(bytesPerBatch))
	cfg.n_slots = C.uint32_t(nSlots)
	if os.Getenv("GPU_DEFER") == "1" {
		cfg.flags |= C.SSE_FLAG_DEFER
	}
	if os.Getenv("GPU_COUNTERS") == "1" {
		cfg.flags |= C.SSE_FLAG_COUNTERS
	}
	var ctx *C.sse_ctx
	if pages := envUint32("GPU_LINE_POOL_PAGES"); pages > 0 {
		maxLine := envUint32("GPU_LINE_POOL_MAX_LINE")
		if maxLine == 0 {
			maxLine = uint32(C.SSE_MAX_LINE_BYTES)
		}
		pool := C.sse_line_pool{struct_size: C.uint32_t(unsafe.Sizeof(C.sse_line_pool{})),
			page_bytes: C.uint32_t(envUint32("GPU_LINE_POOL_PAGE_BYTES")), pool_pages: C.uint32_t(pages), max_line_bytes: C.uint32_t(maxLine)}
		if err := statusErr("sse_init_ex", C.sse_init_ex(C.int(device), &cfg, &pool, &ctx)); err != nil {
			return nil, err
		}
		if maxPages := envUint32("GPU_LINE_POOL_MAX_PAGES"); maxPages > 0 {
			if cfg.flags&C.SSE_FLAG_DEFER == 0 {
				C.sse_destroy(ctx)
				return nil, errors.New("GPU_LINE_POOL_MAX_PAGES requires GPU_DEFER=1")
			}
			if err := statusErr("sse_line_pool_set_growth", C.sse_line_pool_set_growth(ctx, C.uint32_t(maxPages))); err != nil {
				C.sse_destroy(ctx)
				return nil, err
			}
		}
		return &Context{c: ctx}, nil
	}
	if err := statusErr("sse_init", C.sse_init(C.int(device), &cfg, &ctx)); err != nil {
		return nil, err
	}
	return &Context{c: ctx}, nil
}

// Counters returns what the kernels did for the batch collected in slot (SSE_FLAG_COUNTERS, GPU_COUNTERS=1): valid after
// Collect and before Release. The batcher adds them up and exports them as monotonic counters.
func (x *Context) Counters(slot C.int) (C.sse_counters, error) {
	var k C.sse_counters
	k.struct_size = C.uint32_t(unsafe.Sizeof(k))
	err := statusErr("sse_counters_read", C.sse_counters_read(x.c, slot, &k))
	return k, err
}

// LinePoolStats returns the pages of the line pool held now and the most ever held at once.
func (x *Context) LinePoolStats() (inUse, highWater uint32, err error) {
	var u, h C.uint32_t
	err = statusErr("sse_line_pool_stats", C.sse_line_pool_stats(x.c, &u, &h))
	return uint32(u), uint32(h), err
}

// LinePoolCapacity returns the line pool's pages now (after the growths of the batches collected so far) and its growth
// limit (0: no growth).
func (x *Context) LinePoolCapacity() (pages, maxPages uint32, err error) {
	var p, m C.uint32_t
	err = statusErr("sse_line_pool_capacity", C.sse_line_pool_capacity(x.c, &p, &m))
	return uint32(p), uint32(m), err
}

// Trim gives back what on-demand growth (GPU_DEFER=1) took: a line pool with a growth limit shrinks to max(minPages, pages
// held, 1) pages, and every slot's decode arenas go back to the config's capacities (a slot that holds a batch at its
// Release). Connections holding lines go on unchanged. It waits for the batches already submitted to finish on the device.
func (x *Context) Trim(minPages uint32) error {
	return statusErr("sse_trim", C.sse_trim(x.c, C.uint32_t(minPages)))
}

// MemoryHeld returns the device and pinned host bytes the context holds now, grown pool and arenas included.
func (x *Context) MemoryHeld() (device, pinned uint64, err error) {
	var d, p C.uint64_t
	err = statusErr("sse_memory_held", C.sse_memory_held(x.c, &d, &p))
	return uint64(d), uint64(p), err
}

func (x *Context) Close() { C.sse_destroy(x.c) }

// Batch is one acquired slot: Arena and Segs alias pinned memory owned by the library.
type Batch struct {
	Slot  C.int
	Arena []byte
	Segs  []C.sse_seg
	nSegs uint32
	off   uint32
}

func (x *Context) Acquire() (*Batch, error) {
	var slot C.int
	var b C.sse_batch
	if err := statusErr("sse_acquire", C.sse_acquire(x.c, &slot, &b)); err != nil {
		return nil, err
	}
	return &Batch{Slot: slot,
		Arena: unsafe.Slice((*byte)(unsafe.Pointer(b.in_arena)), int(b.in_arena_bytes)),
		Segs:  unsafe.Slice(b.segs, int(b.max_segs))}, nil
}

// Add copies the bytes read from one connection since the previous batch (at most one segment per connection).
func (b *Batch) Add(conn uint32, mode uint8, data []byte) error {
	if int(b.nSegs) >= len(b.Segs) || int(b.off)+len(data)+16 > len(b.Arena) {
		return errors.New("ssegpu: batch full")
	}
	copy(b.Arena[b.off:], data)
	b.Segs[b.nSegs] = C.sse_seg{conn: C.uint32_t(conn), in_off: C.uint32_t(b.off), in_len: C.uint32_t(len(data)), mode: C.uint8_t(mode)}
	b.nSegs++
	b.off = (b.off + uint32(len(data)) + 15) &^ 15
	return nil
}

func (x *Context) Submit(b *Batch) error {
	return statusErr("sse_submit", C.sse_submit(x.c, b.Slot, C.uint32_t(b.nSegs), C.uint32_t(b.off)))
}

// Poll reports, without blocking, whether the work Submit queued for the batch (kernels and the counters' copy to the host)
// has completed, so that Collect waits only for the batch's own result copies. With GPU_DEFER=1 a Collect after a ready Poll
// may still run the decode stage again, when the slot's decode arenas grow.
func (x *Context) Poll(b *Batch) (bool, error) {
	rc := C.sse_poll(x.c, b.Slot)
	if rc < 0 {
		return false, statusErr("sse_poll", rc)
	}
	return rc == 1, nil
}

// Result views the pinned result buffers; valid until Release.
type Result struct{ r C.sse_result }

func (x *Context) Collect(b *Batch) (*Result, error) {
	res := &Result{}
	if err := statusErr("sse_collect", C.sse_collect(x.c, b.Slot, &res.r)); err != nil {
		return nil, err
	}
	return res, nil
}

func (x *Context) Release(b *Batch) error { return statusErr("sse_release", C.sse_release(x.c, b.Slot)) }
func (x *Context) ResetConn(conn uint32) error {
	return statusErr("sse_reset_conn", C.sse_reset_conn(x.c, C.uint32_t(conn)))
}

// Frames calls fn with a FRESH copy of every frame of segment i, in order: the receiver of the reference's
// chan []byte owns each element (provider.go:322), so the pinned arena must not be handed out.
func (r *Result) Frames(i uint32, fn func(line []byte)) (terminated bool) {
	segs := unsafe.Slice(r.r.segs, int(r.r.n_segs))
	frames := unsafe.Slice(r.r.frames, int(r.r.n_frames))
	runs := unsafe.Slice(r.r.runs, int(r.r.n_runs))
	run := segs[i].run
	for {
		for k := run.frame_first; k < run.frame_first+run.frame_count; k++ {
			f := frames[k]
			// arena offset: >= in_base is a span of the batch's own input arena (zero-copy frame), else the out arena
			src := unsafe.Slice((*byte)(unsafe.Pointer(C.sse_at(&r.r, f.off))), int(f.len))
			line := make([]byte, int(f.len))
			copy(line, src)
			fn(line)
		}
		if run.next == C.SSE_NONE {
			break
		}
		run = runs[run.next]
	}
	return segs[i].flags&C.SSE_SEG_TERMINATED != 0
}

// Telemetry is one client response's telemetry fold (sse_telemetry_*): api/middlewares/telemetry.go:190-277 evaluated from
// the records of the upstream streams that make up the response (one at a time: a plain stream, or each iteration of an MCP
// agent) and from the frames the handler writes itself. The batcher of the connection it is attached to feeds it while the
// connection is open; the handler feeds it after that and finishes it once the response is written. Never concurrently.
type Telemetry struct {
	f    *C.sse_telemetry_fold
	open sync.WaitGroup // connections attached and not yet closed: Finish and Free wait for none
}

func NewTelemetry() *Telemetry { return &Telemetry{f: C.sse_telemetry_new()} }

// Feed folds segment i of a collected batch: the deliver step calls it for a tapped connection, after the segment's frames
// went to the connection's channel. An error (SSE_ERR_UNDECODED: a line past the nesting limit) means the fold is short:
// the batcher closes the stream, as for the agent fold.
func (t *Telemetry) Feed(r *Result, i uint32) error {
	return statusErr("sse_telemetry_feed", C.sse_telemetry_feed(t.f, &r.r, C.uint32_t(i)))
}

// FeedBytes folds frames the handler writes to the client itself: the MCP agent's error frames and its single final
// "data: [DONE]\n\n". b must end on a '\n'.
func (t *Telemetry) FeedBytes(b []byte) error {
	if len(b) == 0 {
		return nil
	}
	return statusErr("sse_telemetry_feed_bytes", C.sse_telemetry_feed_bytes(t.f, (*C.uint8_t)(unsafe.Pointer(&b[0])), C.size_t(len(b))))
}

// ToolCall is one merged tool call of the response (telemetry.go:268-274).
type ToolCall struct{ ID, Type, Name, Arguments string }

func goBytes(b C.sse_bytes) string { return C.GoStringN((*C.char)(unsafe.Pointer(b.p)), C.int(b.n)) }

// Finish returns the response's usage (prompt, completion, total) and tool calls. irregular is true when a "\n\n" piece held
// several lines starting with "data: " (DESIGN.md section 5, deviation 4): the figures are then not the reference's.
// Feed nothing after it.
func (t *Telemetry) Finish() (usage [3]int64, calls []ToolCall, irregular bool, err error) {
	var u C.sse_usage
	var n C.size_t
	rc := C.sse_telemetry_finish(t.f, &u, nil, 0, &n)
	if n > 0 {
		arr := make([]C.sse_tool_call, int(n))
		rc = C.sse_telemetry_finish(t.f, &u, &arr[0], n, &n)
		for _, a := range arr[:int(n)] {
			calls = append(calls, ToolCall{ID: goBytes(a.id), Type: goBytes(a._type), Name: goBytes(a.name), Arguments: goBytes(a.arguments)})
		}
	}
	if rc < 0 {
		return usage, nil, false, statusErr("sse_telemetry_finish", rc)
	}
	return [3]int64{int64(u.prompt_tokens), int64(u.completion_tokens), int64(u.total_tokens)}, calls, rc == 1, nil
}

func (t *Telemetry) Free() { C.sse_telemetry_free(t.f) }

// Deferred reports whether the batch took only the first Consumed(i) bytes of segment i (SSE_FLAG_DEFER): the rest has to be
// submitted again, first in the connection's queue.
func (r *Result) Deferred(i uint32) bool {
	return unsafe.Slice(r.r.segs, int(r.r.n_segs))[i].flags&C.SSE_SEG_DEFERRED != 0
}

// Consumed is the number of segment i's bytes the batch took (its whole length unless Deferred).
func (r *Result) Consumed(i uint32) uint32 {
	return uint32(unsafe.Slice(r.r.segs, int(r.r.n_segs))[i].consumed)
}
