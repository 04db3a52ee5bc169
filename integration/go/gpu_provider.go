// gpuProvider / gpuRegistry: the two types a maintainer adds so that the GPU path sits behind the reference's own
// interfaces with api/routes.go and the middleware chain unchanged. NOT COMPILED HERE (no Go toolchain in the image).
//
//   cmd/gateway/main.go:171   providerRegistry := registry.NewProviderRegistry(cfg.Providers, logger)
// becomes
//   batchers, err := ssegpu.Batchers(newBatcher) // one per entry of GPU_DEVICES
//   providerRegistry := ssegpu.WrapRegistry(registry.NewProviderRegistry(cfg.Providers, logger), batchers)
package ssegpu

import (
	"context"
	"io"
	"net/http"
	"os"
	"strconv"
	"strings"

	"github.com/inference-gateway/inference-gateway/providers/client"
	"github.com/inference-gateway/inference-gateway/providers/core"
	"github.com/inference-gateway/inference-gateway/providers/registry"
	"github.com/inference-gateway/inference-gateway/providers/types"
)

// Batcher is one device's batcher: one goroutine, locked to its OS thread, owning one Context whose connections stay on it
// for life (carry state, line-pool pages and FIFO order are per context). Each tick (RunTick below):
//  1. acquire -> drain pending reads of its connections into the batch (<= GPU_BATCH_USEC or GPU_BATCH_BYTES) -> submit;
//  2. collect every batch Poll reports done, oldest first, fan frames out to the per-stream channels, release;
//  3. while GPU_BATCH_DEPTH batches are still uncollected, collect the oldest one, blocking.
// At GPU_BATCH_DEPTH=1 (the default) a batch is collected in the tick that submitted it. Deeper, the host fills batch k+1
// while the device runs batch k. Bytes leave a connection's queue when they are submitted; with GPU_DEFER=1 (see
// NewContext) a segment can come back Deferred: its unconsumed tail goes back to the head of that connection's queue,
// connections with such a tail are drained first into the next batch, and a connection is not drained again while it is in
// an uncollected batch (its tail must come before its newer bytes). The host mirror is ssegw_new_multi / ssegw_pump.
type Batcher interface {
	// Open registers a new upstream stream; the returned id addresses its slot until Close. tel, when not nil, is the
	// client response's telemetry fold (mode must then carry ModeParse or ModeR): the deliver step feeds it every segment
	// whose frames it delivers to this connection, until Close (ssegw_stream_with_telemetry is the host mirror). One fold
	// feeds one open connection at a time; an MCP session attaches it to each iteration's connection in turn.
	Open(mode uint8, tel *Telemetry) (conn uint32, frames <-chan []byte)
	// Feed hands over bytes read from the upstream body (any cut points). EOF/err closes the stream after the
	// lines already queued, and those in uncollected batches, were delivered; the unterminated tail is dropped
	// (provider.go:323-330).
	Feed(conn uint32, data []byte)
	// Close releases the connection; once it returns, nothing collected later is delivered or fed to its fold.
	Close(conn uint32)
	// Open streams, for placement.
	Streams() int
	// Trim runs Context.Trim between two ticks of the batcher's goroutine. When to call it (e.g. a timer after bursts of
	// long lines) is the operator's policy; the batcher never trims on its own.
	Trim(minPages uint32) error
	// MemoryHeld is Context.MemoryHeld, e.g. for export as gauges.
	MemoryHeld() (device, pinned uint64, err error)
}

// inFlight is one submitted batch and the connections (with their generation: a connection closed and opened again
// while the batch was in flight gets nothing of it) whose bytes it holds.
type inFlight struct {
	b   *Batch
	who []member
}

type member struct {
	conn uint32
	gen  uint64
	data []byte     // the bytes submitted (a view of the batch's pinned arena), for the deferred tail
	tel  *Telemetry // the connection's telemetry fold at submit time, nil without a tap
}

// feedTap is the telemetry half of the deliver step for segment i of a collected batch, held by m. The deliver step calls
// it next to the agent fold's feed, after the segment's frames went to the connection's channel, and only when m.gen is
// still the connection's generation and the connection is neither closed nor failed, so that nothing is fed after Close.
// It reports whether the stream must be closed: the fold met a line past the nesting limit (SSE_ERR_UNDECODED).
func feedTap(m member, res *Result, i uint32) (closeStream bool) {
	return m.tel != nil && m.tel.Feed(res, i) != nil
}

// RunTick is steps 2 and 3 of a tick, after step 1 appended the submitted batch (if any) to q. deliver fans one collected
// batch out (frames, Deferred tails, agent folds, telemetry taps through feedTap, counters) in submission order; a failed
// batch closes its streams.
func RunTick(x *Context, q []inFlight, depth int, deliver func(inFlight, *Result, error)) ([]inFlight, error) {
	collect := func() {
		f := q[0]
		q = q[1:]
		res, err := x.Collect(f.b)
		deliver(f, res, err)
		x.Release(f.b)
	}
	for len(q) > 0 {
		done, err := x.Poll(q[0].b)
		if err != nil {
			return q, err
		}
		if !done {
			break
		}
		collect()
	}
	for len(q) >= depth {
		collect()
	}
	return q, nil
}

// Batchers builds one Batcher per entry of GPU_DEVICES (comma-separated device ordinals, default "0"; an ordinal may repeat,
// which gives independent contexts on one GPU), each with GPU_BATCH_DEPTH (1..8, default 1) batches in flight.
func Batchers(newBatcher func(device int, depth int) (Batcher, error)) ([]Batcher, error) {
	depth := int(envUint32("GPU_BATCH_DEPTH"))
	if depth == 0 {
		depth = 1
	}
	devs := os.Getenv("GPU_DEVICES")
	if devs == "" {
		devs = "0"
	}
	var out []Batcher
	for _, d := range strings.Split(devs, ",") {
		dev, err := strconv.Atoi(strings.TrimSpace(d))
		if err != nil {
			return nil, err
		}
		b, err := newBatcher(dev, depth)
		if err != nil {
			return nil, err
		}
		out = append(out, b)
	}
	return out, nil
}

type gpuRegistry struct {
	inner registry.ProviderRegistry
	bs    []Batcher
}

func WrapRegistry(inner registry.ProviderRegistry, bs []Batcher) registry.ProviderRegistry {
	return &gpuRegistry{inner: inner, bs: bs}
}
func (g *gpuRegistry) GetProviders() map[types.Provider]*registry.ProviderConfig { return g.inner.GetProviders() }
func (g *gpuRegistry) BuildProvider(id types.Provider, c client.Client) (core.IProvider, error) {
	p, err := g.inner.BuildProvider(id, c)
	if err != nil {
		return nil, err
	}
	return &gpuProvider{IProvider: p, bs: g.bs}, nil
}

// pick is the batcher with the fewest open streams (the first on a tie): a stream stays on it for its whole life.
func pick(bs []Batcher) Batcher {
	best := bs[0]
	for _, b := range bs[1:] {
		if b.Streams() < best.Streams() {
			best = b
		}
	}
	return best
}

type modeKey struct{}
type telemetryKey struct{}

// WithMode is how the MCP agent asks for ModeR on its provider stream.
func WithMode(ctx context.Context, mode uint8) context.Context { return context.WithValue(ctx, modeKey{}, mode) }

// WithTelemetry puts the client response's telemetry fold into the request context (StreamingTelemetry does, for
// streaming chat completions): the provider attaches it to the stream it opens.
func WithTelemetry(ctx context.Context, t *Telemetry) context.Context {
	return context.WithValue(ctx, telemetryKey{}, t)
}

// TelemetryFrom is the response's fold, or nil when telemetry is off or the request is not a streaming chat completion.
func TelemetryFrom(ctx context.Context) *Telemetry {
	t, _ := ctx.Value(telemetryKey{}).(*Telemetry)
	return t
}

// gpuProvider embeds the stock provider (nine methods for free) and replaces only the stream reader.
type gpuProvider struct {
	core.IProvider
	bs []Batcher
	// OpenUpstream re-implements provider.go:277-305 (unexported helpers there): build URL, force
	// stream_options.include_usage, POST, map non-200 to *core.HTTPError. ~30 lines, unchanged semantics.
	OpenUpstream func(ctx context.Context, req types.CreateChatCompletionRequest) (*http.Response, error)
}

func (p *gpuProvider) StreamChatCompletions(ctx context.Context, req types.CreateChatCompletionRequest) (<-chan []byte, error) {
	resp, err := p.OpenUpstream(ctx, req)
	if err != nil {
		return nil, err // before streaming: (nil, err), *core.HTTPError carries the upstream status
	}
	b := pick(p.bs)
	mode, _ := ctx.Value(modeKey{}).(uint8) // ModeP, or ModeR when the MCP agent asked for it (WithMode)
	tel := TelemetryFrom(ctx)
	if tel != nil && mode&ModeR == 0 {
		mode |= ModeParse // the tap needs the records: same frames as ModeP
	}
	if tel != nil {
		tel.open.Add(1)
	}
	conn, frames := b.Open(mode, tel)
	go func() {                     // socket reads stay on the host; one goroutine per stream as in provider.go:308
		defer resp.Body.Close()
		if tel != nil {
			defer tel.open.Done() // after b.Close: the middleware may then finish and free the fold
		}
		defer b.Close(conn)
		buf := make([]byte, 32<<10)
		for {
			n, rerr := resp.Body.Read(buf)
			if n > 0 {
				b.Feed(conn, buf[:n])
			}
			if rerr != nil || ctx.Err() != nil { // io.EOF or read error: log only, close (provider.go:323-330)
				_ = io.EOF
				return
			}
		}
	}()
	return frames, nil
}
