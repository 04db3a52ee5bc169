// gpuProvider / gpuRegistry: the two types a maintainer adds so that the GPU path sits behind the reference's own
// interfaces with api/routes.go and the middleware chain unchanged. NOT COMPILED HERE (no Go toolchain in the image).
//
//   cmd/gateway/main.go:171   providerRegistry := registry.NewProviderRegistry(cfg.Providers, logger)
// becomes
//   providerRegistry := ssegpu.WrapRegistry(registry.NewProviderRegistry(cfg.Providers, logger), batcher)
package ssegpu

import (
	"context"
	"io"
	"net/http"

	"github.com/inference-gateway/inference-gateway/providers/client"
	"github.com/inference-gateway/inference-gateway/providers/core"
	"github.com/inference-gateway/inference-gateway/providers/registry"
	"github.com/inference-gateway/inference-gateway/providers/types"
)

// Batcher owns the per-GPU contexts. Connections shard by hash(conn) % nGPU and stay on their GPU for life
// (carry state and FIFO order are per device). One goroutine per GPU, locked to its OS thread, runs:
//   acquire -> drain pending reads of its connections into the batch (<= GPU_BATCH_USEC or GPU_BATCH_BYTES) ->
//   submit -> collect -> fan frames out to the per-stream channels -> release.
// With GPU_DEFER=1 (see NewContext) a segment can come back Deferred: its unconsumed tail goes back to the head of that
// connection's queue, and connections with such a tail are drained first into the next batch.
type Batcher interface {
	// Open registers a new upstream stream; the returned id addresses its slot until Close.
	Open(mode uint8) (conn uint32, frames <-chan []byte)
	// Feed hands over bytes read from the upstream body (any cut points). EOF/err closes the stream after the
	// lines already queued were delivered; the unterminated tail is dropped (provider.go:323-330).
	Feed(conn uint32, data []byte)
	Close(conn uint32)
}

type gpuRegistry struct {
	inner registry.ProviderRegistry
	b     Batcher
}

func WrapRegistry(inner registry.ProviderRegistry, b Batcher) registry.ProviderRegistry {
	return &gpuRegistry{inner: inner, b: b}
}
func (g *gpuRegistry) GetProviders() map[types.Provider]*registry.ProviderConfig { return g.inner.GetProviders() }
func (g *gpuRegistry) BuildProvider(id types.Provider, c client.Client) (core.IProvider, error) {
	p, err := g.inner.BuildProvider(id, c)
	if err != nil {
		return nil, err
	}
	return &gpuProvider{IProvider: p, b: g.b}, nil
}

// gpuProvider embeds the stock provider (nine methods for free) and replaces only the stream reader.
type gpuProvider struct {
	core.IProvider
	b Batcher
	// OpenUpstream re-implements provider.go:277-305 (unexported helpers there): build URL, force
	// stream_options.include_usage, POST, map non-200 to *core.HTTPError. ~30 lines, unchanged semantics.
	OpenUpstream func(ctx context.Context, req types.CreateChatCompletionRequest) (*http.Response, error)
}

func (p *gpuProvider) StreamChatCompletions(ctx context.Context, req types.CreateChatCompletionRequest) (<-chan []byte, error) {
	resp, err := p.OpenUpstream(ctx, req)
	if err != nil {
		return nil, err // before streaming: (nil, err), *core.HTTPError carries the upstream status
	}
	conn, frames := p.b.Open(ModeP) // the MCP agent asks for ModeR via a context key instead
	go func() {                     // socket reads stay on the host; one goroutine per stream as in provider.go:308
		defer resp.Body.Close()
		defer p.b.Close(conn)
		buf := make([]byte, 32<<10)
		for {
			n, rerr := resp.Body.Read(buf)
			if n > 0 {
				p.b.Feed(conn, buf[:n])
			}
			if rerr != nil || ctx.Err() != nil { // io.EOF or read error: log only, close (provider.go:323-330)
				_ = io.EOF
				return
			}
		}
	}()
	return frames, nil
}
