// StreamingTelemetry: the telemetry middleware for streaming chat completions on the GPU path. NOT COMPILED HERE (no Go
// toolchain in the image).
//
// The stock middleware (api/middlewares/telemetry.go) copies every byte written to the client into a buffer (:37-54) and,
// after the handler returns, splits it on "\n\n" and unmarshals the pieces (:190-277). On the GPU path the device has already
// decoded every line it would parse, so for a streaming request this middleware puts a telemetry fold into the request
// context instead: the provider attaches it to the upstream stream it opens (gpuProvider.StreamChatCompletions), the
// batcher feeds it the records of what it delivers, and the MCP agent feeds it what it writes itself (HostFrame). Nothing is
// buffered. Non-streaming requests, and every other path, go to the stock middleware unchanged.
//
// One difference from the stock middleware (DESIGN.md section 5): the fold counts what reached the stream's channel, the
// stock middleware what the handler wrote. When the client goes away (ctx.Done()), up to the channel's 100 elements
// delivered but never written are counted here and not there.
//
//	cmd/gateway/main.go: r.Use(telemetryMiddleware.Middleware())
//
// becomes
//
//	r.Use(ssegpu.StreamingTelemetry(telemetryMiddleware.Middleware(), otelTelemetry, logger))
package ssegpu

import (
	"bytes"
	"context"
	"encoding/json"
	"io"
	"strings"
	"time"

	"github.com/gin-gonic/gin"
	"github.com/inference-gateway/inference-gateway/logger"
	"github.com/inference-gateway/inference-gateway/otel"
)

// providerPrefixes: the model prefixes, and then the query substrings, by which telemetry.go:71-120 names the provider.
var providerPrefixes = []string{"openai", "anthropic", "groq", "cohere", "ollama", "cloudflare", "deepseek", "google",
	"mistral", "moonshot", "ollama_cloud"}

func providerOf(model, rawQuery string) string {
	for _, p := range providerPrefixes {
		if strings.HasPrefix(model, p+"/") {
			return p
		}
	}
	for _, p := range providerPrefixes[:len(providerPrefixes)-1] { // the query fallback knows no ollama_cloud
		if strings.Contains(rawQuery, p) {
			return p
		}
	}
	return "unknown"
}

// toolType is telemetry.go's classifyToolType (:323-330): "mcp" for names with the "mcp_" prefix.
func toolType(name string) string {
	if strings.HasPrefix(name, "mcp_") {
		return "mcp"
	}
	return "standard_tool_use"
}

// StreamingTelemetry wraps the stock telemetry middleware: streaming chat completions are recorded from a fold, anything
// else goes to stock.
func StreamingTelemetry(stock gin.HandlerFunc, tm otel.OpenTelemetry, log logger.Logger) gin.HandlerFunc {
	return func(c *gin.Context) {
		if !strings.Contains(c.Request.URL.Path, "/v1/chat/completions") {
			stock(c)
			return
		}
		start := time.Now()
		body, _ := io.ReadAll(c.Request.Body)
		c.Request.Body = io.NopCloser(bytes.NewBuffer(body))
		var req struct {
			Model  string `json:"model"`
			Stream *bool  `json:"stream"`
		}
		_ = json.Unmarshal(body, &req)
		if req.Stream == nil || !*req.Stream {
			stock(c) // non-streaming responses keep the stock body parse
			return
		}
		tel := NewTelemetry()
		c.Request = c.Request.WithContext(WithTelemetry(c.Request.Context(), tel))

		c.Next()
		// a client that went away ends the handler before the provider's reader has closed its connection: wait for it, so
		// that no batcher feeds the fold after this
		tel.open.Wait()
		defer tel.Free()

		provider := providerOf(req.Model, c.Request.URL.RawQuery)
		if provider == "unknown" {
			log.Warn("unknown provider detected", "model", req.Model, "path", c.Request.URL.Path, "query", c.Request.URL.RawQuery)
			return
		}
		ctx := c.Request.Context()
		tm.RecordResponseStatus(ctx, provider, c.Request.Method, c.Request.URL.Path, c.Writer.Status())
		tm.RecordRequestDuration(ctx, provider, c.Request.Method, c.Request.URL.Path, float64(time.Since(start).Milliseconds()))
		usage, calls, irregular, err := tel.Finish()
		if err != nil || irregular {
			log.Debug("telemetry fold: figures may differ from a body parse", "irregular", irregular, "error", err)
		}
		tm.RecordTokenUsage(ctx, provider, req.Model, usage[0], usage[1], usage[2])
		for _, tc := range calls {
			tm.RecordToolCallCount(ctx, provider, req.Model, toolType(tc.Name), tc.Name)
		}
	}
}

// HostFrame is what mcp.Agent calls for every frame it writes to the client itself, next to the channel send: its error
// frames (agent.go:151-152, :275) and its single final "data: [DONE]\n\n" (:140-143). The batcher feeds only bytes that
// came from upstream, so without this the fold's last-four-pieces window would be off by the [DONE].
func HostFrame(ctx context.Context, frame []byte) {
	if t := TelemetryFrom(ctx); t != nil {
		_ = t.FeedBytes(frame)
	}
}
