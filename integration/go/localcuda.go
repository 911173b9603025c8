//go:build localcuda

// Package llms — `local-cuda` provider: the in-process H100 engine behind the existing Chat seam.
//
// Drop this file into the reference at pkg/llms/localcuda.go and build with
//     CGO_ENABLED=1 go build -tags localcuda ./cmd/kube-copilot        (the reference Dockerfile:17 uses CGO_ENABLED=0)
// with CGO_CFLAGS=-I<repo>/include and CGO_LDFLAGS="-L<repo>/opsagent_b200/lib -lopsagent_b200".
// It has NOT been compiled here (no Go toolchain in the build image); opsagent_b200/host/localcuda_client.hpp is the
// compiled C++ twin with identical semantics, exercised by tests/test_host_cpp.py.
package llms

/*
#include <stdlib.h>
#include "opsagent_b200.h"
*/
import "C"

import (
	"context"
	"fmt"
	"math"
	"os"
	"runtime"
	"strings"
	"sync"
	"time"
	"unsafe"

	"github.com/sashabaranov/go-openai"
)

// LocalCUDAClient has the fields and the Chat method of OpenAIClient (openai.go:29-35,69).
type LocalCUDAClient struct {
	Retries int
	Backoff time.Duration
	engine  *C.oa_engine
}

var (
	engineOnce sync.Once
	engineInst *C.oa_engine
	engineErr  error
)

// NewLocalCUDAClient mirrors NewOpenAIClient(apiKey, baseURL) (openai.go:38): it still demands a non-empty key so
// callers (pkg/assistants/simple.go:316, pkg/handlers/execute.go:138) need no change; baseURL "cuda://llama-3-8b"
// selects the model.  The engine is a process singleton because the reference builds a client per request.
func NewLocalCUDAClient(apiKey string, baseURL string) (*LocalCUDAClient, error) {
	if apiKey == "" {
		return nil, fmt.Errorf("OPENAI_API_KEY is not set")
	}
	engineOnce.Do(func() {
		runtime.LockOSThread() // oa_last_error() is thread-local
		defer runtime.UnlockOSThread()
		// cuda://<preset> names the model to load; anything else after the scheme (the handler's "gpt-4" default, execute.go:168-171)
		// falls back to $OPSAGENT_LOCAL_MODEL or llama-3-8b — requests are then answered under model_aliases "*"
		model := os.Getenv("OPSAGENT_LOCAL_MODEL")
		if m := strings.TrimPrefix(baseURL, "cuda://"); m != baseURL {
			switch m {
			case "llama-3.2-1b", "llama-3-8b", "qwen2.5-32b", "llama-3-70b":
				model = m
			}
		}
		if model == "" {
			model = "llama-3-8b"
		}
		// model_aliases "*": the reference forwards req.CurrentModel, or "gpt-4" when it is empty (pkg/handlers/execute.go:168-171);
		// a single-model local engine answers to whatever name the unmodified caller sends
		cfg := C.CString(fmt.Sprintf(`{"model": %q, "max_batch": 256, "max_seq_len": 16384, "model_aliases": "*"}`, model))
		defer C.free(unsafe.Pointer(cfg))
		if rc := C.oa_engine_create(cfg, &engineInst); rc != 0 {
			engineErr = fmt.Errorf("oa_engine_create: %d %s", int(rc), C.GoString(C.oa_last_error()))
		}
	})
	if engineErr != nil {
		return nil, engineErr
	}
	return &LocalCUDAClient{Retries: 5, Backoff: time.Second, engine: engineInst}, nil
}

// Chat — same signature and error behaviour as (*OpenAIClient).Chat (openai.go:69-104).
//
// Threading: the goroutine blocks in ONE cgo call at a time (oa_chat_wait_ex with a bounded timeout, re-entered until the completion is
// there), and error text comes back in a caller-owned buffer (the *_ex entry points), never through the thread-local oa_last_error() — so no
// runtime.LockOSThread: a goroutine may migrate between OS threads around cgo calls and nothing here depends on thread identity.
// Hundreds of goroutines batch inside the engine (continuous batching); a request whose goroutine gives up is cancelled so that it stops
// consuming KV pages and decode slots.
func (c *LocalCUDAClient) Chat(model string, maxTokens int, prompts []openai.ChatCompletionMessage) (string, error) {
	return c.ChatContext(context.Background(), model, maxTokens, prompts)
}

// ChatContext is Chat with cancellation (the reference passes context.Background() to CreateChatCompletion, openai.go:79; a caller
// with a deadline can use this directly).
func (c *LocalCUDAClient) ChatContext(ctx context.Context, model string, maxTokens int, prompts []openai.ChatCompletionMessage) (string, error) {
	if len(prompts) == 0 {
		return "", fmt.Errorf("prompts cannot be empty") // the caller checks this too (pkg/assistants/simple.go:312)
	}
	msgs := (*[1 << 20]C.oa_msg)(C.malloc(C.size_t(len(prompts)) * C.size_t(unsafe.Sizeof(C.oa_msg{}))))[:len(prompts):len(prompts)]
	defer C.free(unsafe.Pointer(&msgs[0]))
	for i, p := range prompts {
		msgs[i].role = C.CString(p.Role)
		msgs[i].content = C.CString(p.Content)
		defer C.free(unsafe.Pointer(msgs[i].role))
		defer C.free(unsafe.Pointer(msgs[i].content))
	}
	cmodel := C.CString(model)
	defer C.free(unsafe.Pointer(cmodel))
	req := C.oa_chat_req{model: cmodel, msgs: &msgs[0], n_msgs: C.int32_t(len(prompts)), max_tokens: C.int32_t(maxTokens),
		temperature: C.float(math.SmallestNonzeroFloat32)}
	const errCap = 512
	errBuf := (*C.char)(C.malloc(errCap))
	defer C.free(unsafe.Pointer(errBuf))

	backoff := c.Backoff
	for try := 0; try < c.Retries; try++ {
		var ticket C.uint64_t
		rc := int(C.oa_chat_submit_ex(c.engine, &req, &ticket, errBuf, errCap))
		for rc == 0 {
			var resp C.oa_chat_resp
			rc = int(C.oa_chat_wait_ex(c.engine, ticket, 250 /* ms */, &resp, errBuf, errCap))
			if rc == 0 {
				out := C.GoStringN(resp.content, C.int(resp.content_len))
				C.oa_free_resp(&resp)
				return out, nil
			}
			if rc != 408 { // anything but "not finished yet"
				break
			}
			if err := ctx.Err(); err != nil {
				C.oa_chat_cancel(c.engine, ticket)
				return "", err
			}
			rc = 0
		}
		err := &openai.APIError{HTTPStatusCode: rc, Message: C.GoString(errBuf)}
		switch rc {
		case 401:
			return "", err
		case 429, 500:
			time.Sleep(backoff)
			backoff *= 2
			continue
		default:
			return "", err
		}
	}
	return "", fmt.Errorf("OpenAI request throttled after retrying %d times", c.Retries)
}

// ServeLocalCUDA starts the engine library's own OpenAI-compatible HTTP endpoint (csrc/http_server.cpp: POST /v1/chat/completions incl.
// `tools`, GET /v1/models, GET /api/perf/stats) on the process-wide engine, for the callers that cannot go through the Chat seam: the swarm-go
// flows build their own OpenAI client from OPENAI_API_BASE (pkg/workflows/swarm.go:80-89).  A maintainer calls it once at start-up
// (cmd/kube-copilot/main.go) and points OPENAI_API_BASE at the returned URL.  `addr` is "host:port" ("127.0.0.1:0" picks a free port).
func ServeLocalCUDA(addr string) (string, error) {
	if _, err := NewLocalCUDAClient("local", "cuda://"); err != nil {
		return "", err
	}
	host, port, ok := strings.Cut(addr, ":")
	if !ok {
		return "", fmt.Errorf("ServeLocalCUDA: addr must be host:port")
	}
	runtime.LockOSThread() // oa_http_last_error() is thread-local
	defer runtime.UnlockOSThread()
	opts := C.CString(fmt.Sprintf(`{"host": %q, "port": %s, "require_key": 1}`, host, port))
	defer C.free(unsafe.Pointer(opts))
	var front *C.oa_http
	engines := []*C.oa_engine{engineInst}
	if rc := C.oa_http_start(&engines[0], 1, opts, &front); rc != 0 {
		return "", fmt.Errorf("oa_http_start: %d %s", int(rc), C.GoString(C.oa_http_last_error()))
	}
	return fmt.Sprintf("http://%s:%d/v1", host, int(C.oa_http_port(front))), nil
}
