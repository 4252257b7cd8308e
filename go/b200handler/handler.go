// Package b200handler is the cgo shim that drops the GPU engine into CrowdLlama's worker path.
//
// It builds a crowdllama.UnifiedAPIHandler (pkg/crowdllama/api.go:19) with the same contract as
// crowdllama.WorkerAPIHandler (api.go:45-96), replacing the HTTP round trip to Ollama
// (callOllamaAPI, api.go:108-160) by one blocking C call into libclengine.so.
//
// NOTE: this package cannot be compiled in the build image (no Go toolchain, no module proxy); it is
// the reference-side binding a maintainer adds.  The C-ABI it binds is exercised by the Python
// ctypes binding and tests in this repository.  See INTEGRATION.md.
package b200handler

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../crowdllama_b200/lib -lclengine -Wl,-rpath,${SRCDIR}/../../crowdllama_b200/lib
#include <stdlib.h>
#include "clengine.h"
extern int goFrameCallback(void* user, uint8_t* msg, size_t len);   // //export in callbacks.go
*/
import "C"

import (
	"context"
	"fmt"
	"math"
	"runtime/cgo"
	"unsafe"

	"google.golang.org/protobuf/proto"

	llamav1 "github.com/crowdllama/crowdllama-pb/llama/v1"
	"github.com/crowdllama/crowdllama/pkg/crowdllama"
)

// Engine owns one GPU (one worker process per GPU; the 8 GPUs of a box are 8 worker peers).
type Engine struct {
	h     *C.cl_engine
	model string
}

// Config mirrors the CROWDLLAMA_* knobs added for the GPU worker (pkg/config/config.go:58-79 style).
type Config struct {
	Device     int    // CROWDLLAMA_B200_DEVICE
	ModelName  string // name advertised in Resource.SupportedModels and matched exactly (manager.go:349-354), e.g. "llama3:8b"
	ModelDir   string // CROWDLLAMA_B200_MODEL_DIR: HF checkpoint directory (*.safetensors + config.json [+ tokenizer.json]) or one .safetensors file
	Preset     string // architecture when ModelDir has no config.json / synthetic weights: "llama3-8b" | "mistral-7b" | "tinyllama-1.1b"
	Tokenizer  string // tokenizer.json outside ModelDir (optional; ModelDir/tokenizer.json is picked up by the engine itself)
	ChatFamily string // "llama3" | "mistral" | "zephyr" | "chatml" | "" (auto-detect from the added tokens)
	Seed       uint64 // synthetic weights only (ModelDir == "")
	MaxBatch   int
	KVBytes    int64
}

func lastErr(rc C.int) error {
	return fmt.Errorf("%s: %s", C.GoString(C.cl_strerror(rc)), C.GoString(C.cl_last_error()))
}

func cstr(s string) (*C.char, func()) {
	if s == "" {
		return nil, func() {}
	}
	p := C.CString(s)
	return p, func() { C.free(unsafe.Pointer(p)) }
}

// New replaces "start the embedded Ollama server" (cmd/crowdllama/main.go:283-297).
func New(cfg Config) (*Engine, error) {
	var c C.cl_engine_config
	C.cl_default_engine_config(&c)
	name, f1 := cstr(cfg.ModelName)
	preset, f2 := cstr(cfg.Preset)
	dir, f3 := cstr(cfg.ModelDir)
	defer f1()
	defer f2()
	defer f3()
	c.device, c.model_name, c.preset, c.weights_path = C.int32_t(cfg.Device), name, preset, dir
	c.weights_seed, c.max_batch, c.max_seqs = C.uint64_t(cfg.Seed), C.int32_t(cfg.MaxBatch), C.int32_t(cfg.MaxBatch)
	c.kv_pool_bytes, c.start_scheduler = C.int64_t(cfg.KVBytes), 1
	var h *C.cl_engine
	if rc := C.cl_engine_create(&c, &h); rc != C.CL_OK {
		return nil, lastErr(rc)
	}
	e := &Engine{h: h, model: cfg.ModelName}
	if cfg.Tokenizer != "" {
		tok, f4 := cstr(cfg.Tokenizer)
		fam, f5 := cstr(cfg.ChatFamily)
		defer f4()
		defer f5()
		if rc := C.cl_engine_load_tokenizer(h, tok, fam); rc != C.CL_OK {
			err := lastErr(rc)
			e.Close()
			return nil, err
		}
	}
	return e, nil
}

func (e *Engine) Close() { C.cl_engine_destroy(e.h) }

// Handler returns the drop-in for crowdllama.WorkerAPIHandler(ollamaBaseURL).  It is safe to call from many
// goroutines (one per inbound stream, pkg/peer/peer.go:177-182): the library enqueues into the engine's
// continuous-batching scheduler and blocks; each in-flight call pins one OS thread.
//
// The request travels as bytes through cl_handle_message_stream, so GenerateRequest.Options (field 4: seed,
// temperature, num_predict ... — the §8f-row-3 wire extension) is applied inside the library exactly as for streamed
// requests, and ctx cancellation (gateway timeout, client gone) reaches the scheduler: the frame callback returns
// nonzero once ctx is done and the request ends with done_reason "cancelled".  A request without options gets
// Ollama's defaults, like the reference (api.go:109-118 sends none).  Response fields as api.go:77-92: WorkerId
// "worker", TotalDuration = UnixNano (kept bug-for-bug), one Done=true message.
func (e *Engine) Handler() crowdllama.UnifiedAPIHandler {
	return func(ctx context.Context, req *llamav1.BaseMessage) (*llamav1.BaseMessage, error) {
		generateReq := req.GetGenerateRequest()
		if generateReq == nil { // api.go:48-51
			return nil, fmt.Errorf("expected GenerateRequest, got different message type")
		}
		// Ask the engine for frames even though one message goes back: the frame callback is where ctx is polled, so
		// a cancelled request stops decoding within one batch of tokens instead of running to num_predict.
		one := proto.Clone(req).(*llamav1.BaseMessage)
		one.GetGenerateRequest().Stream = true
		var text []byte
		var last *llamav1.GenerateResponse
		err := e.HandleStream(ctx, one, func(frame *llamav1.BaseMessage) error {
			if g := frame.GetGenerateResponse(); g != nil {
				text = append(text, g.Response...)
				last = g
			}
			return nil
		})
		if err != nil {
			return nil, err
		}
		if ctx.Err() != nil {
			return nil, ctx.Err()
		}
		if last == nil || !last.Done {
			return nil, fmt.Errorf("failed to call GPU engine: no final response frame")
		}
		last.Response = string(text) // api.go:80: the full assistant text in ONE message (the reference never streams, api.go:155)
		return &llamav1.BaseMessage{Message: &llamav1.BaseMessage_GenerateResponse{GenerateResponse: last}}, nil
	}
}

// HandleStream is the streaming form (SURVEY.md §8f row 4; the reference rejects stream:true, api.go:155): the
// request is handed to libclengine as bytes, every response frame (Done=false text deltas, then Done=true) comes
// back through emit on the calling goroutine.  A failing emit or a done ctx cancels the request inside the engine.
func (e *Engine) HandleStream(ctx context.Context, req *llamav1.BaseMessage, emit func(*llamav1.BaseMessage) error) error {
	raw, err := proto.Marshal(req)
	if err != nil {
		return err
	}
	var emitErr error
	h := cgo.NewHandle(func(frame []byte) error {
		if ctx.Err() != nil {
			return ctx.Err()
		}
		var m llamav1.BaseMessage
		if err := proto.Unmarshal(frame, &m); err != nil {
			emitErr = err
			return err
		}
		if err := emit(&m); err != nil {
			emitErr = err
			return err
		}
		return nil
	})
	defer h.Delete()
	buf := C.CBytes(raw) // copied: C never retains Go memory
	defer C.free(buf)
	if rc := C.cl_handle_message_stream(e.h, (*C.uint8_t)(buf), C.size_t(len(raw)), nil,
		C.cl_frame_cb(C.goFrameCallback), unsafe.Pointer(&h)); rc != C.CL_OK {
		return fmt.Errorf("failed to call GPU engine: %w", lastErr(rc))
	}
	return emitErr
}

// AdvertisedThroughput quantises the engine's capacity figure to half-octave buckets, AdvertisedLoad to two levels —
// the same rule as crowdllama_b200/router.py (advertised_throughput / advertised_load) and INTEGRATION.md "What to
// advertise": FindBestWorker (pkg/peermanager/manager.go:338-387) takes a strict maximum over metadata that is
// 10-30 s old, so numbers that move with the load send every request to one worker between two refreshes.
// cl_stats.tokens_per_sec is already load-independent (memory bandwidth / model bytes x max_batch); the measured rate
// is cl_stats.measured_tokens_per_sec and must NOT be advertised.
func AdvertisedThroughput(tokensPerSec float64) float64 {
	if tokensPerSec <= 0 {
		return 0
	}
	return math.Round(math.Pow(2, math.Round(math.Log2(tokensPerSec)*2)/2)*10) / 10
}

// Load = 1 only once a whole extra batch is waiting (cl_stats.load >= 2): the metadata is older than a request lasts,
// and a flag at load >= 1 shuns every worker that happened to be full at refresh time (tools/route_sim.py).
func AdvertisedLoad(load float64) float64 {
	if load >= 2 {
		return 1
	}
	return 0
}

// Stats feeds truthful routing metadata into crowdllama.Resource (pkg/crowdllama/types.go:30-40),
// replacing the constants at pkg/peer/peer.go:319-358.
func (e *Engine) Stats(r *crowdllama.Resource) error {
	var s C.cl_stats
	if rc := C.cl_engine_stats(e.h, &s); rc != C.CL_OK {
		return lastErr(rc)
	}
	r.TokensThroughput = AdvertisedThroughput(float64(s.tokens_per_sec))
	r.Load = AdvertisedLoad(float64(s.load))
	r.VRAMGB, r.GPUModel = int(s.vram_gb), C.GoString(&s.gpu_model[0])
	r.SupportedModels = []string{e.model}
	return nil
}
