// Package b200engine is the cgo binding a KubeAI maintainer adds (internal/b200engine/engine.go) to serve
// /openai/v1/chat/completions and /openai/v1/completions from the in-process H100 engine instead of proxying to a backend
// pod (internal/modelproxy/handler.go:96-159, internal/manager/run.go:267-275).
//
// It binds include/b200engine.h one to one; no logic lives here.  This image has no Go toolchain, so the file is
// committed as source and is not compiled by the repository's build: the same entry points are exercised through ctypes
// (kubeai_b200/_lib.py) and by the C++ process entry points (cmd/b200serve.cc), and tests/test_abi.py checks that every
// function this file calls is declared in the header and exported by libb200engine.so.
//
// Build inside KubeAI:  CGO_ENABLED=1 (Dockerfile:24 sets 0 today),  CGO_CFLAGS=-I<repo>/include,
//                       CGO_LDFLAGS="-L<repo>/kubeai_b200/lib -lb200engine -lcudart".
package b200engine

/*
#cgo LDFLAGS: -lb200engine -lcudart
#include <stdlib.h>
#include "b200engine.h"

// trampolines: cgo cannot pass Go funcs as C callbacks directly
extern int goBegin(void* ud, int status, char* ctype);
extern int goWrite(void* ud, char* data, size_t n);
static b200_response_writer make_writer(void* ud) {
  b200_response_writer w = { ud, (int (*)(void*, int, const char*))goBegin, (int (*)(void*, const char*, size_t))goWrite };
  return w;
}
*/
import "C"

import (
	"errors"
	"io"
	"net/http"
	"runtime/cgo"
	"unsafe"
)

type Engine struct{ h *C.b200_engine }

func New(device int, cfg func(*C.b200_config)) (*Engine, error) {
	var c C.b200_config
	C.b200_config_default(&c)
	c.device = C.int32_t(device)
	if cfg != nil {
		cfg(&c)
	}
	var h *C.b200_engine
	if rc := C.b200_engine_create(&c, &h); rc != 0 {
		return nil, errors.New(C.GoString(C.b200_last_error()))
	}
	return &Engine{h}, nil
}

// SpeculativeConfig applies vLLM's --speculative-config JSON (the "ngram" method only; KubeAI passes it through
// Model.spec.args) to an engine config; use it inside New's cfg callback.  Without it speculation stays off, the
// b200_config_default setting.
func SpeculativeConfig(c *C.b200_config, json string) error {
	s := C.CString(json)
	defer C.free(unsafe.Pointer(s))
	if rc := C.b200_speculative_config_parse(s, c); rc != 0 {
		return errors.New(C.GoString(C.b200_last_error()))
	}
	return nil
}

// Token-level API (what a Go-side SSE writer would use): submit, then wait+poll until finished.
func (e *Engine) Submit(ids []int32, maxTokens int) (uint64, error) {
	sp := C.b200_sampling{max_tokens: C.int32_t(maxTokens), ignore_eos: 0}
	var id C.uint64_t
	if rc := C.b200_submit(e.h, (*C.int32_t)(unsafe.Pointer(&ids[0])), C.int32_t(len(ids)), &sp, &id); rc != 0 {
		return 0, errors.New(C.GoString(C.b200_last_error()))
	}
	return uint64(id), nil
}

func (e *Engine) Poll(id uint64, buf []int32) (n int, finished int, u C.b200_usage, err error) {
	var cn, fin C.int32_t
	C.b200_wait(e.h, C.uint64_t(id), 200000) // 200 ms; loop on timeout to observe ctx.Done()
	if rc := C.b200_poll(e.h, C.uint64_t(id), (*C.int32_t)(unsafe.Pointer(&buf[0])), C.int32_t(len(buf)), &cn, &fin, &u); rc != 0 {
		return 0, 0, u, errors.New(C.GoString(C.b200_last_error()))
	}
	return int(cn), int(fin), u, nil
}

// Embedding API (an engine created with runner = 1, pooling): one request per input; Embedding blocks at most 200 ms and
// returns the vector (len = the model's hidden size) once finished is B200_FINISH_STOP.
func (e *Engine) SubmitEmbed(ids []int32, normalize bool) (uint64, error) {
	var id C.uint64_t
	norm := C.int32_t(0)
	if normalize {
		norm = 1
	}
	if rc := C.b200_submit_embed(e.h, (*C.int32_t)(unsafe.Pointer(&ids[0])), C.int32_t(len(ids)), norm, &id); rc != 0 {
		return 0, errors.New(C.GoString(C.b200_last_error()))
	}
	return uint64(id), nil
}

func (e *Engine) Embedding(id uint64, vec []float32) (finished int, u C.b200_usage, err error) {
	var fin C.int32_t
	C.b200_wait(e.h, C.uint64_t(id), 200000)
	if rc := C.b200_poll_embedding(e.h, C.uint64_t(id), (*C.float)(unsafe.Pointer(&vec[0])), C.int32_t(len(vec)), &fin, &u); rc != 0 {
		return 0, u, errors.New(C.GoString(C.b200_last_error()))
	}
	return int(fin), u, nil
}

// Score API (a pooling engine with num_labels > 0, a cross-encoder): one request per tokenized (query, document) pair;
// Score blocks at most 200 ms and returns the scores (len = num_labels) once finished is B200_FINISH_STOP.
func (e *Engine) SubmitScore(ids []int32, useActivation bool) (uint64, error) {
	var id C.uint64_t
	act := C.int32_t(0)
	if useActivation {
		act = 1
	}
	if rc := C.b200_submit_score(e.h, (*C.int32_t)(unsafe.Pointer(&ids[0])), C.int32_t(len(ids)), act, &id); rc != 0 {
		return 0, errors.New(C.GoString(C.b200_last_error()))
	}
	return uint64(id), nil
}

func (e *Engine) Score(id uint64, scores []float32) (finished int, u C.b200_usage, err error) {
	var fin C.int32_t
	C.b200_wait(e.h, C.uint64_t(id), 200000)
	if rc := C.b200_poll_score(e.h, C.uint64_t(id), (*C.float)(unsafe.Pointer(&scores[0])), C.int32_t(len(scores)), &fin, &u); rc != 0 {
		return 0, u, errors.New(C.GoString(C.b200_last_error()))
	}
	return int(fin), u, nil
}

// SubmitN starts n parallel samples of one prompt (vLLM's n): one prefill, n request ids for Poll / Abort.
func (e *Engine) SubmitN(prompt []int32, sp *C.b200_sampling, n int) ([]uint64, error) {
	ids := make([]C.uint64_t, n)
	if rc := C.b200_submit_n(e.h, (*C.int32_t)(unsafe.Pointer(&prompt[0])), C.int32_t(len(prompt)), sp, C.int32_t(n), &ids[0]); rc != 0 {
		return nil, errors.New(C.GoString(C.b200_last_error()))
	}
	out := make([]uint64, n)
	for i, id := range ids {
		out[i] = uint64(id)
	}
	return out, nil
}

// WaitAny blocks (at most 200 ms) until any member of one SubmitN group has tokens to Poll or is finished, so a Go-side
// writer streams n choices without waiting behind one that is preempted.
func (e *Engine) WaitAny(ids []uint64) {
	c := make([]C.uint64_t, len(ids))
	for i, id := range ids {
		c[i] = C.uint64_t(id)
	}
	C.b200_wait_any(e.h, &c[0], C.int32_t(len(c)), 200000)
}

func (e *Engine) Abort(id uint64) { C.b200_abort(e.h, C.uint64_t(id)) } // client went away: frees the KV blocks

// Failed reports whether a CUDA failure has poisoned this replica; the serving shell then drops it from the endpoint
// set the way reconcileEndpoints drops a vanished pod (internal/loadbalancer/group.go:119-131).
func (e *Engine) Failed() bool { return C.b200_engine_is_failed(e.h) != 0 }

func (e *Engine) Close() { C.b200_engine_destroy(e.h) }

// Whole-handler API: the C++ shell does parse -> route -> generate -> SSE; Go only forwards bytes.
type Server struct{ h *C.b200_server }

// NewServer wires one engine per local GPU behind the router (strategy: 0 LeastLoad, 1 PrefixHash,
// api/k8s/v1/model_types.go:173-209 defaults for the CHWBL parameters).
func NewServer(model string, strategy int, engines []*Engine) (*Server, error) {
	cm := C.CString(model)
	defer C.free(unsafe.Pointer(cm))
	cfg := C.b200_server_config{model: cm, strategy: C.int32_t(strategy), mean_load_pct: 125, replication: 256,
		prefix_char_length: 100, max_retries: 3, default_max_tokens: 256, vocab: 128256, max_model_len: 2048,
		enable_sampling: 1, enable_logprobs: 1, enable_logits_processors: 1, enable_prompt_logprobs: 1,
		max_n: 128} // the engines' max_num_seqs (b200_config_default)
	hs := make([]*C.b200_engine, len(engines))
	for i, e := range engines {
		hs[i] = e.h
	}
	var s *C.b200_server
	if rc := C.b200_server_create(&cfg, (**C.b200_engine)(unsafe.Pointer(&hs[0])), C.int32_t(len(hs)), &s); rc != 0 {
		return nil, errors.New(C.GoString(C.b200_last_error()))
	}
	return &Server{s}, nil
}

func (s *Server) Close() { C.b200_server_destroy(s.h) }

// Tokenizer is the checkpoint's tokenizer.json (Llama-3 family) loaded on the host side of the ABI: what the backend pod does
// with the model directory internal/modelcontroller/engine_vllm.go:34-41 hands it.
type Tokenizer struct{ h *C.b200_tokenizer }

func LoadTokenizer(tokenizerJSON string) (*Tokenizer, error) {
	cp := C.CString(tokenizerJSON)
	defer C.free(unsafe.Pointer(cp))
	var t *C.b200_tokenizer
	if rc := C.b200_tokenizer_load(cp, &t); rc != 0 {
		return nil, errors.New(C.GoString(C.b200_last_error()))
	}
	return &Tokenizer{t}, nil
}

func (t *Tokenizer) Close() { C.b200_tokenizer_destroy(t.h) }

// UseTokenizer makes the server render prompts with the Llama-3 chat template, stop at <|eot_id|> / <|end_of_text|> and
// detokenise its stream incrementally.  The tokenizer must outlive the server.
func (s *Server) UseTokenizer(t *Tokenizer) error {
	if rc := C.b200_server_set_tokenizer(s.h, t.h); rc != 0 {
		return errors.New(C.GoString(C.b200_last_error()))
	}
	return nil
}

//export goBegin
func goBegin(ud unsafe.Pointer, status C.int, ctype *C.char) C.int {
	w := cgo.Handle(uintptr(ud)).Value().(http.ResponseWriter)
	w.Header().Set("Content-Type", C.GoString(ctype))
	w.Header().Set("X-Proxy", "lingo") // internal/modelproxy/handler.go:60
	w.WriteHeader(int(status))
	return 0
}

//export goWrite
func goWrite(ud unsafe.Pointer, data *C.char, n C.size_t) C.int {
	w := cgo.Handle(uintptr(ud)).Value().(http.ResponseWriter)
	if _, err := w.Write(C.GoBytes(unsafe.Pointer(data), C.int(n))); err != nil {
		return 1 // client gone -> the shell aborts the sequence
	}
	if f, ok := w.(http.Flusher); ok {
		f.Flush() // text/event-stream: flush per chunk, as ReverseProxy does
	}
	return 0
}

// ServeHTTP is a drop-in for modelproxy.Handler (mounted at /openai/v1/{chat/,}completions,
// internal/openaiserver/handler.go:38-39).
func (s *Server) ServeHTTP(w http.ResponseWriter, r *http.Request) {
	body, err := io.ReadAll(r.Body)
	if err != nil || len(body) == 0 {
		http.Error(w, `{"error":"bad request: reading body"}`, http.StatusBadRequest)
		return
	}
	h := cgo.NewHandle(w)
	defer h.Delete()
	cw := C.make_writer(unsafe.Pointer(uintptr(h)))
	m, p, ct := C.CString(r.Method), C.CString("/openai"+r.URL.Path), C.CString(r.Header.Get("Content-Type"))
	defer C.free(unsafe.Pointer(m)); defer C.free(unsafe.Pointer(p)); defer C.free(unsafe.Pointer(ct))
	C.b200_server_handle(s.h, m, p, ct, (*C.char)(unsafe.Pointer(&body[0])), C.size_t(len(body)), &cw)
}
