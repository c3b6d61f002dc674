/* b200engine.h — C ABI of the in-process H100 inference engine (the b200 prefix is historical).
 *
 * This is the drop-in boundary described in SURVEY.md §8(b).  The reference (kubeai-project/kubeai)
 * has no FFI: a backend is an HTTP server reached through
 *     internal/modelproxy/handler.go:158   proxy.ServeHTTP(w, pr.httpRequest())
 * after internal/loadbalancer/load_balancer.go:191 AwaitBestAddress picked an "ip:port".
 * The replacement keeps those Go interfaces (modelproxy/handler.go:18-25) and swaps the HTTP hop for
 * the calls below (cgo binding shown in INTEGRATION.md).  Every function returns 0 on success and a
 * negative b200_status on failure; b200_last_error() gives the message for the calling thread.
 * Plain pointers and sizes only; the caller owns every buffer it passes; the engine copies before
 * returning.  No exceptions cross this boundary.
 */
#ifndef B200ENGINE_H
#define B200ENGINE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  B200_OK = 0,
  B200_ERR_INVALID = -1,   /* bad argument / shape */
  B200_ERR_CUDA = -2,      /* CUDA runtime / launch failure */
  B200_ERR_OOM = -3,       /* device or KV pool exhausted */
  B200_ERR_NOT_FOUND = -4, /* unknown request id / tensor name */
  B200_ERR_NO_DEVICE = -5, /* no CUDA device: the product path never falls back to CPU */
  B200_ERR_CANCELLED = -6, /* context cancelled while waiting (router) */
  B200_ERR_TIMEOUT = -7
} b200_status;

const char* b200_last_error(void);
/* "kubeai-b200 <version> sm_90a" */
const char* b200_version(void);

/* ------------------------------------------------------------------ engine (one per GPU replica)
 * Replaces the backend pod that internal/modelcontroller/engine_vllm.go:82-100 launches. */

typedef struct b200_tokenizer b200_tokenizer;   /* csrc/tokenizer.cc, declared with its functions below */
typedef struct b200_engine b200_engine;

typedef struct {
  int32_t device;             /* CUDA ordinal */
  /* model architecture (Llama family; head_dim is fixed at 128, q_heads == 4 * kv_heads) */
  int32_t num_layers, hidden, q_heads, kv_heads, intermediate, vocab;
  float rms_eps;              /* 1e-5 */
  float rope_theta;           /* 500000 */
  int32_t max_model_len;      /* vLLM --max-model-len */
  int32_t max_num_seqs;       /* vLLM --max-num-seqs */
  int32_t max_batched_tokens; /* vLLM --max-num-batched-tokens (per-step token budget) */
  int64_t num_kv_blocks;      /* 16-token pages in the pool; 0 = size from kv_fraction of free HBM */
  float kv_fraction;          /* vLLM --gpu-memory-utilization analogue (of free memory), default 0.85 */
  int32_t enable_prefix_caching;
  int32_t eos_token_id;       /* -1 = none */
  uint64_t seed;              /* seeded random-init weights (no checkpoints offline) */
  float init_scale;           /* multiplies the lm_head init so greedy logits are separated; default 4 */
  int32_t manual_step;        /* 1 = no background thread; caller drives b200_engine_step() */
  int32_t record_steps;       /* >0 = keep the device-side inputs of the last N steps for b200_engine_replay */
  /* RoPE frequency scaling (HF config.json "rope_scaling" / "rope_parameters"; vLLM rotary_embedding/__init__.py get_rope):
   * 0 = none, 1 = "linear" (positions / factor), 2 = "llama3" (Llama-3.1+: per-frequency factor between the low and high
   * wavelength bounds).  b200_config_from_hf fills these; any other rope_type is refused there. */
  int32_t rope_scaling_type;
  float rope_factor, rope_low_freq_factor, rope_high_freq_factor;
  int32_t rope_original_max_pos;
} b200_config;

typedef struct {
  int32_t max_tokens;
  float temperature;          /* only greedy (temperature < 1e-5, vllm/v1/sample/sampler.py:17) is implemented */
  int32_t ignore_eos;
  int32_t num_stop_ids;
  const int32_t* stop_ids;
} b200_sampling;

typedef struct {
  int32_t prompt_tokens;
  int32_t cached_tokens;      /* usage.prompt_tokens_details.cached_tokens (api/openai/v1/usage.go:5-25) */
  int32_t completion_tokens;
} b200_usage;

enum { B200_RUNNING = 0, B200_FINISH_STOP = 1, B200_FINISH_LENGTH = 2, B200_FINISH_ABORTED = 3, B200_FINISH_ERROR = 4 };

typedef struct {
  int64_t steps;              /* forward steps executed */
  int32_t running, waiting;
  int64_t kv_blocks_total, kv_blocks_free;
  int64_t prompt_tokens, cached_prompt_tokens, generated_tokens;
  int64_t preemptions;
  double last_step_device_us; /* CUDA-event time of the last forward */
  double total_device_us;     /* sum over steps */
  int64_t last_step_tokens;   /* tokens in the last forward (T) */
  int64_t kernel_launches;    /* kernels launched by this engine so far */
  int64_t h2d_bytes, d2h_bytes; /* step inputs copied to the device / sampled ids copied back, totals */
} b200_stats;

typedef struct {
  int32_t tokens;             /* T of the step */
  int32_t decode_seqs, prefill_seqs, sampled;
  int64_t kv_tokens_read;     /* unique K/V tokens streamed by this step: sum over sequences of their context length */
  double device_us;
} b200_step_info;

void b200_config_default(b200_config* cfg);          /* Llama-3-8B shape, vLLM-like limits */
int b200_engine_create(const b200_config* cfg, b200_engine** out);
void b200_engine_destroy(b200_engine* e);

int b200_submit(b200_engine* e, const int32_t* prompt_ids, int32_t n, const b200_sampling* sp, uint64_t* req_id);
/* Drain newly generated token ids (at most cap).  *finished gets a B200_FINISH_* code or 0. */
int b200_poll(b200_engine* e, uint64_t req_id, int32_t* out_ids, int32_t cap, int32_t* n_out, int32_t* finished,
              b200_usage* usage);
/* Block until the request has undrained tokens or is finished (B200_ERR_TIMEOUT otherwise). */
int b200_wait(b200_engine* e, uint64_t req_id, int64_t timeout_us);
int b200_abort(b200_engine* e, uint64_t req_id);
/* Forget a finished request (frees its host-side record). */
int b200_release(b200_engine* e, uint64_t req_id);
int b200_stats_get(b200_engine* e, b200_stats* out);
/* 1 when a CUDA failure has poisoned this replica (every request fails with B200_FINISH_ERROR / B200_ERR_CUDA from then on):
 * the serving shell drops such a replica from the router's endpoint set (internal/loadbalancer/group.go:119-131). */
int b200_engine_is_failed(b200_engine* e);

/* manual_step mode: run one scheduler iteration + forward; *info may be NULL. Returns 1 if a step ran, 0 if idle. */
/* on != 0: requests that arrive between two steps are admitted in a fixed order (prompt content) instead of arrival order,
 * so concurrent clients that submit the same requests between the same steps get the same batches on every run.
 * Default 0 (first come, first served). */
int b200_engine_set_fixed_admission(b200_engine* e, int32_t on);
/* Submitted requests not yet finished (queued, running, or between chunks of a prompt). */
int32_t b200_engine_unfinished(b200_engine* e);
int b200_engine_step(b200_engine* e, b200_step_info* info);
/* manual_step mode: up to max_steps iterations back to back on the calling thread, pipelined the way the engine's own
 * loop thread runs: the tokens of step N are handed to the waiting API threads after step N+1 has been enqueued on the
 * GPU.  Returns when max_steps steps ran or the engine had nothing to run for idle_timeout_us.  infos (optional) gets
 * one entry per step, *n_done the number of steps that ran. */
int b200_engine_run(b200_engine* e, int32_t max_steps, int64_t idle_timeout_us, b200_step_info* infos, int32_t* n_done);
/* Re-run the forward passes of the last `n` recorded steps from their HBM-resident inputs,
 * `repeat` times back to back; returns CUDA-event milliseconds and what those steps carried. */
int b200_engine_replay(b200_engine* e, int32_t n, int32_t repeat, double* ms_total, int64_t* tokens,
                       int64_t* sampled, int64_t* kv_tokens_read, int64_t* launches);
/* Recording on (default) = each step's device inputs go to the replay ring; off = ring is frozen. */
int b200_engine_set_recording(b200_engine* e, int32_t on);
/* Timing aid: forward() does not launch the kernel classes in `mask` (bit 1 << B200_K_*); outputs are then garbage.
 * Replaying the same steps with and without a class gives its marginal cost under PDL overlap. */
int b200_engine_set_skip_mask(b200_engine* e, uint32_t mask);
/* Kernel classes of the forward pass, for per-class device timing. */
enum { B200_K_EMBED = 0, B200_K_NORM, B200_K_GEMM_QKV, B200_K_ROPE, B200_K_ATTN_DECODE, B200_K_ATTN_PREFILL,
       B200_K_GEMM_O, B200_K_GEMM_GU, B200_K_SILU, B200_K_GEMM_DOWN, B200_K_GEMM_LM, B200_K_ARGMAX, B200_K_NUM };
/* Re-run the last `n` recorded steps with a CUDA-event pair around every launch (on the engine's
 * stream) and return total microseconds and launch counts per kernel class (arrays of B200_K_NUM). */
int b200_engine_profile(b200_engine* e, int32_t n, double* class_us, int64_t* class_launches, int32_t num_classes);
/* Same, restricted to the recorded steps whose token count lies in [min_tokens, max_tokens] (decode-only steps vs
 * prefill bursts); also returns how many steps matched and their token / sampled-row / KV-token totals. */
int b200_engine_profile_range(b200_engine* e, int32_t n, int32_t min_tokens, int32_t max_tokens, double* class_us,
                              int64_t* class_launches, int32_t num_classes, int64_t* steps, int64_t* tokens,
                              int64_t* sampled, int64_t* kv_tokens_read);
/* Drop every cached prefix block (after a replay, which clobbers KV contents). */
int b200_engine_reset_prefix_cache(b200_engine* e);

/* Weights / buffers by name ("embed", "lm_head", "final_norm", "layers.<i>.{wqkv,wo,wgu,wdown,norm1,norm2}",
 * "cos_sin").  Tests copy weights out for the CPU oracle or write their own in. */
int b200_engine_tensor_info(b200_engine* e, const char* name, uint64_t* num_bytes, void** device_ptr);
int b200_engine_tensor_read(b200_engine* e, const char* name, void* host_dst, uint64_t cap);
int b200_engine_tensor_write(b200_engine* e, const char* name, const void* host_src, uint64_t n);
/* Debug/parity: run a plain forward over `n` tokens of ONE sequence (positions 0..n-1, fresh KV pages taken from
 * the pool and returned afterwards) and copy the bf16 logits of every position to host_logits [n, vocab]. */
int b200_engine_forward_logits(b200_engine* e, const int32_t* ids, int32_t n, void* host_logits_bf16);
/* Parity hook for decode steps (manual_step mode): with keep != 0 the lm_head of every later step leaves the complete
 * bf16 logits of its sampled rows in HBM (the serving path only keeps what the argmax needs); read_logits copies the
 * first `rows` rows [rows, vocab] of the last step, in the order the step sampled them (scheduling order). */
int b200_engine_set_keep_logits(b200_engine* e, int32_t keep);
int b200_engine_read_logits(b200_engine* e, void* host_logits_bf16, int32_t rows);

/* ------------------------------------------------------------------ checkpoints (SURVEY.md §8f-2)
 * HF-layout Llama checkpoints: <dir>/config.json + model.safetensors[.index.json] (BF16/F16/F32 tensors).
 * The reference mounts such a directory into the backend pod (internal/modelcontroller/model_source.go:231-287). */
/* Fill the architecture fields of cfg from <dir>/config.json; rejects head_dim != 128 and GQA != 4:1. */
int b200_config_from_hf(const char* dir, b200_config* cfg);
/* Replace the seeded weights of an idle engine with the checkpoint's (q/k/v and gate/up fused on load). */
int b200_engine_load_safetensors(b200_engine* e, const char* path);
/* JSON listing of the tensors of a checkpoint (dir, shard index or single file); returns the length needed. */
int64_t b200_safetensors_list(const char* path, char* buf, size_t cap);

/* ------------------------------------------------------------------ router
 * Port of internal/loadbalancer group / CHWBL / LeastLoad (group.go:25-150, balance_chwbl.go:14-162,
 * balance_least_load.go:3-23).  "Endpoints" are GPU replicas; address strings are kept so the
 * reference's tests can be replayed literally. */
typedef struct b200_router b200_router;
enum { B200_LB_LEAST_LOAD = 0, B200_LB_PREFIX_HASH = 1 };

int b200_router_create(int32_t replication, b200_router** out);
void b200_router_destroy(b200_router* r);
/* reconcileEndpoints (group.go:108-137): names/addresses parallel arrays; adapters[i] is a comma-separated list or NULL. */
int b200_router_set_endpoints(b200_router* r, const char* const* names, const char* const* addresses,
                              const char* const* adapters, int32_t n);
/* getBestAddr (group.go:53-88).  Blocks until an endpoint (serving `adapter`) exists or timeout_us passes
 * (<0 = forever, 0 = don't block).  addr_out receives the chosen address; *endpoint_token identifies the
 * endpoint for b200_router_done (the `done func()` of the Go API). */
int b200_router_pick(b200_router* r, int32_t strategy, const char* adapter, const char* prefix, int32_t prefix_len,
                     int32_t mean_load_pct, int64_t timeout_us, char* addr_out, int32_t addr_cap,
                     uint64_t* endpoint_token);
int b200_router_done(b200_router* r, uint64_t endpoint_token);
/* group.addInFlight (group.go:147-150) on a named endpoint; used by the replayed reference tests */
int b200_router_add_inflight(b200_router* r, const char* name, int64_t delta);
int b200_router_inflight(b200_router* r, const char* name, int64_t* endpoint_inflight, int64_t* total_inflight);
/* Prometheus text of the hash-lookup metrics (internal/metrics/metrics.go:19-26,51-76: iterations histogram with
 * buckets 1..1024, per-endpoint initial/final/default counters); returns the length needed. */
int64_t b200_router_metrics(b200_router* r, char* buf, size_t cap);
/* cespare/xxhash v1.1.0 Sum64 (seed 0) as used at balance_chwbl.go:140-142 */
uint64_t b200_xxh64(const void* data, size_t len);

/* ------------------------------------------------------------------ serving shell
 * internal/openaiserver + internal/modelproxy restated around the in-process engine: route table
 * (openaiserver/handler.go:20-49), ServeHTTP/proxyHTTP incl. error bodies and <=max_retries re-picks
 * (modelproxy/handler.go:57-159, request.go:45-63), ParseRequest (apiutils/request.go:64-225),
 * Prefix (api/openai/v1/chat_completions.go:525-543), the requests-active gauge
 * (metrics/metrics.go:16-27); plus tokenizer/chat template and vLLM-framed SSE (SURVEY.md K12/K13).
 * A Go http.Handler calls b200_server_handle with a writer that forwards to http.ResponseWriter. */
typedef struct b200_server b200_server;
typedef struct {
  void* ud;
  int (*begin)(void* ud, int status, const char* content_type); /* WriteHeader; non-zero return = client gone */
  int (*write)(void* ud, const char* data, size_t len);         /* Write + Flush;  non-zero return = client gone */
} b200_response_writer;
typedef struct {
  const char* model;           /* Model.metadata.name served by every replica */
  const char* adapters;        /* comma-separated adapter names, or NULL */
  int32_t strategy;            /* B200_LB_* (api/k8s/v1/model_types.go:173-209) */
  int32_t mean_load_pct;       /* default 125 */
  int32_t replication;         /* default 256 */
  int32_t prefix_char_length;  /* default 100 */
  int32_t max_retries;         /* default 3 (internal/manager/run.go:267) */
  int32_t default_max_tokens;  /* when the request has no max_tokens */
  int32_t vocab;               /* tokenizer range == engine vocab */
  int32_t max_model_len;
} b200_server_config;
int b200_server_create(const b200_server_config* cfg, b200_engine* const* replicas, int32_t n, b200_server** out);
void b200_server_destroy(b200_server* s);
/* One request through the handler chain; path includes the "/openai" prefix.  Returns the HTTP status. */
int b200_server_handle(b200_server* s, const char* method, const char* path, const char* content_type,
                       const char* body, size_t body_len, const b200_response_writer* writer);
/* apiutils.ParseRequest alone (parity tests): returns 0 or the HTTP status of the error; out_json receives
 * {"model","adapter","requested_model","prefix"} or {"error": ...}.  prefix_chars < 0 keeps the server's setting. */
int b200_server_parse_request(b200_server* s, const char* path, const char* content_type, const char* body,
                              size_t body_len, int32_t prefix_chars, char* out_json, size_t cap);
/* Plain HTTP/1.1 listener in front of b200_server_handle (thread per connection, chunked SSE). port 0 = ephemeral. */
int b200_server_listen(b200_server* s, const char* host, int32_t port, int32_t* bound_port);
/* Prometheus text (kubeai_inference_requests_active + engine gauges); returns the full length. */
int b200_server_metrics(b200_server* s, char* buf, size_t cap);
/* Fault injection for the retry path: the next `count` submits on `replica` fail; count < 0 = every submit fails, which
 * stands for an engine in the failed state: the first failure drops the replica from the router's endpoint set. */
/* Attach a tokenizer (b200_tokenizer_load; not owned, must outlive the server; NULL detaches): prompts are then rendered with
 * the Llama-3 chat framing / <|begin_of_text|> + encoded text, <|eot_id|> and <|end_of_text|> end a generation, and output text is
 * detokenised incrementally.  Without one the server keeps the synthetic tokenizer (SURVEY.md §8d). */
int b200_server_set_tokenizer(b200_server* s, const b200_tokenizer* t);
/* Host-only: the token ids the server would submit for this request body (parse + chat template + tokenizer).  Returns the
 * count (may exceed cap), -1 with b200_last_error() = "<status> <message>" when the request is rejected. */
int64_t b200_server_render_prompt(b200_server* s, const char* path, const char* content_type, const char* body, size_t len,
                                  int32_t* ids, size_t cap);
int b200_server_inject_fault(b200_server* s, int32_t replica, int32_t count);
/* Synthetic tokenizer (ids 0..255 = bytes; " wxyz" spellings round-trip every id). Return the full count/length. */
int b200_tokenize(int32_t vocab, const char* text, size_t len, int32_t* out, int32_t cap);
int b200_detokenize(int32_t vocab, const int32_t* ids, int32_t n, char* out, size_t cap);

/* ------------------------------------------------------------------ load generator
 * benchmarks/multi-turn-chat-go restated (main.go:26-136, benchmark/runner.go:153-352), plus
 * p50/p99 TTFT and a synthetic thread generator of the published workload's shape. */
typedef struct {
  const char* request_model;        /* Config.RequestModel */
  int32_t max_concurrent_threads;   /* Config.MaxConcurrentThreads */
  int32_t max_completion_tokens;    /* Config.MaxCompletionTokens */
  float temperature;                /* Config.Temperature (sent explicitly; 0 = greedy) */
  int32_t thread_count;             /* main.go:110-116 trim after the seeded shuffle; 0 = all */
  int64_t seed;
  double request_timeout_s;
  int32_t synth_threads;            /* used when threads_json == NULL */
  double synth_mean_msgs;           /* user messages per thread, clipped geometric on [5,30]; published mean 7.38 */
  int32_t synth_mean_words;         /* tokens per user message (log-normal mean) */
  int32_t vocab;
} b200_harness_config;
typedef struct {
  int32_t input_thread_count;
  double input_messages_per_thread_mean;
  double duration_s;
  int32_t request_count, failed_threads;
  double request_duration_mean_s, chunks_per_request_mean;
  double run_output_throughput, run_total_throughput;   /* tokens/s over the whole run incl. ramp */
  double ttft_mean_s, itl_mean_s;                        /* runner.go:228-229 arithmetic */
  double ttft_p50_s, ttft_p90_s, ttft_p99_s, itl_p50_s, itl_p99_s;   /* added for BASELINE.json's metric */
  int64_t prompt_tokens, cached_prompt_tokens, completion_tokens, total_tokens;
  char first_error[256];
} b200_harness_result;
void b200_harness_config_default(b200_harness_config* cfg);
/* JSON of the synthetic threads (same format as threads_json); returns the length needed (excl. NUL). */
int64_t b200_harness_synth_threads(const b200_harness_config* cfg, char* buf, size_t cap);
/* server != NULL: in-process transport (b200_server_handle); else HTTP/1.1 to host:port.
 * threads_json: the reference's input format [{"id":..,"messages":[{"role","content"},..]},..] or NULL = synthetic. */
/* Requests the load generators running in this process are about to have in flight: conversations in progress plus free
 * slots that a conversation still waiting to start will take.  Stepping an engine only while b200_engine_unfinished()
 * equals this makes the batches of a multi-turn run independent of client thread timing. */
int64_t b200_harness_expected_inflight(void);
int b200_harness_run(b200_server* server, const char* host, int32_t port, const b200_harness_config* cfg,
                     const char* threads_json, size_t threads_len, b200_harness_result* out);

/* ------------------------------------------------------------------ op-level entry points
 * Raw device pointers (bf16 unless noted) + a cudaStream_t passed as void* (NULL = default stream).
 * These are what the per-kernel parity tests and the microbenchmarks call. */
/* Schedule of b200_op_gemm: 2 = split-K sized to the device (default), 1 = every tile over its whole K.  Returns the
 * active variant. */
int b200_set_gemm_variant(int32_t v);
/* ---- byte-level BPE tokenizer over a local HF tokenizer.json of the Llama-3 family (csrc/tokenizer.cc).  Replaces, on the
 * host side of this ABI, the tokenizer + chat template the reference's backend pod applies to the model directory it is given
 * (internal/modelcontroller/engine_vllm.go:34-41).  Host-only: no GPU needed.  Other pipelines are refused at load time. */
int b200_tokenizer_load(const char* tokenizer_json_path, b200_tokenizer** out);
void b200_tokenizer_destroy(b200_tokenizer* t);
int32_t b200_tokenizer_vocab_size(const b200_tokenizer* t);
int32_t b200_tokenizer_token_id(const b200_tokenizer* t, const char* content);   /* -1 if absent */
/* Both return the full length (which may exceed cap: call again with a larger buffer), -1 on bad arguments.
 * allow_special: added / special tokens spelled in the text become their ids (as HF `encode` does). */
int64_t b200_tokenizer_encode(const b200_tokenizer* t, const char* text, size_t len, int32_t allow_special, int32_t* ids, size_t cap);
int64_t b200_tokenizer_decode(const b200_tokenizer* t, const int32_t* ids, size_t n, int32_t skip_special, char* buf, size_t cap);
/* Incremental detokenisation of a generated stream: a token may end inside a UTF-8 sequence, so push returns only complete text
 * (id < 0 flushes what is held).  The pushes concatenated equal b200_tokenizer_decode of all ids. */
typedef struct b200_detok_stream b200_detok_stream;
b200_detok_stream* b200_tokenizer_stream_new(const b200_tokenizer* t, int32_t skip_special);
void b200_tokenizer_stream_free(b200_detok_stream* d);
int64_t b200_tokenizer_stream_push(b200_detok_stream* d, int32_t id, char* buf, size_t cap);
/* Llama-3 instruct chat framing of n (role, content) messages; add_generation_prompt appends the assistant header. */
int64_t b200_tokenizer_chat_llama3(const b200_tokenizer* t, const char* const* roles, const char* const* contents, int32_t n,
                                   int32_t add_generation_prompt, int32_t* ids, size_t cap);

/* Host-only (no GPU needed): how a projection [N, K] of a step of T tokens is scheduled on a device with `sms` SMs.
 * out8: [0] token-tile size, [1] token tiles, [2] tiles (128 weight rows x token tile), [3] K-splits per tile, [4] CTAs,
 * [5] rule that chose the splits (1 one token tile, 2 several), [6] 0, [7] 0. */
int b200_schedule_query(int32_t N, int32_t K, int32_t T, int32_t sms, int32_t* out8);
/* Host-only: CTAs per (sequence, KV head) the engine gives decode attention when `num_work` sequences decode. */
int b200_attn_split_query(int32_t num_work, int32_t kv_heads, int32_t max_ctx, int32_t sms);
/* GEMM phase tracing: the wgmma GEMM records no timestamps, so only NULL (tracing off) is accepted; any buffer is
 * refused with B200_ERR_INVALID. */
int b200_op_gemm_trace(void* trace_dev);
/* Same contraction in the engine's form whatever the variant: split-K sized to the device, the partials summed in-kernel
 * in split order; N % 8 == 0 (the elementwise consumers read output rows 16 bytes at a time). */
int b200_op_gemm_deferred(const void* w, const void* x, void* out, int32_t N, int32_t T, int32_t K, void* stream);
int b200_op_gemm(const void* w, const void* x, void* out, int32_t N, int32_t T, int32_t K, void* stream);
/* The fused projection GEMM (csrc/gemm_wgmma.cu): acc = X' W^T with the split-K reduction finished in the kernel, a prologue (pro 0: X' = x; 1: X' = RMSNorm(x) from the per-slab sums of squares ssq_in [T, ssq_slabs] and norm_w)
 * and an epilogue on the bf16-rounded result (epi 0: out [T, N]; 1: out (in/out, residual) += acc, ssq_out [T, N/128], and
 * optionally (T <= 128) the RMSNorm of the new residual for the next projection;
 * 2: out [T, N/2] = silu(gate) * up with gate/up rows interleaved in 64-row blocks of w; 3: neox RoPE of q/k heads, q ->
 * out (the fused qkv buffer, ldo), k/v -> kv_layer pages; 4 (T <= 128): argmax_out [T] = argmax_n acc[t, n < n_valid]).  pro 1 needs T <= 128.
 * force, T <= 128: 0 automatic split count, n >= 1 or -n <= -2: n K-splits per tile, -1 automatic; T > 128: 0 automatic
 * token tile, >= 64 the requested token tile: the largest of 64 / 128 / 256 not above it.
 * schedule_out (optional, 3 ints): K-splits per tile, rule that chose them (0 force, 1 device-filling for one token tile,
 * 2 device-filling over several), CTAs launched. */
typedef struct {
  int32_t N, T, K, x_rows;
  int32_t pro, epi, force;
  const void* w;
  const void* x;
  const float* ssq_in;
  int32_t ssq_slabs;
  const void* norm_w;
  float eps;
  void* out;
  int32_t ldo;
  float* ssq_out;
  const int32_t* positions;
  const int32_t* slots;
  const void* cos_sin;
  void* kv_layer;
  int32_t q_heads, kv_heads, max_pos;
  int32_t* argmax_out;
  int32_t n_valid;
  /* epi 1 only, optional: also write normed_out [T, N] = RMSNorm(new residual) * norm_w_out (the next projection's input) */
  void* normed_out;
  const void* norm_w_out;
} b200_gemm3_args;
int b200_op_gemm3(const b200_gemm3_args* a, void* stream, int32_t* schedule_out);
int b200_op_embed(const void* table, const int32_t* ids, void* out, int32_t T, int32_t H, int32_t vocab, void* stream);
int b200_op_rmsnorm(const void* x, void* residual, const void* w, void* out, const int32_t* row_index, int32_t rows,
                    int32_t H, float eps, void* stream);
int b200_op_rope_kvwrite(void* qkv, const int32_t* positions, const int32_t* slots, const void* cos_sin,
                         void* kv_layer, int32_t T, int32_t q_heads, int32_t kv_heads, int32_t max_pos, void* stream);
int b200_op_silu_mul(const void* gate_up, void* out, int32_t T, int32_t I, void* stream);
int b200_op_argmax(const void* logits, int32_t* out, int32_t S, int32_t V, int32_t ld, void* stream);
/* work: int32[num_work][4] = {q_tok0, q_count, q_pos0, seq}; kv_layer: [block][2][kv_heads][16][128] */
int b200_op_paged_attn(const void* q, int32_t ldq, void* out, int32_t ldo, const void* kv_layer,
                       const int32_t* block_tables, int32_t max_blocks, const int32_t* work, int32_t num_work,
                       int32_t q_heads, int32_t kv_heads, float scale, int32_t decode, void* stream);
/* Decode attention with each work item's context split over `split` >= 1 CTAs per KV head (what the engine does when a step
 * has fewer decoding sequences than the device has SMs / kv_heads) and a merge of the partial softmax states. */
int b200_op_paged_attn_decode_split(const void* q, int32_t ldq, void* out, int32_t ldo, const void* kv_layer,
                                    const int32_t* block_tables, int32_t max_blocks, const int32_t* work, int32_t num_work,
                                    int32_t q_heads, int32_t kv_heads, float scale, int32_t split, void* stream);
/* Chunked-prefill attention on wgmma (csrc/attention_wgmma.cu): work items (q_tok0, q_count <= 64, q_pos0, seq), one CTA per
 * (work item, q head); q rows are read from the fused qkv buffer [q_rows, ldq] (q heads first). */
int b200_op_paged_attn_prefill_tc(const void* qkv, int32_t q_rows, int32_t ldq, void* out, int32_t ldo, const void* kv_layer,
                                  const int32_t* block_tables, int32_t max_blocks, const int32_t* work, int32_t num_work,
                                  int32_t q_heads, int32_t kv_heads, float scale, void* stream);
int b200_op_init_uniform(void* p, uint64_t n, uint32_t seed, float scale, float offset, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200ENGINE_H */
