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
  /* model architecture (Llama family; q_heads / kv_heads = 1..16 query heads per KV head, head size in head_dim below) */
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
  /* n-gram speculative decoding (vLLM's --speculative-config {"method": "ngram", ...}): each decoding sequence proposes up
   * to num_speculative_tokens drafts, the tokens that followed the longest suffix n-gram (prompt_lookup_min..max tokens)
   * at the earliest of its longest earlier occurrences in the context (vLLM's tie rule), and the step verifies them; a draft is accepted exactly when it
   * equals the token the sampler draws from its row, so the output stream is the non-speculative one.
   * num_speculative_tokens: 0 = off, else 1..k_max(G), k_max(G) = min(B200_MAX_SPEC_TOKENS, 16 / G - 1) with G =
   * q_heads / kv_heads (3 for G <= 4, 2 for G = 5, 1 for G = 6..8, 0 above).  Lookup lengths: 0 = unset (both unset: 5 and
   * 5; one unset takes the other's value); 1 <= min <= max otherwise B200_ERR_INVALID at b200_engine_create. */
  int32_t num_speculative_tokens;
  int32_t prompt_lookup_min, prompt_lookup_max;
  /* head size D: 64 or 128; 0 = 128.  q_heads * D and (q_heads + 2 * kv_heads) * D must be multiples of 128 (at D = 64:
   * an even q_heads), otherwise B200_ERR_INVALID at b200_engine_create.  The KV pool holds 2 * kv_heads * 16 * D bf16 per
   * page and layer, so D = 64 fits twice the tokens in the same memory. */
  int32_t head_dim;
  /* what the engine runs (vLLM's --runner): 0 = generate (b200_submit / b200_submit_n), 1 = pooling (b200_submit_embed: each
   * request is a prompt whose last position's final-normed hidden state, L2-normalised on request, is its embedding; no
   * lm_head is allocated or loaded, and num_speculative_tokens must be 0).  b200_config_from_hf sets 1 for a LlamaModel /
   * MistralModel checkpoint and 0 for a *ForCausalLM one; a caller may set 1 on a ForCausalLM checkpoint. */
  int32_t runner;
  /* sliding-window attention span of the checkpoint (Mistral's sliding_window), 0 = none.  The kernels attend to the whole
   * context, which inside the window is the same attention: b200_engine_create refuses max_model_len > sliding_window. */
  int32_t sliding_window;
  /* score head (vLLM's pooling runner on a *ForSequenceClassification checkpoint): 0 = none, the pooling runner serves
   * embeddings; 1..B200_MAX_SCORE_LABELS = a score weight [num_labels, hidden] ("score") applied to the final-normed last
   * position in fp32, requests submitted with b200_submit_score.  Needs runner = pooling; no lm_head is allocated. */
  int32_t num_labels;
  /* the activation a score request gets when it asks for one (vLLM's PoolerClassify / get_act_fn): 0 = by label count
   * (sigmoid at 1 label, softmax over the labels above), 1 = sigmoid, 2 = softmax, 3 = none (regression) */
  int32_t score_activation;
  /* how the serving shell tokenizes a (query, document) pair for a score head: 0 = the tokenizer's pair template (vLLM's
   * use_sep_token = true, its default), 1 = its single template over the text query + document (use_sep_token = false).
   * b200_config_from_hf sets it from config.json; the engine itself does not read it. */
  int32_t score_join_pair;
} b200_config;

enum { B200_RUNNER_GENERATE = 0, B200_RUNNER_POOLING = 1 };
/* labels a score head may have: one warp applies the activation, lane l holding logit l */
#define B200_MAX_SCORE_LABELS 32

/* drafts per step at most: a verify item's G query heads times its 1 + m positions share decode attention's 16-row tile,
 * so 3 drafts fill it at G = 4 and fewer fit at larger G (k_max(G) above) */
#define B200_MAX_SPEC_TOKENS 3

/* Sampling follows vLLM V1 (vllm/v1/sample/sampler.py, ops/topk_topp_sampler.py), made deterministic: the token is a pure
 * function of the logits row, these parameters, the seed and the index of the token in the generation (csrc/sampling.cu).
 * Zero means "off" for every field after stop_ids, so a zero-initialised struct asks for greedy decoding. */
typedef struct {
  int32_t max_tokens;
  float temperature;          /* finite, >= 0; < 1e-5 (vllm/v1/sample/sampler.py _SAMPLING_EPS) = greedy argmax */
  int32_t ignore_eos;
  int32_t num_stop_ids;
  const int32_t* stop_ids;
  float top_p;                /* in [0, 1]; 0 or 1 = off */
  int32_t top_k;              /* >= -1; 0, -1 or >= vocab = off */
  int32_t has_seed;           /* 0: the engine draws a seed for the request (not reproducible, as in vLLM and OpenAI) */
  uint64_t seed;
  /* Log-probabilities of every generated token (vLLM's raw_logprobs: log_softmax in fp32 of the bf16 logits, before
   * temperature / top-k / top-p; the sampled tokens do not change), read with b200_poll_logprobs. */
  int32_t logprobs;           /* 0 = off */
  int32_t top_logprobs;       /* 0..B200_MAX_LOGPROBS most likely tokens per position; > 0 needs logprobs */
  /* Logits edits (vLLM's logits processors and penalties, csrc/penalties.cu), applied in fp32 to the raw bf16 row in this
   * order and rounded back to bf16 before the token is chosen; logprobs still read the raw row:
   *   logit_bias: l += bias (clamped to [-100, 100]);  min_tokens: the stop ids and EOS (even with ignore_eos, as vLLM's
   *   all_stop_token_ids) are -inf while fewer than min_tokens tokens exist;  repetition_penalty r for tokens in the prompt
   *   or the output: l *= (l > 0 ? 1/r : r);  l -= frequency_penalty * count;  l -= presence_penalty * (count > 0).
   * min_p (sampled rows only) keeps the tokens with p >= min_p * p_max, after temperature and before top-k / top-p. */
  float presence_penalty;     /* [-2, 2] */
  float frequency_penalty;    /* [-2, 2] */
  float repetition_penalty;   /* >= 0; 0 = off (read as 1) */
  float min_p;                /* [0, 1] */
  int32_t min_tokens;         /* 0..max_tokens */
  int32_t num_logit_bias;     /* 0..B200_MAX_LOGIT_BIAS; ids in [0, vocab), finite values; a repeated id keeps its last */
  const int32_t* logit_bias_ids;
  const float* logit_bias_values;
  /* Prompt log-probabilities (vLLM's prompt_logprobs), read with b200_poll_prompt_logprobs: for prompt positions k = 1..n-1,
   * the raw log-probability of prompt token k from the row at position k-1, its rank and that row's top_prompt_logprobs
   * most likely tokens.  Such a request does not read the prefix cache (vLLM's skip_reading_prefix_cache). */
  int32_t prompt_logprobs;      /* 0 = off */
  int32_t top_prompt_logprobs;  /* 0..B200_MAX_LOGPROBS */
} b200_sampling;

#define B200_MAX_LOGPROBS 20     /* vLLM's default max_logprobs */
#define B200_MAX_LOGIT_BIAS 1024 /* logit_bias entries per request; also the stop ids of a request with min_tokens */

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
  /* speculative decoding (vLLM's SpecDecodingStats): verify rows proposed, draft tokens in them, drafts accepted, and
   * accepted drafts by position in the draft */
  int64_t spec_drafts, spec_draft_tokens, spec_accepted_tokens;
  int64_t spec_accepted_per_pos[B200_MAX_SPEC_TOKENS];
} b200_stats;

typedef struct {
  int32_t tokens;             /* T of the step */
  int32_t decode_seqs, prefill_seqs, sampled;
  int64_t kv_tokens_read;     /* unique K/V tokens streamed by this step: sum over sequences of their context length */
  double device_us;
  int32_t draft_tokens;       /* speculative drafts verified in the step, and those accepted */
  int32_t accepted_tokens;
} b200_step_info;

void b200_config_default(b200_config* cfg);          /* Llama-3-8B shape, vLLM-like limits */
int b200_engine_create(const b200_config* cfg, b200_engine** out);
void b200_engine_destroy(b200_engine* e);

int b200_submit(b200_engine* e, const int32_t* prompt_ids, int32_t n, const b200_sampling* sp, uint64_t* req_id);
/* Parallel sampling (vLLM's n): n requests that share one prompt, prefilled once.  req_ids[0..n) receive n request ids, each
 * usable with every per-request call below.  Member i samples with seed + i when sp has a seed (vLLM's
 * ParentRequest._get_child_sampling_params), else with a seed of its own drawn by the engine; otherwise every member uses sp.
 * When the prompt is computed, the members fork: they share its full KV pages by reference and each gets its own copy of
 * the partly filled last page.  All n run at once, so 1 <= n <= max_num_seqs; n > 1 needs temperature >= 1e-5 (vLLM's
 * "n must be 1 when using greedy sampling").  B200_ERR_INVALID otherwise.  n = 1 is b200_submit. */
int b200_submit_n(b200_engine* e, const int32_t* prompt_ids, int32_t n_prompt, const b200_sampling* sp, int32_t n,
                  uint64_t* req_ids);
/* Pooling runner only (b200_submit and b200_submit_n are refused there, and this call by a generate runner, with
 * B200_ERR_INVALID): one embedding request of 1..max_model_len prompt ids.  It is scheduled, chunked, prefix-cached and
 * preempted like any prompt, and finishes (B200_FINISH_STOP) at the step that computes its last position.  normalize != 0:
 * the vector is L2-normalised in fp32 (vLLM's embed default), else it is the fp32 of the bf16 final-normed hidden row.
 * b200_wait, b200_abort and b200_release work on it as on any request. */
int b200_submit_embed(b200_engine* e, const int32_t* ids, int32_t n, int32_t normalize, uint64_t* req_id);
/* The embedding of a b200_submit_embed request: *finished gets a B200_FINISH_* code or 0, and once it is B200_FINISH_STOP
 * out[0..dim) gets the vector (dim must be the model's hidden size, else B200_ERR_INVALID).  usage: prompt and cached
 * tokens, completion_tokens 0. */
int b200_poll_embedding(b200_engine* e, uint64_t req_id, float* out, int32_t dim, int32_t* finished, b200_usage* usage);
/* Score head only (num_labels > 0; such an engine refuses b200_submit_embed, and an embedding or generate engine refuses
 * this call, with B200_ERR_INVALID): one score request of 1..max_model_len prompt ids (a cross-encoder's tokenized pair).
 * It is scheduled, chunked and prefix-cached like an embedding request and finishes (B200_FINISH_STOP) at the step that
 * computes its last position.  use_activation != 0: the logits get the engine's score_activation, else they are the raw
 * fp32 logits. */
int b200_submit_score(b200_engine* e, const int32_t* ids, int32_t n, int32_t use_activation, uint64_t* req_id);
/* The scores of a b200_submit_score request: *finished gets a B200_FINISH_* code or 0, and once it is B200_FINISH_STOP
 * out[0..num_labels) gets them (num_labels must be the engine's, else B200_ERR_INVALID).  usage as b200_poll_embedding. */
int b200_poll_score(b200_engine* e, uint64_t req_id, float* out, int32_t num_labels, int32_t* finished, b200_usage* usage);
/* Drain newly generated token ids (at most cap).  *finished gets a B200_FINISH_* code or 0. */
int b200_poll(b200_engine* e, uint64_t req_id, int32_t* out_ids, int32_t cap, int32_t* n_out, int32_t* finished,
              b200_usage* usage);
/* b200_poll with each token's log-probability record (the request must have been submitted with logprobs, else
 * B200_ERR_INVALID).  Both calls drain the same cursor.  For token k: out_logprob[k] is its own log-probability,
 * out_top_ids / out_top_logprob[k * B200_MAX_LOGPROBS + j], j < top_logprobs, the most likely tokens in descending order
 * (lowest id on equal logits); the rest of each row is left as it was. */
int b200_poll_logprobs(b200_engine* e, uint64_t req_id, int32_t* out_ids, float* out_logprob, int32_t* out_top_ids,
                       float* out_top_logprob, int32_t cap, int32_t* n_out, int32_t* finished, b200_usage* usage);
/* The prompt log-probabilities of a request submitted with prompt_logprobs (else B200_ERR_INVALID).  *n_out = 0 until every
 * record exists (no later than the first generated token is polled), then n_prompt - 1: record k is prompt token k + 1's
 * out_logprob[k] and out_rank[k], and out_top_ids / out_top_logprob[k * B200_MAX_LOGPROBS + j], j < top_prompt_logprobs,
 * the most likely tokens at that position.  cap < n_prompt - 1 is B200_ERR_INVALID.  The token cursor does not move. */
int b200_poll_prompt_logprobs(b200_engine* e, uint64_t req_id, float* out_logprob, int32_t* out_rank, int32_t* out_top_ids,
                              float* out_top_logprob, int32_t cap, int32_t* n_out);
/* Block until the request has undrained tokens or is finished (B200_ERR_TIMEOUT otherwise). */
int b200_wait(b200_engine* e, uint64_t req_id, int64_t timeout_us);
/* Block until any of ids[0..count) has undrained tokens or is finished (B200_ERR_TIMEOUT otherwise).  count 1 is b200_wait;
 * with count > 1 the ids must be members of one b200_submit_n call (else B200_ERR_INVALID). */
int b200_wait_any(b200_engine* e, const uint64_t* ids, int32_t count, int64_t timeout_us);
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

/* Weights / buffers by name ("embed", "lm_head", "final_norm", "score", "layers.<i>.{wqkv,wo,wgu,wdown,norm1,norm2}",
 * "cos_sin").  Tests copy weights out for the CPU oracle or write their own in. */
int b200_engine_tensor_info(b200_engine* e, const char* name, uint64_t* num_bytes, void** device_ptr);
int b200_engine_tensor_read(b200_engine* e, const char* name, void* host_dst, uint64_t cap);
int b200_engine_tensor_write(b200_engine* e, const char* name, const void* host_src, uint64_t n);
/* Debug/parity: run a plain forward over `n` tokens of ONE sequence (positions 0..n-1, fresh KV pages taken from
 * the pool and returned afterwards) and copy the bf16 logits of every position to host_logits [n, vocab]. */
int b200_engine_forward_logits(b200_engine* e, const int32_t* ids, int32_t n, void* host_logits_bf16);
/* Parity hook for decode steps (manual_step mode): with keep != 0 the lm_head of every later step leaves the complete
 * bf16 logits of its sampled rows in HBM (the serving path only keeps what the argmax needs); read_logits copies the
 * first `rows` rows [rows, vocab] of the last step, in the order the step sampled them (scheduling order).  For a step
 * with a row at temperature >= 1e-5 these are the raw rows, before the sparse edits. */
int b200_engine_set_keep_logits(b200_engine* e, int32_t keep);
int b200_engine_read_logits(b200_engine* e, void* host_logits_bf16, int32_t rows);

/* ------------------------------------------------------------------ checkpoints (SURVEY.md §8f-2)
 * HF-layout Llama checkpoints: <dir>/config.json + model.safetensors[.index.json] (BF16/F16/F32 tensors).
 * The reference mounts such a directory into the backend pod (internal/modelcontroller/model_source.go:231-287). */
/* Fill the architecture fields of cfg from <dir>/config.json, head_dim included (config.json "head_dim", else hidden /
 * q_heads); rejects a head_dim other than 64 and 128, an odd q_heads at head_dim 64, a head_dim that contradicts the
 * q_proj / k_proj rows of the safetensors in <dir> (when there are any), and a GQA ratio whose kv_heads does
 * not divide q_heads or that has more than 16 query heads per KV head. */
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
  /* 1: requests with temperature >= 1e-5 are sampled (temperature / top_p / top_k / seed, see b200_sampling); 0: they get
   * a 400 and the server decodes greedily only, as before sampling existed (a zero-initialised config keeps that) */
  int32_t enable_sampling;
  /* 1: serve logprobs (chat: "logprobs": true + "top_logprobs" 0..20; completions: "logprobs" 0..20) in vLLM's response
   * format; 0: they get a 400, as before logprobs existed (a zero-initialised config keeps that) */
  int32_t enable_logprobs;
  /* 1: serve presence_penalty, frequency_penalty, repetition_penalty, min_p, min_tokens and logit_bias (see b200_sampling);
   * 0: they get a 400, as before logits edits existed (a zero-initialised config keeps that) */
  int32_t enable_logits_processors;
  /* 1: serve prompt_logprobs (both routes) and echo (completions) in vLLM's response format; 0: they get a 400, as before
   * prompt logprobs existed (a zero-initialised config keeps that) */
  int32_t enable_prompt_logprobs;
  /* k >= 2: serve "n" up to k on both routes (b200_submit_n; k at most the engines' max_num_seqs), with vLLM's checks;
   * 0 or 1: n > 1 gets a 400, as before parallel sampling existed (a zero-initialised config keeps that) */
  int32_t max_n;
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
/* vLLM's --speculative-config JSON for the n-gram method, applied to cfg: {"method": "ngram", "num_speculative_tokens": k,
 * "prompt_lookup_min": a, "prompt_lookup_max": b} (the lookup lengths optional, null = unset).  Any other method, k
 * outside 1..B200_MAX_SPEC_TOKENS, a lookup length below 1, min > max or an unknown key is B200_ERR_INVALID with a message
 * (b200_last_error) and leaves cfg unchanged.  Host-only. */
int b200_speculative_config_parse(const char* json, b200_config* cfg);
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
/* A score pair's ids, as vLLM tokenizes (query a, document b) for a cross-encoder: join 0 = HF tokenizer(text=a,
 * text_pair=b), the tokenizer.json's TemplateProcessing "pair" template (b200_config.score_join_pair 0, vLLM's
 * use_sep_token = true); join 1 = tokenizer(text=a + b), its "single" template (use_sep_token = false).  Without a template
 * in the file, or with add_special_tokens 0, the encodings are concatenated without special tokens.  Returns the full
 * count (may exceed cap), -1 on bad arguments. */
int64_t b200_tokenizer_encode_pair(const b200_tokenizer* t, const char* a, size_t alen, const char* b, size_t blen,
                                   int32_t join, int32_t add_special_tokens, int32_t* ids, size_t cap);
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
/* Host-only: the n-gram proposer of speculative decoding (vLLM's _find_longest_matched_ngram_and_propose_tokens) on
 * toks[0..n): the longest suffix of length min_n..max_n that occurred earlier, at the earliest of its longest earlier
 * occurrences (vLLM's tie rule), and up to k tokens that followed it, never past max_model_len - n nor the end of toks.
 * Writes them to out[0..k) and returns their count (0: no match); B200_ERR_INVALID on bad arguments. */
int32_t b200_ngram_propose(const int32_t* toks, int32_t n, int32_t min_n, int32_t max_n, int32_t k, int32_t max_model_len,
                           int32_t* out);
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
  /* epi 3: head size 64 or 128 (0 = 128); a 128-row slab of w holds 128 / head_dim heads, each classified on its own */
  int32_t head_dim;
} b200_gemm3_args;
int b200_op_gemm3(const b200_gemm3_args* a, void* stream, int32_t* schedule_out);
int b200_op_embed(const void* table, const int32_t* ids, void* out, int32_t T, int32_t H, int32_t vocab, void* stream);
int b200_op_rmsnorm(const void* x, void* residual, const void* w, void* out, const int32_t* row_index, int32_t rows,
                    int32_t H, float eps, void* stream);
/* Last-token pooling's tail, as a pooling engine runs it on its pooled rows: out[s] (fp32 [rows, H], device) = the final
 * RMSNorm (weight w, eps) of bf16 row row_index[s] of hidden, bit-identical in bf16 to b200_op_rmsnorm over the same rows,
 * then, when flags[s] != 0, divided by max(sqrt(sum of its squares), 1e-12) in fp32 (F.normalize).  H % 256 == 0 and
 * H <= 8192; row_index and flags are device int32 [rows]. */
int b200_op_pool_rows(const void* hidden, const void* w, const int32_t* row_index, const int32_t* flags, int32_t rows,
                      int32_t H, float eps, float* out, void* stream);
/* A score head's tail, as a score-head engine runs it on its pooled rows: out[s, 0..num_labels) (fp32 [rows, num_labels],
 * device) = the logits score_w [num_labels, H] . y, y the final RMSNorm (weight norm_w, eps) of bf16 row row_index[s] of
 * hidden, bit-identical in bf16 to b200_op_rmsnorm over the same rows; fp32 sums in a fixed order (per label each thread's
 * FMAs in visit order, then the warp sums in warp order).  flags[s] != 0 then applies `activation` (b200_config's
 * score_activation: 0 by label count, 1 sigmoid, 2 softmax, 3 none).  H % 256 == 0 and H <= 8192, 1 <= num_labels <=
 * B200_MAX_SCORE_LABELS; row_index and flags are device int32 [rows]. */
int b200_op_score_rows(const void* hidden, const void* norm_w, const void* score_w, const int32_t* row_index,
                       const int32_t* flags, int32_t rows, int32_t H, int32_t num_labels, int32_t activation, float eps,
                       float* out, void* stream);
int b200_op_rope_kvwrite(void* qkv, const int32_t* positions, const int32_t* slots, const void* cos_sin,
                         void* kv_layer, int32_t T, int32_t q_heads, int32_t kv_heads, int32_t max_pos, void* stream);
/* b200_op_rope_kvwrite at head size head_dim = 64 or 128: qkv rows of (q_heads + 2 * kv_heads) * head_dim, cos_sin rows of
 * head_dim (cos | sin), kv_layer [block][2][kv_heads][16][head_dim].  b200_op_rope_kvwrite is this at 128. */
int b200_op_rope_kvwrite_hd(void* qkv, const int32_t* positions, const int32_t* slots, const void* cos_sin,
                            void* kv_layer, int32_t T, int32_t q_heads, int32_t kv_heads, int32_t max_pos, int32_t head_dim,
                            void* stream);
int b200_op_silu_mul(const void* gate_up, void* out, int32_t T, int32_t I, void* stream);
/* out [T, I] = bf16(bf16(silu(gate)) * up) of gate_up [T, 2 I].  interleaved 0: each row is [gate | up]; 1: the engine's
 * layout, 64 gate columns, their 64 up columns, the next 64 gate columns, ... (I % 64 == 0).  b200_op_silu_mul is this
 * at 0. */
int b200_op_silu_mul_il(const void* gate_up, void* out, int32_t T, int32_t I, int32_t interleaved, void* stream);
int b200_op_argmax(const void* logits, int32_t* out, int32_t S, int32_t V, int32_t ld, void* stream);
/* One sampled row's parameters, as the engine packs them into a step: temperature < 1e-5 = greedy; top_k <= 0 or >= V and
 * top_p <= 0 or >= 1 = off; the noise is Philox4x32-10 with key (seed_lo, seed_hi) and counter (v / 4, n, 0, 0), n = the
 * index of the token being generated. */
typedef struct {
  float temperature;
  int32_t top_k;
  float top_p;
  uint32_t seed_lo, seed_hi;
  int32_t n;
  float min_p;                /* 0 = off: keep the tokens with p >= min_p * p_max (a fixed predicate on z_v - z_max) */
} b200_sample_row;
/* out[s] = the token sampled from bf16 logits row s ([S, ld], ld % 8 == 0, V <= ld) under rows[s]; rows and out are device
 * memory.  Greedy rows give the same token as b200_op_argmax. */
int b200_op_sample(const void* logits, int32_t ld, const b200_sample_row* rows, int32_t S, int32_t V, int32_t* out, void* stream);
/* Log-probabilities of bf16 logits rows [S, ld] (ld % 8 == 0, V <= ld), as the engine computes them: out_logprob[s] for
 * tokens[s]; out_top_ids / out_top_logprob [S][B200_MAX_LOGPROBS], entries j < top_n[s] (clamped to 0..20), the most
 * likely tokens in descending order, lowest id on equal logits.  Entries past a row's N are left as they were.  Every
 * pointer is device memory. */
int b200_op_logprobs(const void* logits, int32_t ld, int32_t S, int32_t V, const int32_t* tokens, const int32_t* top_n,
                     float* out_logprob, int32_t* out_top_ids, float* out_top_logprob, void* stream);
/* b200_op_logprobs plus out_rank[s] (device): the number of tokens whose logit is >= that of tokens[s] (vLLM's prompt-logprob
 * rank; equal logits share a rank).  The other outputs are bit-identical to b200_op_logprobs. */
int b200_op_logprobs_rank(const void* logits, int32_t ld, int32_t S, int32_t V, const int32_t* tokens, const int32_t* top_n,
                          float* out_logprob, int32_t* out_rank, int32_t* out_top_ids, float* out_top_logprob, void* stream);
/* The logits edits of b200_sampling on explicit inputs, with the engine's device code: rows[s] (host memory) edits bf16
 * logits row s ([S, ld], device, in place) as a request with those parameters, prompt and output tokens would see it when
 * generating its num_output-th token (min_tokens counts the output; stop_ids are its stops, EOS included by the caller).
 * edited (device [S, ld], optional): gets the edited rows, and `logits` is restored to its raw values, as the engine does
 * after the token selection. */
typedef struct {
  float presence_penalty, frequency_penalty, repetition_penalty;   /* repetition 0 = off */
  int32_t min_tokens;
  int32_t num_prompt;
  const int32_t* prompt;
  int32_t num_output;
  const int32_t* output;
  int32_t num_logit_bias;
  const int32_t* logit_bias_ids;
  const float* logit_bias_values;
  int32_t num_stop_ids;
  const int32_t* stop_ids;
} b200_penalty_row;
int b200_op_penalize(void* logits, int32_t ld, int32_t S, int32_t V, const b200_penalty_row* rows, void* edited, void* stream);
/* The engine's token-history lists on buffers the caller owns, with the engine's device code.  recs (device):
 * [n_slots][cap] records of four 32-bit words {id, count, bias (fp32), flags: 1 prompt, 2 stop, 4 bias}, each list sorted
 * by id; lens (device int32 [n_slots]): the records in use.
 * b200_op_penalty_list: builds list `slot` from row (host) as the engine does when it admits a request (the prompt and
 * output only when some penalty is on; the stop ids only while num_output < min_tokens), writes it to recs[slot][0, n)
 * and sets lens[slot] = n.  n > cap is B200_ERR_INVALID. */
int b200_op_penalty_list(const b200_penalty_row* row, int32_t V, void* recs, int32_t* lens, int32_t n_slots, int32_t cap,
                         int32_t slot, void* stream);
/* One edited row of a launch on those lists: logits row `row`, list `slot`; repetition 0 = off.  history != 0: the update
 * adds the row's sampled token to the list. */
typedef struct {
  int32_t row, slot;
  float presence_penalty, frequency_penalty, repetition_penalty;
  int32_t n_generated, min_tokens, history;
} b200_penalty_slot_row;
/* One penalize_update launch: for each of the n rows (host) with history, sampled[row] (host, [S], ids in [0, V)) joins
 * list `slot`: its count + 1, or a new record {id, 1, 0, 0} in id order while the list has fewer than cap records.  Rows
 * name rows in [0, S) and distinct slots in [0, n_slots). */
int b200_op_penalize_update(const b200_penalty_slot_row* rows, int32_t n, const int32_t* sampled, int32_t S, int32_t V,
                            void* recs, int32_t* lens, int32_t n_slots, int32_t cap, void* stream);
/* b200_op_penalize on those lists: row i of rows (host) edits bf16 logits row rows[i].row ([S, ld], device, in place;
 * distinct rows) from list rows[i].slot; every id of a named list is in [0, V).  edited as in b200_op_penalize. */
int b200_op_penalize_slots(void* logits, int32_t ld, int32_t S, int32_t V, const b200_penalty_slot_row* rows, int32_t n,
                           const void* recs, const int32_t* lens, int32_t n_slots, int32_t cap, void* edited, void* stream);
/* work: int32[num_work][4] = {q_tok0, q_count, q_pos0, seq}; kv_layer: [block][2][kv_heads][16][128]; kv_heads divides
 * q_heads and G = q_heads / kv_heads is 1..16.  Decode attention: every item has 1 <= q_count <= 16 / G consecutive query
 * positions (a speculative verify), position j masked causally at q_pos0 + j, and the item's K/V read once for all of
 * them.  decode = 0 returns B200_ERR_INVALID: chunked prefill is b200_op_paged_attn_prefill_tc[_hd]. */
int b200_op_paged_attn(const void* q, int32_t ldq, void* out, int32_t ldo, const void* kv_layer,
                       const int32_t* block_tables, int32_t max_blocks, const int32_t* work, int32_t num_work,
                       int32_t q_heads, int32_t kv_heads, float scale, int32_t decode, void* stream);
/* The attention entry points at head size head_dim = 64 or 128: q / out rows of head_dim per head, kv_layer
 * [block][2][kv_heads][16][head_dim].  Each function without _hd is its _hd sibling at 128. */
int b200_op_paged_attn_hd(const void* q, int32_t ldq, void* out, int32_t ldo, const void* kv_layer,
                          const int32_t* block_tables, int32_t max_blocks, const int32_t* work, int32_t num_work,
                          int32_t q_heads, int32_t kv_heads, float scale, int32_t decode, int32_t head_dim, void* stream);
/* Decode attention with each work item's context split over `split` >= 1 CTAs per KV head (what the engine does when a step
 * has fewer decoding sequences than the device has SMs / kv_heads) and a merge of the partial softmax states.  Work items
 * and group sizes as b200_op_paged_attn with decode = 1 (q_count up to 16 / G). */
int b200_op_paged_attn_decode_split(const void* q, int32_t ldq, void* out, int32_t ldo, const void* kv_layer,
                                    const int32_t* block_tables, int32_t max_blocks, const int32_t* work, int32_t num_work,
                                    int32_t q_heads, int32_t kv_heads, float scale, int32_t split, void* stream);
int b200_op_paged_attn_decode_split_hd(const void* q, int32_t ldq, void* out, int32_t ldo, const void* kv_layer,
                                       const int32_t* block_tables, int32_t max_blocks, const int32_t* work, int32_t num_work,
                                       int32_t q_heads, int32_t kv_heads, float scale, int32_t split, int32_t head_dim,
                                       void* stream);
/* Chunked-prefill attention on wgmma (csrc/attention_wgmma.cu): work items (q_tok0, q_count <= 64, q_pos0, seq), one CTA per
 * (work item, q head h, reading KV head h / G, G = q_heads / kv_heads in 1..16); q rows are read from the fused qkv buffer
 * [q_rows, ldq] (q heads first). */
int b200_op_paged_attn_prefill_tc(const void* qkv, int32_t q_rows, int32_t ldq, void* out, int32_t ldo, const void* kv_layer,
                                  const int32_t* block_tables, int32_t max_blocks, const int32_t* work, int32_t num_work,
                                  int32_t q_heads, int32_t kv_heads, float scale, void* stream);
int b200_op_paged_attn_prefill_tc_hd(const void* qkv, int32_t q_rows, int32_t ldq, void* out, int32_t ldo, const void* kv_layer,
                                     const int32_t* block_tables, int32_t max_blocks, const int32_t* work, int32_t num_work,
                                     int32_t q_heads, int32_t kv_heads, float scale, int32_t head_dim, void* stream);
int b200_op_init_uniform(void* p, uint64_t n, uint32_t seed, float scale, float offset, void* stream);
/* The fork's page copy: for i < n_pairs and every layer l, the block_bytes at kv + l * layer_stride_bytes + src[i] * block_bytes
 * are copied to dst[i]'s page (src / dst device int32 arrays; a src may repeat).  block_bytes and layer_stride_bytes are
 * 16-byte multiples and kv is 16-byte aligned.  Bit-exact; nothing outside the dst pages is written. */
int b200_op_kv_copy_blocks(void* kv, int32_t num_layers, int64_t layer_stride_bytes, int64_t block_bytes, const int32_t* src,
                           const int32_t* dst, int32_t n_pairs, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200ENGINE_H */
