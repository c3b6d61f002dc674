// In-process inference engine: one instance per GPU replica (SURVEY.md §8a K1-K11, §8b).
// It stands where the reference launches a backend pod (internal/modelcontroller/engine_vllm.go:82-100)
// and is reached through the C ABI in include/b200engine.h instead of the HTTP hop at
// internal/modelproxy/handler.go:158.
//
// Host side (this file): paged-KV block pool with hash-chained prefix cache, continuous-batching
// scheduler with chunked prefill under a per-step token budget (semantics of vLLM's
// v1/core/sched/scheduler.py: running first, then waiting; preempt-by-recompute on KV exhaustion;
// 16-token blocks; a prefix hit covers at most len-1 tokens), the Llama forward as a fixed kernel
// sequence on one CUDA stream, greedy or seeded temperature / top-k / top-p sampling (sampling.cu), thread-safe
// submit/poll/wait/abort.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>
#include <math.h>
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <memory>
#include <mutex>
#include <random>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/b200engine.h"
#include "errors.h"
#include "gemm.h"
#include "gemm3.h"
#include "kernels.h"
#include "hostutil.h"
#include "xxh64.h"

namespace b200 {

namespace {

constexpr int kPage = 16;
typedef __nv_bfloat16 bf16;

#define CK(call)                                                                      \
  do {                                                                                \
    cudaError_t e_ = (call);                                                          \
    if (e_ != cudaSuccess) {                                                          \
      set_error("%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_));   \
      return e_ == cudaErrorMemoryAllocation ? B200_ERR_OOM : B200_ERR_CUDA;          \
    }                                                                                 \
  } while (0)

// ------------------------------------------------------------------ KV block pool + prefix cache
class BlockPool {
 public:
  void init(int64_t n, bool caching) {
    n_ = static_cast<int>(n);
    caching_ = caching;
    ref_.assign(n_, 0);
    prev_.assign(n_, -1);
    next_.assign(n_, -1);
    uid_.assign(n_, 0);
    parent_.assign(n_, 0);
    hash_.assign(n_, 0);
    toks_.assign(static_cast<size_t>(n_) * kPage, 0);
    head_ = tail_ = -1;
    free_ = 0;
    for (int b = 0; b < n_; ++b) push_free(b);
    next_uid_ = 1;
    map_.clear();
  }
  int64_t total() const { return n_; }
  int64_t free_count() const { return free_; }

  // Take a block for writing (evicts its cached identity if it had one).
  int alloc() {
    if (head_ < 0) return -1;
    int b = head_;
    unlink(b);
    drop_identity(b);
    ref_[b] = 1;
    return b;
  }
  void ref(int b) {
    if (ref_[b] == 0) unlink(b);
    ++ref_[b];
  }
  void unref(int b) {
    if (--ref_[b] == 0) push_free(b);
  }
  // Cached full block whose parent chain uid is `parent` and content is toks[0..16): id or -1.
  int lookup(uint64_t parent, const int32_t* toks) const {
    if (!caching_) return -1;
    auto it = map_.find(key_hash(parent, toks));
    if (it == map_.end()) return -1;
    int b = it->second;
    if (parent_[b] != parent || memcmp(&toks_[static_cast<size_t>(b) * kPage], toks, kPage * 4) != 0) return -1;
    return b;
  }
  // Give block b (just filled) a cache identity; returns the chain uid children must use.
  uint64_t publish(int b, uint64_t parent, const int32_t* toks) {
    if (!caching_) return 0;
    int existing = lookup(parent, toks);
    if (existing >= 0) return uid_[existing];  // same content already cached elsewhere: chain to it
    uint64_t h = key_hash(parent, toks);
    if (map_.count(h)) return next_uid_++;  // 64-bit collision with different content: leave uncached
    drop_identity(b);
    uid_[b] = next_uid_++;
    parent_[b] = parent;
    hash_[b] = h;
    memcpy(&toks_[static_cast<size_t>(b) * kPage], toks, kPage * 4);
    map_[h] = b;
    return uid_[b];
  }
  uint64_t uid(int b) const { return uid_[b]; }
  void reset_cache() {
    for (int b = 0; b < n_; ++b) uid_[b] = 0;
    map_.clear();
  }

 private:
  static uint64_t key_hash(uint64_t parent, const int32_t* toks) {
    uint8_t buf[8 + kPage * 4];
    memcpy(buf, &parent, 8);
    memcpy(buf + 8, toks, kPage * 4);
    return xxh64(buf, sizeof(buf), 0);
  }
  void drop_identity(int b) {
    if (uid_[b]) {
      auto it = map_.find(hash_[b]);
      if (it != map_.end() && it->second == b) map_.erase(it);
      uid_[b] = 0;
    }
  }
  void push_free(int b) {
    prev_[b] = tail_;
    next_[b] = -1;
    if (tail_ >= 0) next_[tail_] = b; else head_ = b;
    tail_ = b;
    ++free_;
  }
  void unlink(int b) {
    if (prev_[b] >= 0) next_[prev_[b]] = next_[b]; else head_ = next_[b];
    if (next_[b] >= 0) prev_[next_[b]] = prev_[b]; else tail_ = prev_[b];
    prev_[b] = next_[b] = -1;
    --free_;
  }
  int n_ = 0;
  bool caching_ = true;
  std::vector<int> ref_, prev_, next_;
  std::vector<uint64_t> uid_, parent_, hash_;
  std::vector<int32_t> toks_;
  int head_ = -1, tail_ = -1;
  int64_t free_ = 0;
  uint64_t next_uid_ = 1;
  std::unordered_map<uint64_t, int> map_;
};

// ------------------------------------------------------------------ sequences
// one generated token's log-probabilities (sampling.cu logprobs_rows): its own, then its request's top N
struct LogprobRecord {
  float lp;
  float top_lp[kMaxLogprobs];
  int32_t top_ids[kMaxLogprobs];
};
// one prompt position's record: the next prompt token's log-probability and rank, then the position's top N
struct PromptLogprobRecord {
  LogprobRecord r;
  int32_t rank;
};

// the members of one b200_submit_n call: b200_wait_any sleeps here; every publish to a member bumps gen
struct WaitGroup {
  std::mutex m;
  std::condition_variable cv;
  uint64_t gen = 0;
};

struct Seq {
  uint64_t id = 0;
  std::vector<int32_t> toks;  // prompt + generated
  int n_prompt = 0;
  int n_computed = 0;    // tokens whose KV is in the cache
  int n_published = 0;   // leading full blocks with a cache identity
  uint64_t chain_uid = 0;
  std::vector<int> blocks;
  int max_tokens = 16;
  bool ignore_eos = false;
  std::vector<int32_t> stop_ids;
  // sampling (sampling.cu): temperature < 1e-5 = greedy; top_k <= 0 / top_p >= 1 = off; every request has a seed
  float temperature = 0.f, top_p = 1.f;
  int top_k = 0;
  uint64_t seed = 0;
  int top_logprobs = -1;   // -1: no logprobs; else the N of every generated token's record
  // -1: no prompt logprobs; else the N of every prompt position's record.  plp_done = prompt positions whose record a
  // launched step produces (engine thread): a prompt recomputed after a preemption does not produce them again
  int prompt_logprobs = -1;
  int plp_done = 0;
  // logits edits (penalties.cu): off when every field is at its default; pen_slot = the device record list while admitted
  float min_p = 0.f, presence = 0.f, frequency = 0.f, repetition = 1.f;
  int min_tokens = 0;
  std::vector<int32_t> bias_ids;
  std::vector<float> bias_values;
  int pen_slot = -1;
  bool pen_history() const { return presence != 0.f || frequency != 0.f || repetition != 1.f; }
  bool edits() const { return pen_history() || min_tokens > 0 || !bias_ids.empty(); }
  int n_generated = 0;
  std::atomic<int> n_cached{-1};  // prefix-hit tokens at first admission
  bool admitted = false;
  bool leaving = false;  // finished in the step being completed: swept out of the running list
  // parallel sampling (b200_submit_n), engine thread: the leader (member 0) holds the members 1..n-1 until the step that
  // completes its prompt forks them; they are registered and pollable but never queued before.  fork = the members that
  // fork in the step being launched, fork_tails = their own copies of the prompt's partly filled last page (none when the
  // prompt fills its pages).  group: b200_wait_any of the members.
  std::vector<std::shared_ptr<Seq>> children, fork;
  std::vector<int> fork_tails;
  std::shared_ptr<WaitGroup> group;
  // speculative decoding (engine thread): the drafts proposed for the step being launched (Sched::n_draft of them)
  std::vector<int32_t> draft;
  // pooling runner (b200_submit_embed, or b200_submit_score on a score head): the request's last position is pooled,
  // L2-normalised (or, on a score head, its logits activated) when `normalize`; its vector (the logits on a score head)
  // is written by the engine thread before the finish code is published, and read by API threads once finished
  bool embed = false;
  bool normalize = true;
  std::vector<float> embedding;
  void notify_group() {
    if (!group) return;
    { std::lock_guard<std::mutex> lk(group->m); ++group->gen; }
    group->cv.notify_all();
  }
  // shared with API threads: guarded by m (one lock per request, so a step's 128 wake-ups do not convoy on one mutex)
  std::mutex m;
  std::condition_variable cv;
  std::vector<int32_t> out;
  std::vector<LogprobRecord> lp_out;   // one per token of `out` when top_logprobs >= 0
  std::vector<PromptLogprobRecord> plp_out;   // one per prompt position 0..n_prompt-2 when prompt_logprobs >= 0
  size_t drained = 0;
  int finished = 0;
  uint64_t arrival_key = 0;   // xxh64 of the prompt: admission order among requests that arrive between two steps
  std::atomic<bool> abort_requested{false};
};

struct Sched {
  std::shared_ptr<Seq> s;
  int n;
  int n_plp = 0;   // prompt-logprob rows this chunk produces
  int n_draft = 0; // speculative drafts among the n tokens (after the sequence's last token); Seq::draft holds them
};
// a launched, not yet completed step
struct InFlight {
  std::vector<Sched> sched;
  double t_enter = 0, t_packed = 0, t_launched = 0;
};
// a result not yet visible to the API threads (published while the next step runs on the GPU)
struct Pub {
  std::shared_ptr<Seq> s;
  int32_t tok;
  bool has_tok;
  int code;
  int lp = -1;   // index of the token's record in Engine::pending_lp
  int plp0 = 0, n_plp = 0;   // prompt records pending_plp[plp0, plp0 + n_plp), published before the token
};

struct StepMeta {
  int T = 0, nd = 0, np = 0, S = 0, nseq = 0;
  int ndec_seq = 0, npre_seq = 0;   // sequences that decode (or verify drafts) and that prefill a chunk
  int off_ids = 0, off_pos = 0, off_slots = 0, off_rows = 0, off_dwork = 0, off_pwork = 0, off_btab = 0;
  int off_samp = -1;   // SampleRow per sampled row, packed only when one of them has temperature >= 1e-5
  int samp_words = 6;  // words per SampleRow: 7 when a sampled row has min_p, else 6 (min_p off)
  int off_pen = -1;    // PenaltyRow per row with logits edits, packed only when n_pen > 0
  int n_pen = 0;
  bool pen_update = false;   // some edited row keeps a token history
  int off_lp = -1;     // logprobs rows: n_lp row indices into [0, S), then their n_lp N values; packed only when n_lp > 0
  int n_lp = 0;
  // prompt-logprob rows: n_plp step token indices, their target ids (the next prompt token), their N; packed only when
  // n_plp > 0.  Records go to the plp buffers in this order.
  int off_plp = -1;
  int n_plp = 0;
  // parallel sampling's fork: n_fork source pages, then their n_fork destination pages (kv_copy_blocks after the forward);
  // packed only when n_fork > 0
  int off_fork = -1;
  int n_fork = 0;
  // pooled rows (pooling runner): E step token indices, then their E normalise flags; packed only when E > 0
  int off_pool = -1;
  int E = 0;
  int words = 0;
  int64_t kv_tokens = 0;
  int out_tokens = 0;  // sampled rows that produce a generated token
  int draft_tokens = 0;  // speculative drafts verified by the step
  int dmax_ctx = 0;    // longest context among the decode work items (split-KV decision)
};

struct XMaps {
  CUtensorMap m[kGemmNumBlockN];  // token tiles 32, 64, 128, 256, 512
};

// ------------------------------------------------------------------ head size
// The head size of a config (0 = 128); B200_ERR_INVALID unless it is 64 or 128 and the rows of q and of the whole qkv
// projection are whole 128-row slabs, the unit of the qkv GEMM's RoPE / KV-write epilogue.  A slab holds 128 / D heads and
// classifies each on its own, so it may hold the last k head and the first v head (an odd kv_heads at D = 64).
int head_dim_resolve(const b200_config& c, int* D) {
  const int d = c.head_dim ? c.head_dim : 128;
  if (!attn_head_dim_ok(d) || (c.q_heads * d) % 128 || ((c.q_heads + 2 * c.kv_heads) * d) % 128) {
    set_error("unsupported head_dim %d with %d query and %d KV heads (head_dim 64 or 128; q_heads * head_dim and "
              "(q_heads + 2 * kv_heads) * head_dim must be multiples of 128, so head_dim 64 needs an even q_heads)",
              d, c.q_heads, c.kv_heads);
    return B200_ERR_INVALID;
  }
  *D = d;
  return 0;
}

// ------------------------------------------------------------------ speculative decoding
// The speculative settings of a config with vLLM's defaults for the lookup lengths (config/speculative.py: both unset gives
// 5 and 5, one unset takes the other's value); B200_ERR_INVALID when out of range.  A verify item of the last token and m
// drafts fills G * (1 + m) rows of decode attention's 16-row tile, so G = q_heads / kv_heads caps the drafts at
// 16 / G - 1 (a config whose heads the kernels cannot serve is refused by Engine::init).
int spec_resolve(const b200_config& c, int* k, int* mn, int* mx) {
  *k = *mn = *mx = 0;
  if (c.num_speculative_tokens < 0 || c.num_speculative_tokens > B200_MAX_SPEC_TOKENS) {
    set_error("num_speculative_tokens must be in 0..%d, got %d", B200_MAX_SPEC_TOKENS, c.num_speculative_tokens);
    return B200_ERR_INVALID;
  }
  if (attn_group_ok(c.q_heads, c.kv_heads)) {
    const int G = c.q_heads / c.kv_heads, k_max = std::min(B200_MAX_SPEC_TOKENS, kDecodeRows / G - 1);
    if (c.num_speculative_tokens > k_max) {
      set_error("num_speculative_tokens=%d exceeds %d, the most drafts a verify step holds with %d query heads per KV head",
                c.num_speculative_tokens, k_max, G);
      return B200_ERR_INVALID;
    }
  }
  if (c.prompt_lookup_min < 0 || c.prompt_lookup_max < 0) {
    set_error("prompt_lookup_min and prompt_lookup_max must be >= 1 (0 = unset)");
    return B200_ERR_INVALID;
  }
  int a = c.prompt_lookup_min, b = c.prompt_lookup_max;
  if (!a && !b) a = b = 5;
  else if (!a) a = b;
  else if (!b) b = a;
  if (a > b) {
    set_error("prompt_lookup_min=%d must be <= prompt_lookup_max=%d", a, b);
    return B200_ERR_INVALID;
  }
  if (c.num_speculative_tokens == 0) return 0;
  *k = c.num_speculative_tokens;
  *mn = a;
  *mx = b;
  return 0;
}

}  // namespace

// vLLM's _find_longest_matched_ngram_and_propose_tokens (v1/spec_decode/ngram_proposer.py): a KMP pass over the reversed
// context finds the longest prefix of the reversal, length <= max_n, that recurs later in it, i.e. the longest suffix
// n-gram of the context that occurred before.  Among equally long matches the last one found in the reversal wins, which
// is the earliest occurrence in the context, as there.  Writes the up to k tokens that followed it (never past
// max_model_len - n, nor past the context's end) and returns their count.
int ngram_propose(const int32_t* toks, int n, int min_n, int max_n, int k, int max_model_len, int32_t* out) {
  if (n < min_n) return 0;
  k = std::min(k, max_model_len - n);
  if (k <= 0) return 0;
  auto rev = [&](int i) { return toks[n - 1 - i]; };
  max_n = std::min(max_n, n);   // no match is longer than the context
  thread_local std::vector<int> lps;
  lps.assign(std::max(max_n, 1), 0);   // lps[i] = the longest proper prefix of rev[0..i] that is also its suffix, for i < max_n
  int longest = 0, position = 0, prev = 0;
  for (int i = 1; i < n;) {
    if (rev(prev) == rev(i)) {
      ++prev;
      if (prev >= longest) {   // >=: the later position in the reversal, the earlier occurrence in the context
        longest = prev;
        position = i;
      }
      if (i < max_n) lps[i] = prev;
      if (prev == max_n) prev = lps[max_n - 1];   // never match longer than max_n
      ++i;
    } else if (prev != 0) {
      prev = lps[prev - 1];
    } else {
      ++i;
    }
  }
  if (longest < min_n) return 0;
  const int start = n - 1 - position + longest;
  k = std::min(k, n - start);
  for (int j = 0; j < k; ++j) out[j] = toks[start + j];
  return k;
}

// ------------------------------------------------------------------ engine
struct Engine {
  b200_config cfg;
  int L, H, Hq, Hkv, I, V, QKV;
  int Dh = 128;   // head size: 64 or 128 (b200_config.head_dim)
  bool pooling = false;   // b200_config.runner == B200_RUNNER_POOLING: no lm_head, pooled rows instead of sampled ones
  // score head (pooling runner, b200_config.num_labels > 0): labels L and the activation resolved from score_activation
  int num_labels = 0, score_act = 0;
  int pooled_width() const { return num_labels > 0 ? num_labels : H; }   // floats per pooled row: the vector or the logits
  // n-gram speculative decoding: drafts per decoding sequence (0 = off) and the lookup n-gram lengths
  int spec_k = 0, spec_min = 0, spec_max = 0;
  int Tcap, Scap, max_blocks_per_seq;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int sms = 0;

  // weights
  struct Layer {
    bf16 *wqkv, *wo, *wgu, *wdown, *norm1, *norm2;
    GemmPlan p_qkv, p_o, p_gu, p_down;
  };
  std::vector<Layer> layers;
  bf16 *embed = nullptr, *lm_head = nullptr, *final_norm = nullptr, *cos_sin = nullptr;
  bf16* score = nullptr;   // score head [num_labels, H] (num_labels > 0)
  GemmPlan p_lm;
  bf16* weights_blob = nullptr;
  size_t weights_bytes = 0;
  std::unordered_map<std::string, std::pair<void*, size_t>> tensors;

  // activations
  bf16 *res = nullptr, *x = nullptr, *normed = nullptr, *qkv = nullptr, *attn = nullptr, *gu = nullptr, *act = nullptr,
       *last_hidden = nullptr, *logits = nullptr;
  // step outputs read back by the host: device arrays and their pinned mirrors.  In step order, per sampled row its id;
  // per logprobs row a record of 1 + N floats (the token's lp, then the top N) and N ids; per prompt-logprob row the same
  // and the rank of its target (N = kMaxLogprobs).  for_each_readback: fn(device array, pinned mirror, bytes) for S
  // sampled rows, n_lp logprobs rows and n_plp prompt-logprob rows.
  int* sampled = nullptr;
  float *lp_dev = nullptr, *plp_f_dev = nullptr;
  int *lp_ids_dev = nullptr, *plp_ids_dev = nullptr, *plp_rank_dev = nullptr;
  int32_t *sampled_host = nullptr, *lp_ids_host = nullptr, *plp_ids_host = nullptr, *plp_rank_host = nullptr;
  float *lp_host = nullptr, *plp_f_host = nullptr;
  float *pooled = nullptr, *pooled_host = nullptr;   // per pooled row its fp32 vector [H] or logits [L] (pooling runner)
  template <class F>
  void for_each_readback(size_t S, size_t n_lp, size_t n_plp, size_t E, F fn) {
    const size_t rec = (1 + kMaxLogprobs) * sizeof(float), ids = kMaxLogprobs * sizeof(int32_t);
    fn(sampled, sampled_host, S * sizeof(int32_t));
    fn(lp_dev, lp_host, n_lp * rec);
    fn(lp_ids_dev, lp_ids_host, n_lp * ids);
    fn(plp_f_dev, plp_f_host, n_plp * rec);
    fn(plp_ids_dev, plp_ids_host, n_plp * ids);
    fn(plp_rank_dev, plp_rank_host, n_plp * sizeof(int32_t));
    fn(pooled, pooled_host, E * pooled_width() * sizeof(float));
  }
  int alloc_readbacks(int S, int n_lp, int n_plp, int E);
  // record i of the token (prompt = false) or prompt-logprob readbacks
  LogprobRecord read_record(bool prompt, int i) const {
    const float* src = (prompt ? plp_f_host : lp_host) + static_cast<size_t>(i) * (1 + kMaxLogprobs);
    LogprobRecord r;
    r.lp = src[0];
    memcpy(r.top_lp, src + 1, sizeof(r.top_lp));
    memcpy(r.top_ids, (prompt ? plp_ids_host : lp_ids_host) + static_cast<size_t>(i) * kMaxLogprobs, sizeof(r.top_ids));
    return r;
  }
  // fused epilogues (gemm_wgmma.cu): RoPE + KV write, residual add, SiLU * up and per-slab argmax ride in the projection
  // that produces their input; off (B200_FUSED_DECODE=0 / B200_FUSED_PREFILL=0) each runs as its own elementwise kernel
  float2* cand = nullptr;    // argmax candidates [token][V / 128 slab]
  bool fused_ok = false;     // steps of at most 128 tokens
  bool fused2_ok = false;    // larger steps
  float* attn_ws = nullptr;  // split-KV decode partials
  int attn_split_force = 0;  // B200_ATTN_SPLIT=<parts> (A/B knob; 1 = never split)
  static constexpr int kSplitMaxWork = 18, kSplitMaxParts = 32;
  XMaps xm_normed, xm_attn, xm_act, xm_last;
  float* gemm_ws = nullptr;
  size_t gemm_ws_bytes = 0;
  int* gemm_counters = nullptr;
  int gemm_counters_cap = 0;

  // KV
  bf16* kv = nullptr;
  size_t kv_layer_elems = 0;
  BlockPool pool;

  // logits edits (penalties.cu): max_num_seqs record lists of pen_cap records (pen_lens[slot] in use), the raw values a
  // step's edit pass overwrote [Scap][pen_cap], and the free slots
  PenaltyRec* pen_recs = nullptr;
  int* pen_lens = nullptr;
  uint16_t* pen_save = nullptr;
  int pen_cap = 0;
  std::vector<int> pen_free;
  std::vector<PenaltyRec> pen_tmp_;

  // prompt logprobs: a step's rows go through the final norm, the lm_head and logprobs_rows in groups of plp_G, each
  // group's hidden rows in prompt_hidden [plp_G, H] and its logits in prompt_logits [plp_G, V]; the records go to the
  // prompt-logprob readbacks
  int plp_G = 0;
  bf16 *prompt_hidden = nullptr, *prompt_logits = nullptr;
  XMaps xm_phid;

  // step input staging
  int step_words_cap = 0;
  int32_t* stage_host = nullptr;  // pinned, one per ring slot
  std::vector<int32_t*> stage_dev;
  std::vector<StepMeta> ring_meta;
  int ring_n = 2, ring_pos = 0;
  int64_t recorded = 0;

  // scheduler state (engine thread only)
  std::deque<std::shared_ptr<Seq>> waiting;
  std::vector<std::shared_ptr<Seq>> running;

  // shared state
  std::mutex mu_;
  std::condition_variable cv_work_;
  std::deque<std::shared_ptr<Seq>> incoming;
  std::unordered_map<uint64_t, std::shared_ptr<Seq>> requests;
  uint64_t next_id = 1;
  uint64_t seed_state = 0;   // splitmix64 stream of the seeds of requests that bring none (seeded from std::random_device)
  std::atomic<bool> stop{false};
  std::thread worker;
  b200_stats stats;
  bool fatal = false;
  bool recording = true;        // when false, steps use the scratch ring slot and the recorded ones are kept
  // per-kernel-class device timing (b200_engine_profile): events around every launch of a replayed step
  double step_timing[7] = {0, 0, 0, 0, 0, 0, 0};  // B200_STEP_TIMING accumulators (decode-only steps)
  double step_timing_last_end = 0;
  uint32_t skip_mask = 0;  // debug/timing: kernel classes (1 << B200_K_*) NOT launched by forward() (results are garbage)
  bool profiling = false;
  bool keep_logits = false;
  bool fixed_admission = false;   // b200_engine_set_fixed_admission  // parity hook: lm_head leaves complete bf16 logits (b200_engine_set_keep_logits)
  int last_S = 0;
  std::vector<std::pair<int, cudaEvent_t>> prof_events;  // (class, event) in launch order: start, stop pairs
  size_t prof_used = 0;

  ~Engine();
  int init(const b200_config& c);
  int alloc_all();
  int forward(const StepMeta& m, int32_t* dbuf, bool all_logits, bf16* logits_out);
  // decode attention; with few sequences the context of each is split over several CTAs (attention.cu attn_decode_split)
  int decode_attention(const StepMeta& m, bf16* kv_l, const int* btab, const AttnWork* dwork, float scale) {
    int split = 1;
    if (m.nd <= kSplitMaxWork) split = std::min(attn_split_force > 0 ? attn_split_force : attn_decode_split(m.nd, Hkv, m.dmax_ctx, sms), kSplitMaxParts);
    if (split > 1) ++stats.kernel_launches;   // the merge kernel
    return paged_attention(qkv, QKV, attn, Hq * Dh, kv_l, btab, max_blocks_per_seq, dwork, m.nd, Hq, Hkv, scale, stream, attn_ws, split, Dh);
  }
  int prefill_attention(bf16* kv_l, const int* btab, const AttnWork* pwork, int np, float scale) {
    return paged_attention_prefill_tc(qkv, Tcap, QKV, attn, Hq * Dh, kv_l, btab, max_blocks_per_seq, pwork, np, Hq, Hkv, scale, stream, Dh);
  }
  // one scheduler iteration = launch (schedule, pack, H2D, kernels, D2H enqueue) + complete (sync, apply) + publish
  int schedule(std::vector<Sched>& sched);
  int pack(const std::vector<Sched>& sched, StepMeta* m);
  void add_row(const Seq& q, int token_row, int gen_index);
  int step_words_bound() const;
  int launch(InFlight* f, StepMeta* m);
  int complete(InFlight& f, const StepMeta& m, b200_step_info* info);
  void publish();
  int step(b200_step_info* info);
  int run(int max_steps, int64_t idle_timeout_us, b200_step_info* infos, int* n_done);
  void fail_all();
  void loop();
  std::vector<Pub> pending_pub;
  std::vector<LogprobRecord> pending_lp;   // records of pending_pub entries (Pub::lp)
  std::vector<PromptLogprobRecord> pending_plp;   // prompt records of pending_pub entries (Pub::plp0, n_plp)
  InFlight inflight_;
  std::vector<AttnWork> dwork_, pwork_;  // packing scratch (kept across steps: no per-step allocation)
  std::vector<int> rows_;
  std::vector<int> plp_tok_, plp_tgt_, plp_n_;   // prompt-logprob rows: step token index, target id, N
  std::vector<SampleRow> samp_;          // parameters of the rows in rows_ order
  std::vector<int> lp_rows_, lp_n_;      // logprobs rows (indices into rows_) and their N
  std::vector<PenaltyRow> pen_;          // rows with logits edits
  std::vector<int> fork_src_, fork_dst_; // the step's fork page copies
  std::vector<int> pool_rows_, pool_flags_;   // pooled rows: step token index, normalise flag
  std::vector<int32_t> draft_tmp_;
  void add_drafts(std::vector<Sched>& sched, int* budget);
  int admit_edits(Seq& s);
  bool ensure_blocks(Seq& s, int upto, int tails = 0);
  int plan_fork(Seq& s, int n);
  void finish_group(std::shared_ptr<Seq> s, int code);
  void release_blocks(Seq& s);
  void preempt(std::shared_ptr<Seq> s);
  void finish(std::shared_ptr<Seq> s, int code);
  void admit_prefix(Seq& s);
  const CUtensorMap& xmap(const XMaps& xm, int bn) const { return xm.m[gemm_block_n_index(bn)]; }
  // one projection launch: out[t, n] = x[t, :] . W[n, :] with the epilogue `epi`; the caller fills the epilogue's fields of p
  Gemm3Params proj(const GemmPlan& pl, int epi) const {
    Gemm3Params p;
    memset(&p, 0, sizeof(p));
    p.tm_w = pl.tm_w;
    p.N = pl.N; p.K = pl.K;
    p.pro = GEMM3_PRO_NONE; p.epi = epi;
    p.eps = cfg.rms_eps;
    p.n_valid = pl.N;
    p.ws = gemm_ws; p.ws_bytes = gemm_ws_bytes;
    p.counters = gemm_counters; p.counters_cap = gemm_counters_cap;
    return p;
  }
  int launch_proj(Gemm3Params p, const XMaps& xm, int T) {
    Gemm3Schedule sch;
    if (int rc = gemm3_schedule(p.N, p.K, T, 0, &sch)) return rc;
    p.T = T;
    p.tm_x = xmap(xm, sch.block_n);
    ++stats.kernel_launches;
    return gemm3_launch(p, sch, stream);
  }
};

Engine::~Engine() {
  stop = true;
  cv_work_.notify_all();
  if (worker.joinable()) worker.join();
  publish();
  {
    // nobody will step this engine again: wake every thread still blocked in b200_wait on an unfinished request
    std::vector<std::shared_ptr<Seq>> open;
    {
      std::lock_guard<std::mutex> lk(mu_);
      for (auto& kv : requests) open.push_back(kv.second);
      requests.clear();
    }
    for (auto& s : open) {
      {
        std::lock_guard<std::mutex> lk(s->m);
        if (!s->finished) s->finished = B200_FINISH_ABORTED;
      }
      s->cv.notify_all();
      s->notify_group();
    }
  }
  if (step_timing[0] > 0) {
    const double n = step_timing[0], us = 1e6 / n;
    fprintf(stderr,
            "[b200engine] decode-only steps %.0f: schedule+pack %.1f us, launch %.1f us, wait %.1f us, apply %.1f us, "
            "device %.1f us, between calls %.1f us\n",
            n, step_timing[1] * us, step_timing[2] * us, step_timing[3] * us, step_timing[4] * us, step_timing[5] * us,
            step_timing[6] * us);
  }
  cudaSetDevice(cfg.device);
  if (stream) cudaStreamSynchronize(stream);
  void* frees[] = {weights_blob, res, x, normed, qkv, attn, gu, act, last_hidden, logits, gemm_ws, gemm_counters, kv,
                   cand, attn_ws, pen_recs, pen_lens, pen_save, prompt_hidden, prompt_logits};
  for (void* p : frees)
    if (p) cudaFree(p);
  for (auto p : stage_dev)
    if (p) cudaFree(p);
  if (stage_host) cudaFreeHost(stage_host);
  for_each_readback(0, 0, 0, 0, [](auto* dev, auto* host, size_t) {
    if (dev) cudaFree(dev);
    if (host) cudaFreeHost(host);
  });
  if (ev0) cudaEventDestroy(ev0);
  if (ev1) cudaEventDestroy(ev1);
  if (stream) cudaStreamDestroy(stream);
}

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

static uint64_t splitmix64(uint64_t* state) {
  uint64_t z = (*state += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// the readbacks of up to S sampled, n_lp logprobs, n_plp prompt-logprob and E pooled rows that are not allocated yet
int Engine::alloc_readbacks(int S, int n_lp, int n_plp, int E) {
  cudaError_t ce = cudaSuccess;
  for_each_readback(S, n_lp, n_plp, E, [&](auto*& dev, auto*& host, size_t bytes) {
    if (bytes == 0 || dev || ce != cudaSuccess) return;
    ce = cudaMalloc(&dev, bytes);
    if (ce == cudaSuccess) ce = cudaMallocHost(&host, bytes);
  });
  CK(ce);
  return 0;
}

int Engine::alloc_all() {
  // ---- weights: one blob, 1 KiB-aligned tensors
  struct Item {
    std::string name;
    size_t elems;
    bf16** dst;
    float scale, offset;
  };
  std::vector<Item> items;
  layers.resize(L);
  const float s_h = 1.0f / sqrtf(static_cast<float>(H)), s_i = 1.0f / sqrtf(static_cast<float>(I)),
              s_a = 1.0f / sqrtf(static_cast<float>(Hq * Dh));
  items.push_back({"embed", static_cast<size_t>(V) * H, &embed, 1.0f, 0.f});
  for (int l = 0; l < L; ++l) {
    std::string p = "layers." + std::to_string(l) + ".";
    items.push_back({p + "wqkv", static_cast<size_t>(QKV) * H, &layers[l].wqkv, s_h, 0.f});
    items.push_back({p + "wo", static_cast<size_t>(H) * Hq * Dh, &layers[l].wo, s_a, 0.f});
    items.push_back({p + "wgu", static_cast<size_t>(2) * I * H, &layers[l].wgu, s_h, 0.f});
    items.push_back({p + "wdown", static_cast<size_t>(H) * I, &layers[l].wdown, s_i, 0.f});
    items.push_back({p + "norm1", static_cast<size_t>(H), &layers[l].norm1, 0.1f, 1.0f});
    items.push_back({p + "norm2", static_cast<size_t>(H), &layers[l].norm2, 0.1f, 1.0f});
  }
  items.push_back({"final_norm", static_cast<size_t>(H), &final_norm, 0.1f, 1.0f});
  if (num_labels > 0) items.push_back({"score", static_cast<size_t>(num_labels) * H, &score, s_h, 0.f});
  if (!pooling)   // a pooling engine never runs the lm_head
    items.push_back({"lm_head", static_cast<size_t>(V) * H, &lm_head, s_h * (cfg.init_scale > 0 ? cfg.init_scale : 4.0f), 0.f});
  size_t total = 0;
  std::vector<size_t> offs;
  for (auto& it : items) {
    offs.push_back(total);
    total += align_up(it.elems * 2, 1024);
  }
  const size_t cs_elems = static_cast<size_t>(cfg.max_model_len) * Dh;
  const size_t cs_off = total;
  total += align_up(cs_elems * 2, 1024);
  weights_bytes = total;
  CK(cudaMalloc(&weights_blob, total));
  // gate_up rows live interleaved in 64-row blocks (gate block, matching up block, ...): the decode GEMM's SiLU epilogue
  // needs a gate row and its up row in the same 128-row slab.  The named tensor keeps its logical [gate | up] meaning at
  // the ABI (tensor_read / tensor_write / the checkpoint loader permute), and the seeded init is generated in logical order.
  bf16* gu_tmp = nullptr;
  CK(cudaMalloc(&gu_tmp, static_cast<size_t>(2) * I * H * 2));
  for (size_t i = 0; i < items.size(); ++i) {
    bf16* p = reinterpret_cast<bf16*>(reinterpret_cast<uint8_t*>(weights_blob) + offs[i]);
    *items[i].dst = p;
    tensors[items[i].name] = {p, items[i].elems * 2};
    uint32_t seed = static_cast<uint32_t>(xxh64(items[i].name.data(), items[i].name.size(), cfg.seed));
    const bool is_gu = items[i].name.size() > 4 && items[i].name.compare(items[i].name.size() - 4, 4, ".wgu") == 0;
    if (init_uniform(is_gu ? gu_tmp : p, items[i].elems, seed, items[i].scale, items[i].offset, stream)) return cuda_fail("init_uniform", -2);
    if (is_gu && permute_gate_up(p, gu_tmp, I, H, 1, stream)) return cuda_fail("permute_gate_up", -2);
  }
  CK(cudaStreamSynchronize(stream));
  CK(cudaFree(gu_tmp));
  cos_sin = reinterpret_cast<bf16*>(reinterpret_cast<uint8_t*>(weights_blob) + cs_off);
  tensors["cos_sin"] = {cos_sin, cs_elems * 2};
  {
    // vllm rotary_embedding/base.py:70-92: inv_freq = base^(-2i/d); cache = cos(t*f) | sin(t*f), cast to bf16
    std::vector<bf16> h(cs_elems);
    std::vector<float> inv(Dh / 2);
    for (int i = 0; i < Dh / 2; ++i)
      inv[i] = 1.0f / powf(cfg.rope_theta, static_cast<float>(2 * i) / static_cast<float>(Dh));
    float pos_div = 1.0f;
    if (cfg.rope_scaling_type == 1) {
      // LinearScalingRotaryEmbedding (rotary_embedding/linear_scaling_rope.py): t / factor
      pos_div = cfg.rope_factor;
    } else if (cfg.rope_scaling_type == 2) {
      // Llama3RotaryEmbedding._compute_inv_freq (rotary_embedding/llama3_rope.py:37-54)
      const float orig = static_cast<float>(cfg.rope_original_max_pos);
      const float low_wl = orig / cfg.rope_low_freq_factor, high_wl = orig / cfg.rope_high_freq_factor;
      for (int i = 0; i < Dh / 2; ++i) {
        const float wl = 2.0f * static_cast<float>(M_PI) / inv[i];
        if (wl < high_wl) continue;
        if (wl > low_wl || cfg.rope_low_freq_factor == cfg.rope_high_freq_factor) { inv[i] = inv[i] / cfg.rope_factor; continue; }
        const float smooth = (orig / wl - cfg.rope_low_freq_factor) / (cfg.rope_high_freq_factor - cfg.rope_low_freq_factor);
        inv[i] = (1.0f - smooth) * inv[i] / cfg.rope_factor + smooth * inv[i];
      }
    }
    for (int t = 0; t < cfg.max_model_len; ++t)
      for (int i = 0; i < Dh / 2; ++i) {
        const float f = static_cast<float>(t) / pos_div * inv[i];
        h[static_cast<size_t>(t) * Dh + i] = __float2bfloat16_rn(cosf(f));
        h[static_cast<size_t>(t) * Dh + Dh / 2 + i] = __float2bfloat16_rn(sinf(f));
      }
    CK(cudaMemcpyAsync(cos_sin, h.data(), cs_elems * 2, cudaMemcpyHostToDevice, stream));
    CK(cudaStreamSynchronize(stream));
  }

  // ---- activations
  CK(cudaMalloc(&res, static_cast<size_t>(Tcap) * H * 2));
  CK(cudaMalloc(&x, static_cast<size_t>(Tcap) * H * 2));
  CK(cudaMalloc(&normed, static_cast<size_t>(Tcap) * H * 2));
  CK(cudaMalloc(&qkv, static_cast<size_t>(Tcap) * QKV * 2));
  CK(cudaMalloc(&attn, static_cast<size_t>(Tcap) * Hq * Dh * 2));
  CK(cudaMalloc(&gu, static_cast<size_t>(Tcap) * 2 * I * 2));
  CK(cudaMalloc(&act, static_cast<size_t>(Tcap) * I * 2));
  CK(cudaMalloc(&last_hidden, static_cast<size_t>(Scap) * H * 2));
  CK(cudaMalloc(&logits, static_cast<size_t>(Scap) * V * 2));
  CK(cudaMemset(normed, 0, static_cast<size_t>(Tcap) * H * 2));
  CK(cudaMemset(attn, 0, static_cast<size_t>(Tcap) * Hq * Dh * 2));
  CK(cudaMemset(act, 0, static_cast<size_t>(Tcap) * I * 2));
  CK(cudaMemset(last_hidden, 0, static_cast<size_t>(Scap) * H * 2));
  // the prompt-logprob records come after the KV pool; a pooling step pools at most one row per sequence
  if (int rc = alloc_readbacks(Scap, Scap, 0, pooling ? cfg.max_num_seqs : 0)) return rc;
  CK(cudaMalloc(&cand, static_cast<size_t>(std::min(Scap, 128)) * ((V + 127) / 128) * sizeof(float2)));
  // outputs of the last step, readable by name (b200_engine_tensor_read): sampled ids int32 [S]; the lm_head's per-slab
  // {best logit, index} candidates float2 [S][ceil(V / 128)] when the step sampled through them, else bf16 logits [S][V]
  tensors["step.sampled"] = {sampled, static_cast<size_t>(Scap) * 4};
  tensors["step.argmax_candidates"] = {cand, static_cast<size_t>(std::min(Scap, 128)) * ((V + 127) / 128) * sizeof(float2)};
  tensors["step.logits"] = {logits, static_cast<size_t>(Scap) * V * 2};
  CK(cudaMalloc(&attn_ws, attn_split_ws_bytes(kSplitMaxWork, Hq, kSplitMaxParts, 1 + spec_k, Dh)));
  { const char* e = getenv("B200_ATTN_SPLIT"); attn_split_force = e ? atoi(e) : 0; }
  // split-K workspace and arrival counters: the largest need of any projection at any step size up to Tcap
  {
    const int shapes[5][2] = {{QKV, H}, {H, Hq * Dh}, {2 * I, H}, {H, I}, {V, H}};
    size_t ws_bytes = 1 << 20;
    int counters = 1024;
    const int t_max = std::max(Tcap, Scap);
    for (auto& sh : shapes)
      for (int T = 1;; T = std::min(T < 64 ? 64 : T + 64, t_max)) {   // every token-tile count up to t_max, t_max itself last
        Gemm3Schedule sch;
        if (gemm3_schedule(sh[0], sh[1], T, 0, &sch)) return cuda_fail("gemm3_schedule", -1);
        ws_bytes = std::max(ws_bytes, gemm3_ws_bytes(sh[0], sch, T));
        counters = std::max(counters, gemm3_counters_needed(sh[0], sch, T));
        if (T == t_max) break;
      }
    gemm_ws_bytes = ws_bytes;
    gemm_counters_cap = counters;
  }
  CK(cudaMalloc(&gemm_ws, gemm_ws_bytes));
  CK(cudaMalloc(&gemm_counters, static_cast<size_t>(gemm_counters_cap) * 4));
  CK(cudaMemset(gemm_counters, 0, static_cast<size_t>(gemm_counters_cap) * 4));

  // ---- GEMM plans + activation tensor maps (encoded once; kernels mask rows >= T)
  auto plan = [&](GemmPlan* p, const void* W, int N, int K) {
    return gemm_plan_init(p, W, N, K, K, gemm_ws, gemm_ws_bytes, gemm_counters, gemm_counters_cap);
  };
  for (int l = 0; l < L; ++l) {
    if (plan(&layers[l].p_qkv, layers[l].wqkv, QKV, H) || plan(&layers[l].p_o, layers[l].wo, H, Hq * Dh) ||
        plan(&layers[l].p_gu, layers[l].wgu, 2 * I, H) || plan(&layers[l].p_down, layers[l].wdown, H, I))
      return cuda_fail("gemm_plan_init", -2);
  }
  if (!pooling && plan(&p_lm, lm_head, V, H)) return cuda_fail("gemm_plan_init(lm_head)", -2);
  const int bns[kGemmNumBlockN] = {64, 128, 256};
  for (int i = 0; i < kGemmNumBlockN; ++i) {
    if (gemm_make_x_map(&xm_normed.m[i], normed, Tcap, H, H, bns[i]) ||
        gemm_make_x_map(&xm_attn.m[i], attn, Tcap, Hq * Dh, Hq * Dh, bns[i]) ||
        gemm_make_x_map(&xm_act.m[i], act, Tcap, I, I, bns[i]) ||
        gemm_make_x_map(&xm_last.m[i], last_hidden, Scap, H, H, bns[i]))
      return cuda_fail("gemm_make_x_map", -2);
  }
  // A/B knobs: 0 keeps those steps on plain GEMM outputs + the elementwise kernels.  The fused epilogues need whole
  // 128-row slabs (one head per slab for RoPE, gate/up pairs for SiLU).
  {
    const char* fd = getenv("B200_FUSED_DECODE");
    const char* fp = getenv("B200_FUSED_PREFILL");
    const bool shapes_ok = QKV % 128 == 0 && (2 * I) % 128 == 0;
    fused_ok = shapes_ok && !(fd && atoi(fd) == 0);
    fused2_ok = shapes_ok && !(fp && atoi(fp) == 0);
  }

  // ---- KV pool
  const size_t block_bytes_layer = static_cast<size_t>(2) * Hkv * kPage * Dh * 2;
  int64_t nblocks = cfg.num_kv_blocks;
  if (nblocks <= 0) {
    size_t fr = 0, tot = 0;
    CK(cudaMemGetInfo(&fr, &tot));
    const float frac = cfg.kv_fraction > 0 ? cfg.kv_fraction : 0.85f;
    nblocks = static_cast<int64_t>(static_cast<double>(fr) * frac / (static_cast<double>(block_bytes_layer) * L));
  }
  // vLLM refuses to start when the cache cannot hold one max_model_len sequence (v1/core/kv_cache_utils.py
  // check_enough_kv_cache_memory): a request that needs more pages than the pool could never be admitted
  const int64_t need_blocks = (static_cast<int64_t>(cfg.max_model_len) + kPage - 1) / kPage;
  if (nblocks < 4 || nblocks < need_blocks) {
    set_error("KV pool too small: %lld blocks, one max_model_len=%d sequence needs %lld (lower max_model_len or raise num_kv_blocks / kv_fraction)",
              static_cast<long long>(nblocks), cfg.max_model_len, static_cast<long long>(need_blocks));
    return B200_ERR_OOM;
  }
  if (nblocks > (1 << 27)) nblocks = 1 << 27;
  kv_layer_elems = static_cast<size_t>(nblocks) * 2 * Hkv * kPage * Dh;
  CK(cudaMalloc(&kv, kv_layer_elems * 2 * L));
  // the attention kernel gathers whole pages and masks the rows past a sequence's end: those rows must be finite
  CK(cudaMemsetAsync(kv, 0, kv_layer_elems * 2 * L, stream));
  pool.init(nblocks, cfg.enable_prefix_caching != 0);

  // ---- logits-edit record lists, allocated after the KV pool is sized (they do not change num_kv_blocks).  A list holds
  // one record per distinct id: at most max_model_len history ids, B200_MAX_LOGIT_BIAS bias ids, as many stop ids and EOS.
  pen_cap = cfg.max_model_len + 2 * B200_MAX_LOGIT_BIAS + 1;
  // (one list per running sequence; the saved entries are per edited row, and a speculating sequence edits 1 + k rows)
  CK(cudaMalloc(&pen_recs, static_cast<size_t>(cfg.max_num_seqs) * pen_cap * sizeof(PenaltyRec)));
  CK(cudaMalloc(&pen_lens, static_cast<size_t>(cfg.max_num_seqs) * sizeof(int)));
  CK(cudaMalloc(&pen_save, static_cast<size_t>(Scap) * pen_cap * sizeof(uint16_t)));
  CK(cudaMemsetAsync(pen_lens, 0, static_cast<size_t>(cfg.max_num_seqs) * sizeof(int), stream));
  for (int i = cfg.max_num_seqs - 1; i >= 0; --i) pen_free.push_back(i);

  // ---- prompt-logprob scratch and records, likewise after the KV pool.  A group of 512 rows reads the lm_head once for
  // 512 rows (compute-bound) and keeps the scratch at 512 * V bf16 (131 MB at Llama-3's vocabulary).
  plp_G = std::min(Tcap, 512);
  CK(cudaMalloc(&prompt_hidden, static_cast<size_t>(plp_G) * H * 2));
  CK(cudaMalloc(&prompt_logits, static_cast<size_t>(plp_G) * V * 2));
  CK(cudaMemset(prompt_hidden, 0, static_cast<size_t>(plp_G) * H * 2));
  if (int rc = alloc_readbacks(Scap, Scap, Tcap, pooling ? cfg.max_num_seqs : 0)) return rc;
  // bf16 logits [plp_G, V] of the last group of prompt-logprob rows of the last step
  tensors["step.prompt_logits"] = {prompt_logits, static_cast<size_t>(plp_G) * V * 2};
  for (int i = 0; i < kGemmNumBlockN; ++i)
    if (gemm_make_x_map(&xm_phid.m[i], prompt_hidden, plp_G, H, H, bns[i])) return cuda_fail("gemm_make_x_map", -2);

  // ---- step input ring
  max_blocks_per_seq = (cfg.max_model_len + kPage - 1) / kPage;
  step_words_cap = step_words_bound();
  ring_n = std::max(1, cfg.record_steps) + 1;  // last slot = scratch for unrecorded steps
  CK(cudaMallocHost(&stage_host, static_cast<size_t>(step_words_cap) * 4));
  stage_dev.assign(ring_n, nullptr);
  ring_meta.assign(ring_n, StepMeta());
  for (int i = 0; i < ring_n; ++i) CK(cudaMalloc(&stage_dev[i], static_cast<size_t>(step_words_cap) * 4));
  CK(cudaStreamSynchronize(stream));
  return 0;
}

int Engine::init(const b200_config& c) {
  cfg = c;
  L = c.num_layers; H = c.hidden; Hq = c.q_heads; Hkv = c.kv_heads; I = c.intermediate; V = c.vocab;
  if (int rc = head_dim_resolve(c, &Dh)) return rc;
  pooling = c.runner == B200_RUNNER_POOLING;
  num_labels = c.num_labels;
  // vLLM's PoolerClassify default: sigmoid for one label, softmax for more
  score_act = c.score_activation ? c.score_activation : (num_labels == 1 ? kScoreSigmoid : kScoreSoftmax);
  QKV = (Hq + 2 * Hkv) * Dh;
  // the constraints of every kernel the forward launches, checked here so that a bad shape fails at create time with a
  // message instead of poisoning the replica at its first step: RMSNorm rows are 256-element multiples up to 8192,
  // argmax and the partial readers use 8-element vectors, GEMM K dims are 64-element TMA boxes
  if (L < 1 || H % 256 || H > 8192 || !attn_group_ok(Hq, Hkv) || I % 64 || V < 8 || V % 8 || c.max_model_len < 16 ||
      c.max_num_seqs < 1 || c.max_batched_tokens < 16) {
    set_error("unsupported model/config (need kv_heads to divide q_heads with 1..16 query heads per KV head, hidden %% 256 == 0 "
              "and <= 8192, intermediate %% 64 == 0, vocab %% 8 == 0, max_model_len >= 16)");
    return B200_ERR_INVALID;
  }
  if (c.rope_scaling_type < 0 || c.rope_scaling_type > 2 ||
      (c.rope_scaling_type != 0 && !(c.rope_factor > 0.f)) ||
      (c.rope_scaling_type == 2 && (!(c.rope_low_freq_factor > 0.f) || !(c.rope_high_freq_factor > 0.f) || c.rope_original_max_pos < 1))) {
    set_error("bad rope scaling parameters (type %d)", c.rope_scaling_type);
    return B200_ERR_INVALID;
  }
  Tcap = (c.max_batched_tokens + 15) / 16 * 16;
  if (int rc = spec_resolve(c, &spec_k, &spec_min, &spec_max)) return rc;
  // sampled rows: one per sequence, and one per draft position of a speculating sequence
  Scap = c.max_num_seqs * (1 + spec_k);
  memset(&stats, 0, sizeof(stats));
  {
    std::random_device rd;
    seed_state = (static_cast<uint64_t>(rd()) << 32) ^ rd();
  }
  CK(cudaSetDevice(c.device));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c.device));
  CK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  CK(cudaEventCreate(&ev0));
  CK(cudaEventCreate(&ev1));
  if (int rc = alloc_all()) return rc;
  stats.kv_blocks_total = pool.total();
  stats.kv_blocks_free = pool.free_count();
  if (!c.manual_step) worker = std::thread([this] { loop(); });
  return 0;
}

// ------------------------------------------------------------------ forward pass (fixed kernel sequence)
// Per layer: RMSNorm -> qkv (+ RoPE / KV write) -> attention -> o_proj (+ residual add) -> RMSNorm -> gate_up (+ SiLU * up)
// -> down_proj (+ residual add).  With fused epilogues the elementwise op after a projection runs inside it on the rounded
// bf16 output; without, the same arithmetic runs as a separate kernel on the bf16 tensor (same rounding points, so both forms
// give the same bits).
int Engine::forward(const StepMeta& m, int32_t* dbuf, bool all_logits, bf16* logits_out) {
  const int T = m.T;
  const int* ids = dbuf + m.off_ids;
  const int* pos = dbuf + m.off_pos;
  const int* slots = dbuf + m.off_slots;
  const int* rows = dbuf + m.off_rows;
  const AttnWork* dwork = reinterpret_cast<const AttnWork*>(dbuf + m.off_dwork);
  const AttnWork* pwork = reinterpret_cast<const AttnWork*>(dbuf + m.off_pwork);
  const int* btab = dbuf + m.off_btab;
  const float scale = 1.0f / sqrtf(static_cast<float>(Dh));
  int rc = 0;
  auto launched = [&](int n) { stats.kernel_launches += n; };
  // profiling: P(cls) before a launch group, Q() after it
  auto P = [&](int cls) {
    if (!profiling) return;
    if (prof_used + 2 > prof_events.size()) {
      for (int i = 0; i < 2; ++i) { cudaEvent_t e; cudaEventCreate(&e); prof_events.push_back({cls, e}); }
    }
    prof_events[prof_used].first = cls;
    cudaEventRecord(prof_events[prof_used].second, stream);
  };
  auto Q = [&]() {
    if (!profiling) return;
    cudaEventRecord(prof_events[prof_used + 1].second, stream);
    prof_used += 2;
  };
  auto on = [&](int cls) { return !(skip_mask & (1u << cls)); };
  const bool fused = !all_logits && (T <= 128 ? fused_ok : fused2_ok);
  P(B200_K_EMBED); if (on(B200_K_EMBED)) rc |= embed_gather(embed, ids, res, T, H, V, stream); Q(); launched(1);
  bool x_pending = false;   // `x` holds a projection output that the next RMSNorm still has to add to the residual
  auto norm = [&](const bf16* w, bf16* dst, const int* row_index, int n) {
    if (!x_pending) rc |= rmsnorm(res, nullptr, w, dst, row_index, n, H, cfg.rms_eps, stream);
    else rc |= rmsnorm(x, res, w, dst, row_index, n, H, cfg.rms_eps, stream);
    launched(1);
  };
  // o_proj / down_proj: residual add in the epilogue, or a bf16 `x` the next RMSNorm adds
  auto resadd_proj = [&](const GemmPlan& pl, const XMaps& xm) {
    if (fused) {
      Gemm3Params p = proj(pl, GEMM3_EPI_RESADD);
      p.out = res; p.ldo = H;
      rc |= launch_proj(p, xm, T);
      x_pending = false;
    } else {
      Gemm3Params p = proj(pl, GEMM3_EPI_PLAIN);
      p.out = x; p.ldo = H;
      rc |= launch_proj(p, xm, T);
      x_pending = true;
    }
  };
  for (int l = 0; l < L && !rc; ++l) {
    Layer& ly = layers[l];
    bf16* kv_l = kv + static_cast<size_t>(l) * kv_layer_elems;
    P(B200_K_NORM); if (on(B200_K_NORM)) norm(ly.norm1, normed, nullptr, T); Q();
    P(B200_K_GEMM_QKV);
    if (on(B200_K_GEMM_QKV)) {
      Gemm3Params p = proj(ly.p_qkv, fused ? GEMM3_EPI_ROPE_KV : GEMM3_EPI_PLAIN);
      p.out = qkv; p.ldo = QKV;
      p.positions = pos; p.slots = slots; p.cos_sin = cos_sin; p.kv_layer = kv_l; p.Hq = Hq; p.Hkv = Hkv; p.max_pos = cfg.max_model_len; p.head_dim = Dh;
      rc |= launch_proj(p, xm_normed, T);
    }
    Q();
    if (!fused) { P(B200_K_ROPE); if (on(B200_K_ROPE)) rc |= rope_kv_write(qkv, pos, slots, cos_sin, kv_l, T, Hq, Hkv, cfg.max_model_len, stream, Dh); Q(); launched(1); }
    if (m.nd) { P(B200_K_ATTN_DECODE); if (on(B200_K_ATTN_DECODE)) rc |= decode_attention(m, kv_l, btab, dwork, scale); Q(); launched(1); }
    if (m.np) { P(B200_K_ATTN_PREFILL); if (on(B200_K_ATTN_PREFILL)) rc |= prefill_attention(kv_l, btab, pwork, m.np, scale); Q(); launched(1); }
    P(B200_K_GEMM_O); if (on(B200_K_GEMM_O)) resadd_proj(ly.p_o, xm_attn); Q();
    P(B200_K_NORM); if (on(B200_K_NORM)) norm(ly.norm2, normed, nullptr, T); Q();
    P(B200_K_GEMM_GU);
    if (on(B200_K_GEMM_GU)) {
      Gemm3Params p = proj(ly.p_gu, fused ? GEMM3_EPI_SILU : GEMM3_EPI_PLAIN);
      p.out = fused ? act : gu; p.ldo = fused ? I : 2 * I;
      rc |= launch_proj(p, xm_normed, T);
    }
    Q();
    if (!fused) { P(B200_K_SILU); if (on(B200_K_SILU)) rc |= silu_mul(gu, act, T, I, stream, 1); Q(); launched(1); }
    P(B200_K_GEMM_DOWN); if (on(B200_K_GEMM_DOWN)) resadd_proj(ly.p_down, xm_act); Q();
  }
  if (rc) return cuda_fail("forward", -2);
  if (all_logits) {
    norm(final_norm, normed, nullptr, T);
    Gemm3Params p = proj(p_lm, GEMM3_EPI_PLAIN);
    p.out = logits_out; p.ldo = V;
    rc |= launch_proj(p, xm_normed, T);
  } else if (m.S > 0) {
    P(B200_K_NORM); norm(final_norm, last_hidden, rows, m.S); Q();
    // argmax candidates per 128-row slab in the lm_head epilogue (the candidate buffer holds 128 rows), or bf16 logits.
    // A step with a sampled row (temperature >= 1e-5) writes the logits and selects every row's token in one sample_rows
    // launch, greedy rows included.  A step with a logprobs row writes the logits too, for logprobs_rows, and so does a
    // step with logits edits: they are applied before the token selection and undone after it.
    const bool samp = m.off_samp >= 0;
    const bool cand_ok = !samp && m.n_lp == 0 && m.n_pen == 0 && fused && !keep_logits && m.S <= 128;
    const PenaltyRow* pen_rows = m.n_pen > 0 ? reinterpret_cast<const PenaltyRow*>(dbuf + m.off_pen) : nullptr;
    Gemm3Params p = proj(p_lm, cand_ok ? GEMM3_EPI_ARGMAX : GEMM3_EPI_PLAIN);
    p.out = logits; p.ldo = V; p.cand = cand;
    P(B200_K_GEMM_LM); rc |= launch_proj(p, xm_last, m.S); Q();
    last_S = m.S;
    if (m.n_pen > 0) {
      P(B200_K_ARGMAX);
      rc |= penalize_rows(logits, V, pen_rows, m.n_pen, pen_recs, pen_lens, pen_cap, pen_save, stream);
      Q();
      launched(1);
    }
    P(B200_K_ARGMAX);
    if (samp) rc |= sample_rows(logits, V, dbuf + m.off_samp, m.samp_words, m.S, V, sampled, stream);
    else if (cand_ok) rc |= argmax_candidates(cand, sampled, m.S, (V + 127) / 128, stream);
    else rc |= argmax_rows(logits, sampled, m.S, V, V, stream);
    Q();
    launched(1);
    if (m.n_pen > 0) {   // logprobs and the kept logits read the raw rows
      P(B200_K_ARGMAX);
      rc |= penalize_restore(logits, V, pen_rows, m.n_pen, pen_recs, pen_lens, pen_cap, pen_save, stream);
      Q();
      launched(1);
    }
    if (m.n_lp > 0) {   // after the token selection: it reads the sampled ids
      const int* lr = dbuf + m.off_lp;
      P(B200_K_ARGMAX);
      rc |= logprobs_rows(logits, V, V, lr, lr + m.n_lp, m.n_lp, sampled, lp_dev, 1 + kMaxLogprobs, lp_dev + 1,
                          1 + kMaxLogprobs, lp_ids_dev, stream);
      Q();
      launched(1);
    }
  }
  // pooled rows: the gathered final norm and the L2 normalisation (on a score head: the score logits and their
  // activation) in one launch, into the pooled readback.  Only scratch is written, so a replay changes nothing a later
  // step reads.
  if (!all_logits && m.E > 0) {
    const int* prow = dbuf + m.off_pool;
    const bf16* px = x_pending ? x : res;
    bf16* pres = x_pending ? res : nullptr;
    P(B200_K_NORM);
    if (num_labels > 0) rc |= score_rows(px, pres, final_norm, score, prow, prow + m.E, m.E, H, num_labels, score_act, cfg.rms_eps, pooled, stream);
    else if (!x_pending) rc |= pool_rows(res, nullptr, final_norm, prow, prow + m.E, m.E, H, cfg.rms_eps, pooled, stream);
    else rc |= pool_rows(x, res, final_norm, prow, prow + m.E, m.E, H, cfg.rms_eps, pooled, stream);
    Q();
    launched(1);
  }
  // prompt-logprob rows, plp_G at a time: gathered final norm (the residual is not written back, so the rows can be read
  // again), plain lm_head into the scratch, then the ranked log-softmax into the step's records.  Only scratch is
  // written, so a replay changes nothing a later step reads.
  if (!all_logits && m.n_plp > 0) {
    const int* ptok = dbuf + m.off_plp;
    const int* ptgt = ptok + m.n_plp;
    const int* pn = ptgt + m.n_plp;
    for (int g0 = 0; g0 < m.n_plp && !rc; g0 += plp_G) {
      const int n = std::min(plp_G, m.n_plp - g0);
      P(B200_K_NORM); norm(final_norm, prompt_hidden, ptok + g0, n); Q();
      Gemm3Params p = proj(p_lm, GEMM3_EPI_PLAIN);
      p.out = prompt_logits; p.ldo = V;
      P(B200_K_GEMM_LM); rc |= launch_proj(p, xm_phid, n); Q();
      P(B200_K_ARGMAX);
      rc |= logprobs_rows(prompt_logits, V, V, nullptr, pn + g0, n, ptgt + g0,
                          plp_f_dev + static_cast<size_t>(g0) * (1 + kMaxLogprobs), 1 + kMaxLogprobs,
                          plp_f_dev + static_cast<size_t>(g0) * (1 + kMaxLogprobs) + 1, 1 + kMaxLogprobs,
                          plp_ids_dev + static_cast<size_t>(g0) * kMaxLogprobs, stream, plp_rank_dev + g0);
      Q();
      launched(1);
    }
  }
  if (rc) return cuda_fail("forward(head)", -2);
  return 0;
}

// ------------------------------------------------------------------ scheduler helpers
// Pages for s up to token `upto`, plus `tails` fresh pages for the members it forks in this step (all or nothing)
bool Engine::ensure_blocks(Seq& s, int upto, int tails) {
  const int need = std::max((upto + kPage - 1) / kPage - static_cast<int>(s.blocks.size()), 0);
  if (need + tails == 0) return true;
  if (pool.free_count() < need + tails) return false;
  for (int i = 0; i < need; ++i) s.blocks.push_back(pool.alloc());
  for (int i = 0; i < tails; ++i) s.fork_tails.push_back(pool.alloc());
  return true;
}

// When a chunk of n tokens completes the prompt of a leader with members not forked yet, the members still live fork in
// this step (s.fork); returns the tail pages they need: one each when the prompt ends inside a page
int Engine::plan_fork(Seq& s, int n) {
  s.fork.clear();
  if (s.children.empty() || s.n_computed + n != static_cast<int>(s.toks.size())) return 0;
  for (auto& c : s.children)
    if (!c->abort_requested.load(std::memory_order_relaxed)) s.fork.push_back(c);
  return s.n_prompt % kPage ? static_cast<int>(s.fork.size()) : 0;
}

// s and the members it has not forked yet
void Engine::finish_group(std::shared_ptr<Seq> s, int code) {
  for (auto& c : s->children) finish(c, code);
  s->children.clear();
  finish(std::move(s), code);
}

void Engine::release_blocks(Seq& s) {
  // tail blocks go to the front of the LRU free queue order first (vLLM frees in reverse)
  for (auto it = s.blocks.rbegin(); it != s.blocks.rend(); ++it) pool.unref(*it);
  s.blocks.clear();
  for (int b : s.fork_tails) pool.unref(b);
  s.fork_tails.clear();
  s.fork.clear();
  if (s.pen_slot >= 0) {   // the record list is a function of s.toks: the next admission rebuilds it
    pen_free.push_back(s.pen_slot);
    s.pen_slot = -1;
  }
  s.n_computed = 0;
  s.n_published = 0;
  s.chain_uid = 0;
}

void Engine::preempt(std::shared_ptr<Seq> s) {
  release_blocks(*s);
  s->admitted = false;
  waiting.push_front(s);
  ++stats.preemptions;
}

void Engine::finish(std::shared_ptr<Seq> s, int code) {
  release_blocks(*s);
  pending_pub.push_back({std::move(s), 0, false, code});
}

// Make the last step's tokens / finish codes visible to the API threads and wake them.  Called right after the NEXT
// step has been enqueued, so the wake-ups (one futex per streaming client) overlap GPU work instead of delaying it.
void Engine::publish() {
  for (auto& p : pending_pub) {
    {
      std::lock_guard<std::mutex> lk(p.s->m);
      p.s->plp_out.insert(p.s->plp_out.end(), pending_plp.begin() + p.plp0, pending_plp.begin() + p.plp0 + p.n_plp);
      if (p.has_tok) p.s->out.push_back(p.tok);
      if (p.lp >= 0) p.s->lp_out.push_back(pending_lp[p.lp]);
      if (p.code) p.s->finished = p.code;
    }
    p.s->cv.notify_all();
    p.s->notify_group();
  }
  pending_pub.clear();
  pending_lp.clear();
  pending_plp.clear();
}

void Engine::admit_prefix(Seq& s) {
  // hash-chained full-block lookup; a hit may cover at most len-1 tokens (kv_cache_manager.py:210-222).  A request with
  // prompt logprobs needs the logits of every prompt position, so it reads no cached block (vLLM's
  // skip_reading_prefix_cache); it still publishes its own blocks.
  const int len = static_cast<int>(s.toks.size());
  const int nfull = s.prompt_logprobs >= 0 ? 0 : (len - 1) / kPage;
  uint64_t parent = 0;
  int hit = 0;
  for (int b = 0; b < nfull; ++b) {
    int blk = pool.lookup(parent, &s.toks[static_cast<size_t>(b) * kPage]);
    if (blk < 0) break;
    pool.ref(blk);
    s.blocks.push_back(blk);
    parent = pool.uid(blk);
    ++hit;
  }
  s.n_computed = hit * kPage;
  s.n_published = hit;
  s.chain_uid = parent;
  if (s.n_cached.load() < 0) {
    s.n_cached = s.n_computed;
    stats.cached_prompt_tokens += s.n_computed;
    stats.prompt_tokens += s.n_prompt;
  }
}

// Build the request's record list from its prompt and generated tokens and upload it, once per admission (the first and
// each one after a preemption); from then on only the device changes it.  The stream is idle here (the previous step has
// completed), so waiting for the copy costs its own time only.
int Engine::admit_edits(Seq& s) {
  s.pen_slot = pen_free.back();
  pen_free.pop_back();
  std::vector<int32_t> stops;
  if (s.n_generated < s.min_tokens) {   // vLLM's all_stop_token_ids: the stop ids and EOS, ignore_eos or not
    for (int32_t t : s.stop_ids) if (t >= 0 && t < V) stops.push_back(t);
    if (cfg.eos_token_id >= 0 && cfg.eos_token_id < V) stops.push_back(cfg.eos_token_id);
  }
  const int np = s.n_prompt, no = static_cast<int>(s.toks.size()) - s.n_prompt;
  penalty_records(s.toks.data(), np, s.toks.data() + np, no, s.pen_history(), s.bias_ids.data(), s.bias_values.data(),
                  static_cast<int>(s.bias_ids.size()), stops.data(), static_cast<int>(stops.size()), &pen_tmp_);
  const int n = static_cast<int>(pen_tmp_.size());
  if (n > pen_cap) { set_error("record list of %d entries exceeds %d", n, pen_cap); return B200_ERR_INVALID; }
  CK(cudaMemcpyAsync(pen_recs + static_cast<size_t>(s.pen_slot) * pen_cap, pen_tmp_.data(), static_cast<size_t>(n) * sizeof(PenaltyRec),
                     cudaMemcpyHostToDevice, stream));
  CK(cudaMemcpyAsync(pen_lens + s.pen_slot, &n, sizeof(int), cudaMemcpyHostToDevice, stream));
  CK(cudaStreamSynchronize(stream));
  return 0;
}

// Speculative decoding's drafts, after the running sequences are scheduled and before any admission (vLLM's order: running
// requests, drafts included, then waiting ones).  A running sequence whose prompt is computed and that decodes one token
// this step proposes up to spec_k drafts and verifies them with that token, as n = 1 + m tokens.  The drafts take only
// the budget the running sequences leave and only free pages: they never preempt, and admission gets what they leave.
// Sequences with history penalties (row j would need drafts 0..j-1 in the device history) and a group's fork step do not
// speculate.
void Engine::add_drafts(std::vector<Sched>& sched, int* budget) {
  for (auto& sc : sched) {
    Seq& s = *sc.s;
    const int len = static_cast<int>(s.toks.size());
    if (*budget <= 0) break;
    if (sc.n != 1 || len - s.n_computed != 1 || s.n_generated == 0 || !s.children.empty() || s.pen_history()) continue;
    // the verify emits up to m + 1 tokens: within max_tokens, and the context stays below max_model_len
    const int cap = std::min({spec_k, s.max_tokens - s.n_generated - 1, cfg.max_model_len - len - 1, *budget});
    if (cap <= 0) continue;
    draft_tmp_.resize(spec_k);
    int m = ngram_propose(s.toks.data(), len, spec_min, spec_max, cap, cfg.max_model_len, draft_tmp_.data());
    if (m <= 0) continue;
    if (!ensure_blocks(s, s.n_computed + 1 + m))   // no free page: only the drafts that fit in the pages it holds
      m = std::min(m, static_cast<int>(s.blocks.size()) * kPage - s.n_computed - 1);
    if (m <= 0) continue;
    s.draft.assign(draft_tmp_.begin(), draft_tmp_.begin() + m);
    sc.n += m;
    sc.n_draft = m;
    *budget -= m;
  }
}

// ------------------------------------------------------------------ one scheduler iteration + forward
// schedule(): take the requests that arrived and drop the aborted ones, then schedule the running sequences (running
// first, then admissions, vLLM v1 order).  Every change to sequence state before the step runs is made here, so that
// pack() only reads.  Returns 0, or negative on error.
int Engine::schedule(std::vector<Sched>& sched) {
  {
    // arrival order (vLLM's FCFS); with fixed_admission the requests that arrived since the last step join the queue in
    // a fixed order (prompt content, then length) instead of the order their client threads reached b200_submit
    std::lock_guard<std::mutex> lk(mu_);
    const size_t first = waiting.size();
    while (!incoming.empty()) {
      waiting.push_back(incoming.front());
      incoming.pop_front();
    }
    if (fixed_admission)
      std::stable_sort(waiting.begin() + static_cast<std::ptrdiff_t>(first), waiting.end(),
                     [](const std::shared_ptr<Seq>& a, const std::shared_ptr<Seq>& b) {
                       return a->arrival_key != b->arrival_key ? a->arrival_key < b->arrival_key : a->n_prompt < b->n_prompt;
                     });
  }
  // aborted requests leave first.  A leader whose members have not forked yet stays while any of them is live: the
  // prompt is computed for them, and it leaves at the fork.
  {
    auto aborted = [](const Seq& s) {
      if (!s.abort_requested.load(std::memory_order_relaxed)) return false;
      for (auto& c : s.children)
        if (!c->abort_requested.load(std::memory_order_relaxed)) return false;
      return true;
    };
    size_t k = 0;
    for (size_t i = 0; i < running.size(); ++i) {
      if (aborted(*running[i])) finish_group(running[i], B200_FINISH_ABORTED);
      else running[k++] = running[i];
    }
    running.resize(k);
    for (auto it = waiting.begin(); it != waiting.end();) {
      if (aborted(**it)) {
        finish_group(*it, B200_FINISH_ABORTED);
        it = waiting.erase(it);
      } else {
        ++it;
      }
    }
  }

  sched.clear();
  int budget = cfg.max_batched_tokens;
  bool preempted = false;
  // 1. running requests first (decodes and in-progress prefills)
  for (size_t i = 0; i < running.size() && budget > 0;) {
    auto s = running[i];  // a copy: the preemption loop below pops elements of `running`, possibly this one
    int n = std::min(static_cast<int>(s->toks.size()) - s->n_computed, budget);
    if (n <= 0) { ++i; continue; }
    bool ok = true;
    while (!ensure_blocks(*s, s->n_computed + n, plan_fork(*s, n))) {
      auto victim = running.back();
      running.pop_back();
      preempt(victim);
      preempted = true;
      if (victim == s) { ok = false; break; }
    }
    if (!ok) break;  // s itself was preempted; everything after it is gone too
    sched.push_back({s, n});
    budget -= n;
    ++i;
  }
  if (spec_k > 0 && !preempted) add_drafts(sched, &budget);
  // 2. admit waiting requests.  A parallel-sampling group holds the running slots of its members from the admission of
  // its leader, so the fork always finds a slot, a sampled row and a logits-edit list for each of them.
  int reserved = 0;
  for (auto& s : running) reserved += static_cast<int>(s->children.size());
  while (!preempted && budget > 0 && !waiting.empty() && static_cast<int>(running.size()) + reserved < cfg.max_num_seqs) {
    auto s = waiting.front();
    const int members = static_cast<int>(s->children.size());
    if (static_cast<int>(running.size()) + reserved + 1 + members > cfg.max_num_seqs) break;
    if (!s->admitted) admit_prefix(*s);
    int n = std::min(static_cast<int>(s->toks.size()) - s->n_computed, budget);
    if (!ensure_blocks(*s, s->n_computed + n, plan_fork(*s, n))) {
      release_blocks(*s);
      if (running.empty() && sched.empty()) {
        // nothing else holds pages and it still does not fit: it never will (cannot happen while the pool holds one
        // max_model_len sequence, which init() enforces) — fail it instead of blocking the queue behind it forever
        waiting.pop_front();
        finish_group(s, B200_FINISH_ERROR);
        continue;
      }
      break;
    }
    s->admitted = true;
    waiting.pop_front();
    running.push_back(s);
    reserved += members;
    if (s->edits())
      if (int rc = admit_edits(*s)) return rc;
    sched.push_back({s, n});
    budget -= n;
  }
  // 3. what the step produces for the sequences it runs
  for (auto& sc : sched) {
    Seq& s = *sc.s;
    if (s.prompt_logprobs >= 0) {
      // positions p in [p0, p0 + n) that still need a record: the row at p gives prompt token p + 1's.  The last prompt
      // position is the sampled row, whose record (if asked for) is the first generated token's.
      const int hi = std::min(s.n_computed + sc.n, s.n_prompt - 1);
      sc.n_plp = std::max(hi - std::max(s.n_computed, s.plp_done), 0);
      if (sc.n_plp > 0) s.plp_done = hi;
    }
    if (!s.children.empty() && s.n_computed + sc.n == static_cast<int>(s.toks.size())) {
      // the fork (plan_fork): a member aborted before it leaves here, the others get their logits-edit lists
      for (auto& c : s.children)
        if (std::find(s.fork.begin(), s.fork.end(), c) == s.fork.end()) finish(c, B200_FINISH_ABORTED);
      s.children.clear();
      for (auto& c : s.fork)
        if (c->edits())
          if (int rc = admit_edits(*c)) return rc;
    }
  }
  {
    std::lock_guard<std::mutex> lk(mu_);
    stats.running = static_cast<int>(running.size());
    stats.waiting = static_cast<int>(waiting.size());
    stats.kv_blocks_free = pool.free_count();
  }
  return 0;
}

// One sampled row: logits row `token_row`, drawn as the token with index gen_index of q's generation (so a request
// recomputed after preemption draws the same noise), with q's logits edits and logprobs
void Engine::add_row(const Seq& q, int token_row, int gen_index) {
  rows_.push_back(token_row);
  const int row = static_cast<int>(rows_.size()) - 1;
  samp_.push_back({q.temperature, q.top_k, q.top_p, static_cast<uint32_t>(q.seed), static_cast<uint32_t>(q.seed >> 32),
                   gen_index, q.min_p});
  if (q.pen_slot >= 0)
    pen_.push_back({row, q.pen_slot, q.presence, q.frequency, q.repetition, gen_index, q.min_tokens, q.pen_history() ? 1 : 0});
  if (q.top_logprobs >= 0) {
    lp_rows_.push_back(row);
    lp_n_.push_back(q.top_logprobs);
  }
}

// pack(): the step's device inputs in stage_host, from the sequence state schedule() left, which it only reads.  The
// sections in word order: token ids, positions and KV slots [T] each; the sampled rows' token indices [S]; 4-word aligned,
// the decode and the prefill work lists; the block tables [nseq][max_blocks_per_seq]; then, each only in steps that have
// such a row, the SampleRows, PenaltyRows, logprobs rows, prompt-logprob rows and fork page copies.
int Engine::pack(const std::vector<Sched>& sched, StepMeta* mp) {
  StepMeta& m = *mp;
  m = StepMeta();
  m.nseq = static_cast<int>(sched.size());
  for (auto& sc : sched) m.T += sc.n;
  dwork_.clear();
  pwork_.clear();
  rows_.clear();
  samp_.clear();
  lp_rows_.clear();
  lp_n_.clear();
  pen_.clear();
  plp_tok_.clear();
  plp_tgt_.clear();
  plp_n_.clear();
  fork_src_.clear();
  fork_dst_.clear();
  pool_rows_.clear();
  pool_flags_.clear();
  int32_t* h = stage_host;
  m.off_ids = 0; m.off_pos = m.T; m.off_slots = 2 * m.T;
  int tok = 0;
  for (int si = 0; si < m.nseq; ++si) {
    const Sched& sc = sched[si];
    const Seq& s = *sc.s;
    const int n = sc.n, p0 = s.n_computed, nd = sc.n_draft;
    for (int j = 0; j < n; ++j) {
      const int p = p0 + j;
      h[m.off_ids + tok + j] = j < n - nd ? s.toks[p] : s.draft[j - (n - nd)];
      h[m.off_pos + tok + j] = p;
      h[m.off_slots + tok + j] = s.blocks[p / kPage] * kPage + (p % kPage);
    }
    // the chunk's prompt-logprob rows: the last sc.n_plp positions before min(p0 + n, n_prompt - 1)
    const int plp_hi = std::min(p0 + n, s.n_prompt - 1);
    for (int p = plp_hi - sc.n_plp; p < plp_hi; ++p) {
      plp_tok_.push_back(tok + p - p0);
      plp_tgt_.push_back(s.toks[p + 1]);
      plp_n_.push_back(s.prompt_logprobs);
    }
    if (n == 1 || nd > 0) {
      // a decode, or a speculative verify: its 1 + nd positions share one decode work item (attention.cu)
      dwork_.push_back({tok, n, p0, si});
      m.draft_tokens += nd;
      ++m.ndec_seq;
    } else {
      const int qb = kPrefillQueryBlock;
      for (int j = 0; j < n; j += qb) pwork_.push_back({tok + j, std::min(qb, n - j), p0 + j, si});
      ++m.npre_seq;
    }
    m.kv_tokens += p0 + n;  // unique K/V tokens this sequence streams from HBM (query tiles re-read them from L2)
    if (s.embed && p0 + n == static_cast<int>(s.toks.size())) {
      // the chunk that completes an embedding request's prompt: its last position is pooled
      pool_rows_.push_back(tok + n - 1);
      pool_flags_.push_back(s.normalize ? 1 : 0);
    } else if (p0 + n - nd == static_cast<int>(s.toks.size())) {
      // row j (0..nd) of a verify is drawn as the token with index n_generated + j: accepting draft j exactly when it
      // equals row j's token gives the stream the non-speculative steps would
      for (int j = 0; j <= nd; ++j) add_row(s, tok + n - 1 - nd + j, s.n_generated + j);
      // the fork: the last prompt position is sampled once more for every member that forks, each row with the member's
      // own seed, logits-edit list and logprobs (the gathered final norm reads a row index any number of times)
      for (size_t k = 0; k < s.fork.size(); ++k) {
        add_row(*s.fork[k], tok + n - 1, 0);
        if (!s.fork_tails.empty()) {   // the prompt ends inside its last page: each member gets its own copy
          fork_src_.push_back(s.blocks[s.n_prompt / kPage]);
          fork_dst_.push_back(s.fork_tails[k]);
        }
      }
    }
    tok += n;
  }
  // longest-context work first: CTAs are dispatched in blockIdx order, so the tail of the attention grid is made of
  // the shortest sequences (LPT scheduling) instead of whatever happened to be last
  auto longer = [](const AttnWork& a, const AttnWork& b) { return a.q_pos0 + a.q_count > b.q_pos0 + b.q_count; };
  std::stable_sort(dwork_.begin(), dwork_.end(), longer);
  std::stable_sort(pwork_.begin(), pwork_.end(), longer);
  m.nd = static_cast<int>(dwork_.size());
  m.dmax_ctx = m.nd ? dwork_[0].q_pos0 + dwork_[0].q_count : 0;   // sorted longest-first
  m.np = static_cast<int>(pwork_.size());
  m.S = static_cast<int>(rows_.size());
  m.out_tokens = m.S;
  m.n_pen = static_cast<int>(pen_.size());
  m.n_lp = static_cast<int>(lp_rows_.size());
  m.n_plp = static_cast<int>(plp_tok_.size());
  m.n_fork = static_cast<int>(fork_src_.size());
  m.E = static_cast<int>(pool_rows_.size());
  bool any_sampled = false, any_minp = false;   // (submit zeroes min_p for greedy requests)
  for (auto& r : samp_) {
    any_sampled |= r.temperature >= 1e-5f;
    any_minp |= r.min_p > 0.f;
  }
  for (auto& r : pen_) m.pen_update |= r.history != 0;

  int w = 3 * m.T;
  auto put = [&](const auto& v) {   // appends a section, returns its offset
    const int off = w;
    memcpy(h + w, v.data(), v.size() * sizeof(v[0]));
    w += static_cast<int>(v.size() * sizeof(v[0]) / sizeof(int32_t));
    return off;
  };
  m.off_rows = put(rows_);
  w = (w + 3) & ~3;
  m.off_dwork = put(dwork_);
  m.off_pwork = put(pwork_);
  m.off_btab = w;
  for (int si = 0; si < m.nseq; ++si) {
    const Seq& s = *sched[si].s;
    memcpy(h + w + static_cast<size_t>(si) * max_blocks_per_seq, s.blocks.data(), s.blocks.size() * 4);
  }
  w += m.nseq * max_blocks_per_seq;
  if (any_sampled) {   // greedy-only steps carry no sampling section, and min_p takes a word only in steps that have it
    m.off_samp = w;
    m.samp_words = any_minp ? 7 : 6;
    for (int i = 0; i < m.S; ++i) memcpy(h + w + i * m.samp_words, &samp_[i], m.samp_words * sizeof(int32_t));
    w += m.samp_words * m.S;
  }
  if (m.n_pen > 0) m.off_pen = put(pen_);
  if (m.n_lp > 0) {
    m.off_lp = put(lp_rows_);
    put(lp_n_);
  }
  if (m.n_plp > 0) {
    m.off_plp = put(plp_tok_);
    put(plp_tgt_);
    put(plp_n_);
  }
  if (m.n_fork > 0) {
    m.off_fork = put(fork_src_);
    put(fork_dst_);
  }
  if (m.E > 0) {
    m.off_pool = put(pool_rows_);
    put(pool_flags_);
  }
  m.words = w;
  if (w > step_words_cap) {
    set_error("step staging overflow (%d > %d words)", w, step_words_cap);
    return B200_ERR_INVALID;
  }
  return 0;
}

// The most words pack() writes, section by section.  A step runs at most max_num_seqs sequences (a parallel-sampling
// group holds a running slot per member from its leader's admission) and T <= Tcap tokens; it samples S <= Scap rows (one
// per sequence and fork member, plus one per draft).
int Engine::step_words_bound() const {
  static_assert(sizeof(SampleRow) == 7 * sizeof(int32_t), "SampleRow is 7 words of the step input");
  static_assert(sizeof(PenaltyRow) == 8 * sizeof(int32_t), "PenaltyRow is 8 words of the step input");
  static_assert(sizeof(AttnWork) == 4 * sizeof(int32_t), "AttnWork is 4 words of the step input");
  const int seqs = cfg.max_num_seqs;
  return 3 * Tcap                                 // token ids, positions, KV slots
         + Scap + 3                               // sampled rows' token indices, then the alignment
         + 4 * seqs                               // decode work: one item per decoding sequence
         + 4 * (Tcap / kPrefillQueryBlock + seqs) // prefill work: ceil(n / kPrefillQueryBlock) items per chunk of n tokens
         + seqs * max_blocks_per_seq              // block tables
         + 7 * Scap + 8 * Scap + 2 * Scap         // SampleRows, PenaltyRows, logprobs rows (row, N): at most one each per row
         + 3 * Tcap                               // prompt-logprob rows (token, target, N): at most one per token
         + 2 * seqs                               // fork page copies (source, destination): at most one per member
         + (pooling ? 2 * seqs : 0);              // pooled rows (token, flag): at most one per sequence
}

// launch(): schedule, pack, then enqueue the H2D copy of the step's inputs, the kernels and the D2H of its outputs.
// Returns 0 when there is nothing to run, 1 when a step is in flight, negative on error.
int Engine::launch(InFlight* f, StepMeta* mp) {
  static const bool timing = [] { const char* e = getenv("B200_STEP_TIMING"); return e && atoi(e) != 0; }();
  f->t_enter = timing ? now_s() : 0.0;
  if (int rc = schedule(f->sched)) return rc;
  if (f->sched.empty()) return 0;
  StepMeta m;
  if (int rc = pack(f->sched, &m)) return rc;

  int slot = ring_n - 1;  // scratch
  if (recording && ring_n > 1) {
    slot = ring_pos;
    ring_pos = (ring_pos + 1) % (ring_n - 1);
    ++recorded;
  }
  ring_meta[slot] = m;
  int32_t* dbuf = stage_dev[slot];
  f->t_packed = timing ? now_s() : 0.0;
  // NVTX range per step (SURVEY.md §5): visible in nsys / ncu --nvtx timelines as "step T=<tokens> dec=<n> pre=<n>"
  char nv[64];
  snprintf(nv, sizeof(nv), "step T=%d dec=%d pre=%d", m.T, m.ndec_seq, m.npre_seq);
  nvtxRangePushA(nv);
  CK(cudaMemcpyAsync(dbuf, stage_host, static_cast<size_t>(m.words) * 4, cudaMemcpyHostToDevice, stream));
  CK(cudaEventRecord(ev0, stream));
  int frc = forward(m, dbuf, false, nullptr);
  if (!frc && m.pen_update) {   // here, not in forward(): a replay must not change any history
    ++stats.kernel_launches;
    if (penalize_update(reinterpret_cast<const PenaltyRow*>(dbuf + m.off_pen), m.n_pen, sampled, pen_recs, pen_lens, pen_cap, stream))
      frc = cuda_fail("penalize_update", -2);
  }
  if (!frc && m.n_fork > 0) {   // likewise: after this step wrote the prompt's KV, before the next step writes past it
    ++stats.kernel_launches;
    const size_t block_bytes = static_cast<size_t>(2) * Hkv * kPage * Dh * 2;
    if (kv_copy_blocks(kv, L, static_cast<int64_t>(kv_layer_elems) * 2, static_cast<int64_t>(block_bytes), dbuf + m.off_fork,
                       dbuf + m.off_fork + m.n_fork, m.n_fork, stream))
      frc = cuda_fail("kv_copy_blocks", -2);
  }
  nvtxRangePop();
  if (frc) return frc;
  CK(cudaEventRecord(ev1, stream));
  cudaError_t readback = cudaSuccess;
  for_each_readback(m.S, m.n_lp, m.n_plp, m.E, [&](auto* dev, auto* host, size_t bytes) {
    if (bytes > 0 && readback == cudaSuccess) readback = cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, stream);
  });
  CK(readback);
  f->t_launched = timing ? now_s() : 0.0;
  *mp = m;
  return 1;
}

// complete(): wait for the step, apply the sampled ids to the engine-private sequence state, queue what the API
// threads must see (tokens, finish codes) for publish().
int Engine::complete(InFlight& f, const StepMeta& m, b200_step_info* info) {
  static const bool timing = [] { const char* e = getenv("B200_STEP_TIMING"); return e && atoi(e) != 0; }();
  CK(cudaStreamSynchronize(stream));
  const double ht3 = timing ? now_s() : 0.0;
  float ms = 0.f;
  cudaEventElapsedTime(&ms, ev0, ev1);

  int ri = 0, li = 0, pi = 0, ei = 0;
  int64_t gen = 0;
  int step_accepted = 0, step_verifies = 0;
  int64_t step_accepted_pos[B200_MAX_SPEC_TOKENS] = {};
  bool any_done = false;
  for (int si = 0; si < m.nseq; ++si) {
    const std::shared_ptr<Seq>& sp = f.sched[si].s;
    Seq& s = *sp;
    const int n = f.sched[si].n, nd = f.sched[si].n_draft;
    const bool samples = (s.n_computed + n - nd == static_cast<int>(s.toks.size()));
    s.n_computed += n - nd;
    // publish newly full blocks to the prefix cache
    auto publish_blocks = [&] {
      while ((s.n_published + 1) * kPage <= s.n_computed) {
        const int b = s.n_published;
        s.chain_uid = pool.publish(s.blocks[b], s.chain_uid, &s.toks[static_cast<size_t>(b) * kPage]);
        ++s.n_published;
      }
    };
    publish_blocks();
    // prompt records come back in step order; they are published with (or before) the first generated token
    const int plp0 = static_cast<int>(pending_plp.size()), n_plp = f.sched[si].n_plp;
    for (int k = 0; k < n_plp; ++k, ++pi) pending_plp.push_back({read_record(true, pi), plp_rank_host[pi]});
    if (!samples) {
      if (n_plp > 0) pending_pub.push_back({sp, 0, false, 0, -1, plp0, n_plp});
      continue;
    }
    if (s.embed) {   // pooled rows come back in step order; the request finishes with its vector
      const float* v = pooled_host + static_cast<size_t>(ei++) * pooled_width();
      {
        std::lock_guard<std::mutex> lk(s.m);
        s.embedding.assign(v, v + pooled_width());
      }
      pending_pub.push_back({sp, 0, false, B200_FINISH_STOP});
      release_blocks(s);
      s.leaving = true;
      any_done = true;
      continue;
    }
    // the sampled token of `q` (the next row), its finish code and its logprobs record
    auto take = [&](Seq& q, int32_t* t, int* lp) {
      *t = sampled_host[ri++];
      q.toks.push_back(*t);
      ++q.n_generated;
      ++gen;
      int code = 0;
      if (!q.ignore_eos && cfg.eos_token_id >= 0 && *t == cfg.eos_token_id) code = B200_FINISH_STOP;
      for (int sid : q.stop_ids) if (*t == sid) code = B200_FINISH_STOP;
      if (!code && q.n_generated >= q.max_tokens) code = B200_FINISH_LENGTH;
      if (!code && static_cast<int>(q.toks.size()) >= cfg.max_model_len) code = B200_FINISH_LENGTH;
      *lp = -1;
      if (q.top_logprobs >= 0) {   // records come back in step order, as the ids do
        *lp = static_cast<int>(pending_lp.size());
        pending_lp.push_back(read_record(false, li++));
      }
      return code;
    };
    // emit row j's token t_j for j = 0..nd, stopping after t_j when it differs from draft j (a speculative verify), when
    // it finishes the request, or at the last row.  Every emitted token is the one the non-speculative steps would give.
    int code = 0, emitted = 0;
    for (int j = 0; j <= nd; ++j) {
      int32_t t = 0;
      int lp = -1;
      code = take(s, &t, &lp);
      pending_pub.push_back({sp, t, true, code, lp, j == 0 ? plp0 : 0, j == 0 ? n_plp : 0});
      ++emitted;
      const bool match = j < nd && t == s.draft[j];
      if (match) ++step_accepted_pos[j];
      step_accepted += match;
      if (code || !match) break;
    }
    // the rows after the last emitted one are skipped, but their ids and records were copied back in step order
    ri += nd + 1 - emitted;
    if (s.top_logprobs >= 0) li += nd + 1 - emitted;
    if (nd > 0) {
      // KV at positions p0 .. p0 + emitted - 1 came from the last token and the drafts that equal the emitted tokens.  The
      // KV a rejected draft left at a later position is never read: attention masks by position, and the next step
      // writes that position before its attention reads it.
      s.n_computed += emitted - 1;
      publish_blocks();
      ++step_verifies;
    }
    const bool fork = !s.fork.empty();
    if (fork && s.abort_requested.load(std::memory_order_relaxed)) {
      // a leader aborted before its fork computed the prompt for its members only: it leaves with no token
      s.toks.pop_back();
      --s.n_generated;
      --gen;
      Pub& p = pending_pub.back();
      p.has_tok = false;
      p.lp = -1;
      p.code = code = B200_FINISH_ABORTED;
    }
    if (fork) {
      // members 1..n-1 become running sequences: the prompt's full pages by reference, their own copy of its partly
      // filled last page, the leader's cache chain and prompt records, and the token their own row sampled
      std::vector<PromptLogprobRecord> plp_all;
      if (s.prompt_logprobs >= 0) {
        { std::lock_guard<std::mutex> lk(s.m); plp_all = s.plp_out; }
        plp_all.insert(plp_all.end(), pending_plp.begin() + plp0, pending_plp.begin() + plp0 + n_plp);
      }
      const int shared = s.n_prompt / kPage;   // with a full last page there are no tails: every page is shared
      for (size_t k = 0; k < s.fork.size(); ++k) {
        const std::shared_ptr<Seq>& cp = s.fork[k];
        Seq& c = *cp;
        for (int b = 0; b < shared; ++b) {
          pool.ref(s.blocks[b]);
          c.blocks.push_back(s.blocks[b]);
        }
        if (!s.fork_tails.empty()) c.blocks.push_back(s.fork_tails[k]);
        c.n_computed = s.n_computed;
        c.n_published = s.n_published;
        c.chain_uid = s.chain_uid;
        c.plp_done = s.plp_done;
        c.n_cached = s.n_cached.load();
        c.admitted = true;
        int32_t tc = 0;
        int lpc = -1;
        const int cc = take(c, &tc, &lpc);
        const int pc0 = static_cast<int>(pending_plp.size());
        pending_plp.insert(pending_plp.end(), plp_all.begin(), plp_all.end());
        pending_pub.push_back({cp, tc, true, cc, lpc, pc0, static_cast<int>(plp_all.size())});
        if (cc) release_blocks(c);
        else running.push_back(cp);
      }
      s.fork_tails.clear();   // owned by the members now
      s.fork.clear();
    }
    if (code) {
      release_blocks(s);
      s.leaving = true;
      any_done = true;
    }
  }
  if (any_done) {
    size_t k = 0;
    for (size_t i = 0; i < running.size(); ++i)
      if (!running[i]->leaving) running[k++] = running[i];
    running.resize(k);
  }
  {
    std::lock_guard<std::mutex> lk(mu_);
    ++stats.steps;
    stats.generated_tokens += gen;
    stats.spec_drafts += step_verifies;
    stats.spec_draft_tokens += m.draft_tokens;
    stats.spec_accepted_tokens += step_accepted;
    for (int j = 0; j < B200_MAX_SPEC_TOKENS; ++j) stats.spec_accepted_per_pos[j] += step_accepted_pos[j];
    stats.last_step_device_us = ms * 1000.0;
    stats.total_device_us += ms * 1000.0;
    stats.last_step_tokens = m.T;
    stats.h2d_bytes += static_cast<int64_t>(m.words) * 4;
    for_each_readback(m.S, m.n_lp, m.n_plp, m.E, [&](auto*, auto*, size_t bytes) { stats.d2h_bytes += static_cast<int64_t>(bytes); });
    stats.running = static_cast<int>(running.size());
    stats.waiting = static_cast<int>(waiting.size());
    stats.kv_blocks_free = pool.free_count();
  }
  if (timing) {
    const double ht4 = now_s();
    if (m.np == 0) {
      double* a = step_timing;
      a[0] += 1; a[1] += f.t_packed - f.t_enter; a[2] += f.t_launched - f.t_packed; a[3] += ht3 - f.t_launched;
      a[4] += ht4 - ht3; a[5] += ms * 1e-3;
      if (step_timing_last_end > 0) a[6] += f.t_enter - step_timing_last_end;
    }
    step_timing_last_end = ht4;
  }
  if (info) {
    info->tokens = m.T;
    info->decode_seqs = m.ndec_seq;
    info->prefill_seqs = m.npre_seq;
    info->sampled = m.S;
    info->kv_tokens_read = m.kv_tokens;
    info->device_us = ms * 1000.0;
    info->draft_tokens = m.draft_tokens;
    info->accepted_tokens = step_accepted;
  }
  return 1;
}

// One synchronous iteration (tests, debugging): results are visible to poll() when it returns.
int Engine::step(b200_step_info* info) {
  if (info) memset(info, 0, sizeof(*info));
  InFlight& f = inflight_;
  StepMeta m;
  int rc = launch(&f, &m);
  if (rc == 1) rc = complete(f, m, info);
  publish();
  return rc;
}

// Up to max_steps iterations back to back: step N's tokens are published to the API threads after step N+1 has been
// enqueued.  Stops early when the engine has had nothing to run for idle_timeout_us.
int Engine::run(int max_steps, int64_t idle_timeout_us, b200_step_info* infos, int* n_done) {
  int done = 0, rc = 0;
  double idle_since = -1.0;
  InFlight& f = inflight_;
  while (done < max_steps) {
    StepMeta m;
    rc = launch(&f, &m);
    publish();
    if (rc < 0) break;
    if (rc == 0) {
      const double now = now_s();
      if (idle_since < 0) idle_since = now;
      if ((now - idle_since) * 1e6 >= static_cast<double>(idle_timeout_us)) break;
      std::unique_lock<std::mutex> lk(mu_);
      cv_work_.wait_for(lk, std::chrono::microseconds(200), [this] { return stop.load() || !incoming.empty(); });
      continue;
    }
    idle_since = -1.0;
    b200_step_info* info = infos ? infos + done : nullptr;
    if (info) memset(info, 0, sizeof(*info));
    rc = complete(f, m, info);
    if (rc < 0) break;
    ++done;
  }
  publish();
  if (n_done) *n_done = done;
  return rc < 0 ? rc : 0;
}

// A CUDA failure poisons this replica: fail everything in flight (the router retries elsewhere,
// internal/modelproxy/handler.go:127-155)
void Engine::fail_all() {
  std::vector<std::shared_ptr<Seq>> all(running.begin(), running.end());
  all.insert(all.end(), waiting.begin(), waiting.end());
  running.clear();
  waiting.clear();
  {
    std::lock_guard<std::mutex> lk(mu_);
    fatal = true;
    all.insert(all.end(), incoming.begin(), incoming.end());
    incoming.clear();
  }
  pending_pub.clear();
  pending_lp.clear();
  pending_plp.clear();
  const size_t n_queued = all.size();
  for (size_t i = 0; i < n_queued; ++i) {   // and the members their leaders have not forked yet
    all.insert(all.end(), all[i]->children.begin(), all[i]->children.end());
    all.insert(all.end(), all[i]->fork.begin(), all[i]->fork.end());
  }
  for (auto& s : all) {
    { std::lock_guard<std::mutex> lk(s->m); s->finished = B200_FINISH_ERROR; }
    s->cv.notify_all();
    s->notify_group();
  }
}

void Engine::loop() {
  cudaSetDevice(cfg.device);
  char tname[16];
  snprintf(tname, sizeof(tname), "b200-step-%d", cfg.device);   // visible in /proc/<pid>/task/*/stat and top -H
  pthread_setname_np(pthread_self(), tname);
  InFlight& f = inflight_;
  while (!stop) {
    StepMeta m;
    int rc = launch(&f, &m);
    publish();  // the previous step's tokens reach the clients while this one runs
    if (rc == 1) rc = complete(f, m, nullptr);
    if (rc < 0) {
      fprintf(stderr, "[b200engine] step failed: %s\n", b200_last_error());
      fail_all();
      return;
    }
    if (rc == 0) {
      std::unique_lock<std::mutex> lk(mu_);
      cv_work_.wait_for(lk, std::chrono::milliseconds(50), [this] { return stop.load() || !incoming.empty(); });
    }
  }
  publish();
}

}  // namespace b200

// ====================================================================== C ABI
using namespace b200;

struct b200_engine {
  Engine impl;
};

extern "C" {

void b200_config_default(b200_config* c) {
  memset(c, 0, sizeof(*c));
  c->device = 0;
  c->num_layers = 32; c->hidden = 4096; c->q_heads = 32; c->kv_heads = 8; c->intermediate = 14336; c->vocab = 128256;
  c->rms_eps = 1e-5f;
  c->rope_theta = 500000.0f;
  c->max_model_len = 2048;
  c->max_num_seqs = 128;
  c->max_batched_tokens = 1536;  // six 256-token GEMM tiles; time to first token grows with the budget
  c->num_kv_blocks = 0;
  c->kv_fraction = 0.85f;
  c->enable_prefix_caching = 1;
  c->eos_token_id = -1;
  c->seed = 0;
  c->init_scale = 4.0f;
  c->manual_step = 0;
  c->record_steps = 0;
  c->rope_scaling_type = 0;
  c->rope_factor = 1.0f;
  c->rope_low_freq_factor = 1.0f;
  c->rope_high_freq_factor = 4.0f;
  c->rope_original_max_pos = 8192;
}

int b200_engine_create(const b200_config* cfg, b200_engine** out) {
  if (!cfg || !out) { set_error("null argument"); return B200_ERR_INVALID; }
  {
    int k, mn, mx, d;   // checked before the device so that a bad speculative config or head size reads the same on every host
    if (int rc = spec_resolve(*cfg, &k, &mn, &mx)) return rc;
    if (int rc = head_dim_resolve(*cfg, &d)) return rc;
  }
  if (cfg->runner != B200_RUNNER_GENERATE && cfg->runner != B200_RUNNER_POOLING) {
    set_error("runner must be 0 (generate) or 1 (pooling), got %d", cfg->runner);
    return B200_ERR_INVALID;
  }
  if (cfg->num_labels < 0 || cfg->num_labels > kMaxScoreLabels) {
    set_error("num_labels %d is not supported: a score head has 1 to %d labels (0 = none)", cfg->num_labels, kMaxScoreLabels);
    return B200_ERR_INVALID;
  }
  if (cfg->num_labels > 0 && cfg->runner != B200_RUNNER_POOLING) {
    set_error("a score head (num_labels = %d) needs the pooling runner", cfg->num_labels);
    return B200_ERR_INVALID;
  }
  if (cfg->score_activation < 0 || cfg->score_activation > kScoreNone) {
    set_error("score_activation must be 0 (default), 1 (sigmoid), 2 (softmax) or 3 (none), got %d", cfg->score_activation);
    return B200_ERR_INVALID;
  }
  if (cfg->runner == B200_RUNNER_POOLING && cfg->num_speculative_tokens > 0) {
    set_error("speculative decoding (num_speculative_tokens=%d) needs the generate runner", cfg->num_speculative_tokens);
    return B200_ERR_INVALID;
  }
  // sliding-window attention is not implemented: inside the window it is full attention, which the kernels compute exactly
  if (cfg->sliding_window < 0 || (cfg->sliding_window > 0 && cfg->max_model_len > cfg->sliding_window)) {
    set_error("max_model_len %d exceeds sliding_window %d: attention beyond the sliding window is not supported (lower "
              "max_model_len to at most %d)", cfg->max_model_len, cfg->sliding_window, cfg->sliding_window);
    return B200_ERR_INVALID;
  }
  if (int rc = require_device()) return rc;
  b200_engine* e = new (std::nothrow) b200_engine();
  if (!e) { set_error("host OOM"); return B200_ERR_OOM; }
  int rc = e->impl.init(*cfg);
  if (rc) { delete e; return rc; }
  *out = e;
  return 0;
}

void b200_engine_destroy(b200_engine* e) { delete e; }

int32_t b200_ngram_propose(const int32_t* toks, int32_t n, int32_t min_n, int32_t max_n, int32_t k, int32_t max_model_len,
                           int32_t* out) {
  if (!toks || !out || n < 0 || min_n < 1 || max_n < min_n || k < 0) {
    set_error("b200_ngram_propose: bad arguments (n=%d min_n=%d max_n=%d k=%d)", n, min_n, max_n, k);
    return B200_ERR_INVALID;
  }
  return ngram_propose(toks, n, min_n, max_n, k, max_model_len, out);
}

// b200_submit (members 1) and b200_submit_n
static int submit_impl(b200_engine* e, const int32_t* prompt_ids, int32_t n, const b200_sampling* sp, int32_t members,
                       uint64_t* req_ids) {
  if (!e || !prompt_ids || n <= 0 || !req_ids) { set_error("b200_submit: bad arguments"); return B200_ERR_INVALID; }
  Engine& g = e->impl;
  if (g.pooling) { set_error("this engine runs the pooling runner: submit embedding requests with b200_submit_embed"); return B200_ERR_INVALID; }
  // vLLM's SamplingParams._verify_args / _verify_greedy_sampling; every member runs at once, so max_num_seqs bounds n
  if (members < 1) { set_error("n must be at least 1, got %d.", members); return B200_ERR_INVALID; }
  if (members > g.cfg.max_num_seqs) { set_error("n (%d) exceeds max_num_seqs %d", members, g.cfg.max_num_seqs); return B200_ERR_INVALID; }
  if (members > 1 && !(sp && sp->temperature >= 1e-5f)) { set_error("n must be 1 when using greedy sampling, got %d.", members); return B200_ERR_INVALID; }
  const int max_tokens = sp && sp->max_tokens > 0 ? sp->max_tokens : 16;
  if (n + 1 > g.cfg.max_model_len) { set_error("prompt (%d tokens) exceeds max_model_len %d", n, g.cfg.max_model_len); return B200_ERR_INVALID; }
  if (sp && !(std::isfinite(sp->temperature) && sp->temperature >= 0.f)) { set_error("temperature must be finite and >= 0"); return B200_ERR_INVALID; }
  if (sp && !(sp->top_p >= 0.f && sp->top_p <= 1.f)) { set_error("top_p must be in [0, 1]"); return B200_ERR_INVALID; }
  if (sp && sp->top_k < -1) { set_error("top_k must be >= -1"); return B200_ERR_INVALID; }
  if (sp && (sp->top_logprobs < 0 || sp->top_logprobs > B200_MAX_LOGPROBS)) { set_error("top_logprobs must be in 0..%d", B200_MAX_LOGPROBS); return B200_ERR_INVALID; }
  if (sp && sp->top_logprobs > 0 && !sp->logprobs) { set_error("top_logprobs needs logprobs"); return B200_ERR_INVALID; }
  if (sp && (sp->top_prompt_logprobs < 0 || sp->top_prompt_logprobs > B200_MAX_LOGPROBS)) { set_error("top_prompt_logprobs must be in 0..%d", B200_MAX_LOGPROBS); return B200_ERR_INVALID; }
  if (sp && sp->top_prompt_logprobs > 0 && !sp->prompt_logprobs) { set_error("top_prompt_logprobs needs prompt_logprobs"); return B200_ERR_INVALID; }
  for (int i = 0; i < n; ++i) if (prompt_ids[i] < 0 || prompt_ids[i] >= g.V) { set_error("token id out of range"); return B200_ERR_INVALID; }
  // logits edits: vLLM's SamplingParams._verify_args ranges (repetition_penalty 0 is "off" at this ABI)
  if (sp) {
    if (!(sp->presence_penalty >= -2.f && sp->presence_penalty <= 2.f)) { set_error("presence_penalty must be in [-2, 2]"); return B200_ERR_INVALID; }
    if (!(sp->frequency_penalty >= -2.f && sp->frequency_penalty <= 2.f)) { set_error("frequency_penalty must be in [-2, 2]"); return B200_ERR_INVALID; }
    if (!(sp->repetition_penalty >= 0.f && std::isfinite(sp->repetition_penalty))) { set_error("repetition_penalty must be finite and >= 0"); return B200_ERR_INVALID; }
    if (!(sp->min_p >= 0.f && sp->min_p <= 1.f)) { set_error("min_p must be in [0, 1]"); return B200_ERR_INVALID; }
    if (sp->min_tokens < 0 || sp->min_tokens > max_tokens) { set_error("min_tokens must be in 0..max_tokens (%d)", max_tokens); return B200_ERR_INVALID; }
    if (sp->min_tokens > 0 && sp->num_stop_ids > B200_MAX_LOGIT_BIAS) { set_error("min_tokens takes at most %d stop ids", B200_MAX_LOGIT_BIAS); return B200_ERR_INVALID; }
    if (sp->num_logit_bias < 0 || sp->num_logit_bias > B200_MAX_LOGIT_BIAS) { set_error("logit_bias takes at most %d entries", B200_MAX_LOGIT_BIAS); return B200_ERR_INVALID; }
    if (sp->num_logit_bias > 0 && (!sp->logit_bias_ids || !sp->logit_bias_values)) { set_error("logit_bias: null arrays"); return B200_ERR_INVALID; }
    for (int i = 0; i < sp->num_logit_bias; ++i) {
      if (sp->logit_bias_ids[i] < 0 || sp->logit_bias_ids[i] >= g.V) { set_error("logit_bias id %d out of range [0, %d)", sp->logit_bias_ids[i], g.V); return B200_ERR_INVALID; }
      if (!std::isfinite(sp->logit_bias_values[i])) { set_error("logit_bias values must be finite"); return B200_ERR_INVALID; }
    }
  }
  auto make = [&] {
    auto s = std::make_shared<Seq>();
    s->toks.assign(prompt_ids, prompt_ids + n);
    s->n_prompt = n;
    s->arrival_key = xxh64(prompt_ids, static_cast<size_t>(n) * sizeof(int32_t), 0);
    s->max_tokens = max_tokens;
    s->ignore_eos = sp && sp->ignore_eos;
    if (sp && sp->num_stop_ids > 0 && sp->stop_ids) s->stop_ids.assign(sp->stop_ids, sp->stop_ids + sp->num_stop_ids);
    if (sp) {
      s->temperature = sp->temperature;
      s->top_p = sp->top_p > 0.f ? sp->top_p : 1.f;   // 0 = off at this ABI
      s->top_k = sp->top_k > 0 ? sp->top_k : 0;
      s->top_logprobs = sp->logprobs ? sp->top_logprobs : -1;
      s->prompt_logprobs = sp->prompt_logprobs ? sp->top_prompt_logprobs : -1;
      s->min_p = sp->temperature >= 1e-5f ? sp->min_p : 0.f;   // greedy rows ignore min_p, as in vLLM
      s->presence = sp->presence_penalty;
      s->frequency = sp->frequency_penalty;
      s->repetition = sp->repetition_penalty > 0.f ? sp->repetition_penalty : 1.f;
      s->min_tokens = sp->min_tokens;
      if (sp->num_logit_bias > 0) {
        s->bias_ids.assign(sp->logit_bias_ids, sp->logit_bias_ids + sp->num_logit_bias);
        s->bias_values.assign(sp->logit_bias_values, sp->logit_bias_values + sp->num_logit_bias);
      }
    }
    return s;
  };
  std::vector<std::shared_ptr<Seq>> group;
  for (int i = 0; i < members; ++i) group.push_back(make());
  if (members > 1) {
    auto wg = std::make_shared<WaitGroup>();
    for (auto& s : group) s->group = wg;
    group[0]->children.assign(group.begin() + 1, group.end());
  }
  {
    std::lock_guard<std::mutex> lk(g.mu_);
    if (g.fatal) { set_error("engine is in a failed state"); return B200_ERR_CUDA; }
    for (int i = 0; i < members; ++i) {
      // member i: seed + i (vLLM's ParentRequest._get_child_sampling_params), or a seed of its own
      group[i]->seed = sp && sp->has_seed ? sp->seed + static_cast<uint64_t>(i) : splitmix64(&g.seed_state);
      group[i]->id = g.next_id++;
      g.requests[group[i]->id] = group[i];
      req_ids[i] = group[i]->id;
    }
    g.incoming.push_back(group[0]);
  }
  g.cv_work_.notify_one();
  return 0;
}

// b200_submit_embed and b200_submit_score: one prefill-only request whose last position is pooled
static int submit_pooled(b200_engine* e, const int32_t* ids, int32_t n, int32_t flag, uint64_t* req_id, bool score) {
  const char* fn = score ? "b200_submit_score" : "b200_submit_embed";
  if (!e || !ids || n <= 0 || !req_id) { set_error("%s: bad arguments", fn); return B200_ERR_INVALID; }
  Engine& g = e->impl;
  if (!g.pooling && !score) { set_error("this engine runs the generate runner: embedding requests need an engine created with runner = pooling"); return B200_ERR_INVALID; }
  if (!g.pooling) { set_error("this engine runs the generate runner: score requests need an engine created with runner = pooling and num_labels > 0"); return B200_ERR_INVALID; }
  if (score && g.num_labels == 0) { set_error("this engine has no score head (num_labels = 0): it serves embeddings, submitted with b200_submit_embed"); return B200_ERR_INVALID; }
  if (!score && g.num_labels > 0) { set_error("this engine has a score head (num_labels = %d): submit score requests with b200_submit_score", g.num_labels); return B200_ERR_INVALID; }
  if (n > g.cfg.max_model_len) { set_error("prompt (%d tokens) exceeds max_model_len %d", n, g.cfg.max_model_len); return B200_ERR_INVALID; }
  for (int i = 0; i < n; ++i)
    if (ids[i] < 0 || ids[i] >= g.V) { set_error("token id %d out of range [0, %d)", ids[i], g.V); return B200_ERR_INVALID; }
  auto s = std::make_shared<Seq>();
  s->toks.assign(ids, ids + n);
  s->n_prompt = n;
  s->arrival_key = xxh64(ids, static_cast<size_t>(n) * sizeof(int32_t), 0);
  s->max_tokens = 0;
  s->embed = true;
  s->normalize = flag != 0;
  {
    std::lock_guard<std::mutex> lk(g.mu_);
    if (g.fatal) { set_error("engine is in a failed state"); return B200_ERR_CUDA; }
    s->id = g.next_id++;
    g.requests[s->id] = s;
    *req_id = s->id;
    g.incoming.push_back(s);
  }
  g.cv_work_.notify_one();
  return 0;
}

int b200_submit_embed(b200_engine* e, const int32_t* ids, int32_t n, int32_t normalize, uint64_t* req_id) {
  return submit_pooled(e, ids, n, normalize, req_id, false);
}

int b200_submit_score(b200_engine* e, const int32_t* ids, int32_t n, int32_t use_activation, uint64_t* req_id) {
  return submit_pooled(e, ids, n, use_activation, req_id, true);
}

// b200_poll_embedding (dim = H) and b200_poll_score (dim = num_labels)
static int poll_pooled(b200_engine* e, uint64_t req_id, float* out, int32_t dim, int32_t* finished, b200_usage* usage,
                       bool score) {
  const char* fn = score ? "b200_poll_score" : "b200_poll_embedding";
  if (!e || !finished) { set_error("%s: bad arguments", fn); return B200_ERR_INVALID; }
  Engine& g = e->impl;
  std::shared_ptr<Seq> s;
  {
    std::lock_guard<std::mutex> lk(g.mu_);
    auto it = g.requests.find(req_id);
    if (it != g.requests.end()) s = it->second;
  }
  if (!s) { set_error("unknown request %llu", static_cast<unsigned long long>(req_id)); return B200_ERR_NOT_FOUND; }
  if (!s->embed || score != (g.num_labels > 0)) {
    set_error("request %llu is not %s request", static_cast<unsigned long long>(req_id), score ? "a score" : "an embedding");
    return B200_ERR_INVALID;
  }
  if (dim != g.pooled_width() || !out) {
    set_error("%s: dim %d != %s %d", fn, dim, score ? "num_labels" : "hidden size", g.pooled_width());
    return B200_ERR_INVALID;
  }
  std::lock_guard<std::mutex> lk(s->m);
  *finished = s->finished;
  if (s->finished == B200_FINISH_STOP) memcpy(out, s->embedding.data(), static_cast<size_t>(dim) * sizeof(float));
  if (usage) {
    const int nc = s->n_cached.load();
    usage->prompt_tokens = s->n_prompt;
    usage->cached_tokens = nc < 0 ? 0 : nc;
    usage->completion_tokens = 0;
  }
  return 0;
}

int b200_poll_embedding(b200_engine* e, uint64_t req_id, float* out, int32_t dim, int32_t* finished, b200_usage* usage) {
  return poll_pooled(e, req_id, out, dim, finished, usage, false);
}

int b200_poll_score(b200_engine* e, uint64_t req_id, float* out, int32_t num_labels, int32_t* finished, b200_usage* usage) {
  return poll_pooled(e, req_id, out, num_labels, finished, usage, true);
}

int b200_submit(b200_engine* e, const int32_t* prompt_ids, int32_t n, const b200_sampling* sp, uint64_t* req_id) {
  return submit_impl(e, prompt_ids, n, sp, 1, req_id);
}

int b200_submit_n(b200_engine* e, const int32_t* prompt_ids, int32_t n_prompt, const b200_sampling* sp, int32_t n,
                  uint64_t* req_ids) {
  return submit_impl(e, prompt_ids, n_prompt, sp, n, req_ids);
}

int b200_engine_set_fixed_admission(b200_engine* e, int32_t on) {
  if (!e) { set_error("null engine"); return B200_ERR_INVALID; }
  std::lock_guard<std::mutex> lk(e->impl.mu_);
  e->impl.fixed_admission = on != 0;
  return 0;
}

int32_t b200_engine_unfinished(b200_engine* e) {
  if (!e) { set_error("null engine"); return B200_ERR_INVALID; }
  Engine& g = e->impl;
  std::lock_guard<std::mutex> lk(g.mu_);
  int32_t n = 0;
  for (auto& kv : g.requests) {
    std::lock_guard<std::mutex> ls(kv.second->m);
    if (!kv.second->finished) ++n;
  }
  return n;
}

static std::shared_ptr<Seq> find_req(Engine& g, uint64_t id) {
  auto it = g.requests.find(id);
  return it == g.requests.end() ? nullptr : it->second;
}

// b200_poll and b200_poll_logprobs: one drain cursor, so ids and their records never come apart
static int poll_impl(b200_engine* e, uint64_t req_id, int32_t* out_ids, float* out_lp, int32_t* out_top_ids,
                     float* out_top_lp, int32_t cap, int32_t* n_out, int32_t* finished, b200_usage* usage) {
  if (!e || !n_out) { set_error("b200_poll: bad arguments"); return B200_ERR_INVALID; }
  Engine& g = e->impl;
  std::shared_ptr<Seq> s;
  {
    std::lock_guard<std::mutex> lk(g.mu_);
    s = find_req(g, req_id);
  }
  if (!s) { set_error("unknown request %llu", static_cast<unsigned long long>(req_id)); return B200_ERR_NOT_FOUND; }
  const bool lp = out_lp != nullptr;
  if (lp && s->top_logprobs < 0) { set_error("request %llu was submitted without logprobs", static_cast<unsigned long long>(req_id)); return B200_ERR_INVALID; }
  if (lp && (!out_top_ids || !out_top_lp)) { set_error("b200_poll_logprobs: bad arguments"); return B200_ERR_INVALID; }
  std::lock_guard<std::mutex> lk(s->m);
  int n = static_cast<int>(std::min<size_t>(s->out.size() - s->drained, cap > 0 && out_ids ? cap : 0));
  if (n > 0) memcpy(out_ids, s->out.data() + s->drained, static_cast<size_t>(n) * 4);
  if (lp)
    for (int k = 0; k < n; ++k) {
      const LogprobRecord& r = s->lp_out[s->drained + k];
      out_lp[k] = r.lp;
      memcpy(out_top_ids + static_cast<size_t>(k) * kMaxLogprobs, r.top_ids, s->top_logprobs * sizeof(int32_t));
      memcpy(out_top_lp + static_cast<size_t>(k) * kMaxLogprobs, r.top_lp, s->top_logprobs * sizeof(float));
    }
  s->drained += n;
  *n_out = n;
  if (finished) *finished = (s->drained == s->out.size()) ? s->finished : 0;
  if (usage) {
    const int nc = s->n_cached.load();
    usage->prompt_tokens = s->n_prompt;
    usage->cached_tokens = nc < 0 ? 0 : nc;
    usage->completion_tokens = static_cast<int>(s->out.size());
  }
  return 0;
}

int b200_poll(b200_engine* e, uint64_t req_id, int32_t* out_ids, int32_t cap, int32_t* n_out, int32_t* finished,
              b200_usage* usage) {
  return poll_impl(e, req_id, out_ids, nullptr, nullptr, nullptr, cap, n_out, finished, usage);
}

int b200_poll_logprobs(b200_engine* e, uint64_t req_id, int32_t* out_ids, float* out_logprob, int32_t* out_top_ids,
                       float* out_top_logprob, int32_t cap, int32_t* n_out, int32_t* finished, b200_usage* usage) {
  if (!out_logprob) { set_error("b200_poll_logprobs: bad arguments"); return B200_ERR_INVALID; }
  return poll_impl(e, req_id, out_ids, out_logprob, out_top_ids, out_top_logprob, cap, n_out, finished, usage);
}

int b200_poll_prompt_logprobs(b200_engine* e, uint64_t req_id, float* out_logprob, int32_t* out_rank, int32_t* out_top_ids,
                              float* out_top_logprob, int32_t cap, int32_t* n_out) {
  if (!e || !out_logprob || !out_rank || !out_top_ids || !out_top_logprob || !n_out) { set_error("b200_poll_prompt_logprobs: bad arguments"); return B200_ERR_INVALID; }
  Engine& g = e->impl;
  std::shared_ptr<Seq> s;
  {
    std::lock_guard<std::mutex> lk(g.mu_);
    s = find_req(g, req_id);
  }
  if (!s) { set_error("unknown request %llu", static_cast<unsigned long long>(req_id)); return B200_ERR_NOT_FOUND; }
  if (s->prompt_logprobs < 0) { set_error("request %llu was submitted without prompt_logprobs", static_cast<unsigned long long>(req_id)); return B200_ERR_INVALID; }
  const int want = s->n_prompt - 1;
  if (cap < want) { set_error("b200_poll_prompt_logprobs: cap %d < %d records", cap, want); return B200_ERR_INVALID; }
  std::lock_guard<std::mutex> lk(s->m);
  const int n = static_cast<int>(s->plp_out.size()) == want ? want : 0;
  for (int k = 0; k < n; ++k) {
    const PromptLogprobRecord& r = s->plp_out[k];
    out_logprob[k] = r.r.lp;
    out_rank[k] = r.rank;
    memcpy(out_top_ids + static_cast<size_t>(k) * kMaxLogprobs, r.r.top_ids, s->prompt_logprobs * sizeof(int32_t));
    memcpy(out_top_logprob + static_cast<size_t>(k) * kMaxLogprobs, r.r.top_lp, s->prompt_logprobs * sizeof(float));
  }
  *n_out = n;
  return 0;
}

int b200_wait(b200_engine* e, uint64_t req_id, int64_t timeout_us) {
  if (!e) { set_error("null engine"); return B200_ERR_INVALID; }
  Engine& g = e->impl;
  std::shared_ptr<Seq> s;
  {
    std::lock_guard<std::mutex> lk(g.mu_);
    s = find_req(g, req_id);
  }
  if (!s) { set_error("unknown request"); return B200_ERR_NOT_FOUND; }
  std::unique_lock<std::mutex> lk(s->m);
  auto ready = [&] { return s->out.size() > s->drained || s->finished != 0; };
  if (timeout_us < 0) { s->cv.wait(lk, ready); return 0; }
  if (!s->cv.wait_for(lk, std::chrono::microseconds(timeout_us), ready)) { set_error("timeout"); return B200_ERR_TIMEOUT; }
  return 0;
}

int b200_wait_any(b200_engine* e, const uint64_t* ids, int32_t count, int64_t timeout_us) {
  if (!e || !ids || count < 1) { set_error("b200_wait_any: bad arguments"); return B200_ERR_INVALID; }
  if (count == 1) return b200_wait(e, ids[0], timeout_us);
  Engine& g = e->impl;
  std::vector<std::shared_ptr<Seq>> ss;
  {
    std::lock_guard<std::mutex> lk(g.mu_);
    for (int i = 0; i < count; ++i) {
      auto s = find_req(g, ids[i]);
      if (!s) { set_error("unknown request %llu", static_cast<unsigned long long>(ids[i])); return B200_ERR_NOT_FOUND; }
      ss.push_back(std::move(s));
    }
  }
  WaitGroup* wg = ss[0]->group.get();
  for (auto& s : ss)
    if (!wg || s->group.get() != wg) { set_error("b200_wait_any: the ids are not members of one b200_submit_n call"); return B200_ERR_INVALID; }
  auto ready = [&] {
    for (auto& s : ss) {
      std::lock_guard<std::mutex> lk(s->m);
      if (s->out.size() > s->drained || s->finished != 0) return true;
    }
    return false;
  };
  const auto deadline = std::chrono::steady_clock::now() + std::chrono::microseconds(std::max<int64_t>(timeout_us, 0));
  for (;;) {
    // a publish after this read of gen bumps it after changing the member: the check below or the wait sees it
    uint64_t gen0;
    { std::lock_guard<std::mutex> lk(wg->m); gen0 = wg->gen; }
    if (ready()) return 0;
    std::unique_lock<std::mutex> lk(wg->m);
    auto bumped = [&] { return wg->gen != gen0; };
    if (timeout_us < 0) wg->cv.wait(lk, bumped);
    else if (!wg->cv.wait_until(lk, deadline, bumped)) { set_error("timeout"); return B200_ERR_TIMEOUT; }
  }
}

int b200_abort(b200_engine* e, uint64_t req_id) {
  if (!e) { set_error("null engine"); return B200_ERR_INVALID; }
  Engine& g = e->impl;
  {
    std::lock_guard<std::mutex> lk(g.mu_);
    auto s = find_req(g, req_id);
    if (!s) { set_error("unknown request"); return B200_ERR_NOT_FOUND; }
    s->abort_requested.store(true);
  }
  g.cv_work_.notify_one();
  return 0;
}

int b200_release(b200_engine* e, uint64_t req_id) {
  if (!e) { set_error("null engine"); return B200_ERR_INVALID; }
  Engine& g = e->impl;
  std::shared_ptr<Seq> s;
  {
    std::lock_guard<std::mutex> lk(g.mu_);
    auto it = g.requests.find(req_id);
    if (it == g.requests.end()) { set_error("unknown request"); return B200_ERR_NOT_FOUND; }
    s = it->second;
    g.requests.erase(it);
  }
  bool fin;
  { std::lock_guard<std::mutex> lk(s->m); fin = s->finished != 0; }
  if (!fin) s->abort_requested.store(true);  // released while running: the engine drops it at the next step
  return 0;
}

int b200_stats_get(b200_engine* e, b200_stats* out) {
  if (!e || !out) { set_error("null argument"); return B200_ERR_INVALID; }
  std::lock_guard<std::mutex> lk(e->impl.mu_);
  *out = e->impl.stats;
  return 0;
}

int b200_engine_is_failed(b200_engine* e) {
  if (!e) return 0;
  std::lock_guard<std::mutex> lk(e->impl.mu_);
  return e->impl.fatal ? 1 : 0;
}

int b200_engine_step(b200_engine* e, b200_step_info* info) {
  if (!e) { set_error("null engine"); return B200_ERR_INVALID; }
  if (!e->impl.cfg.manual_step) { set_error("engine was not created with manual_step"); return B200_ERR_INVALID; }
  cudaSetDevice(e->impl.cfg.device);
  return e->impl.step(info);
}

int b200_engine_run(b200_engine* e, int32_t max_steps, int64_t idle_timeout_us, b200_step_info* infos, int32_t* n_done) {
  if (!e || max_steps <= 0) { set_error("b200_engine_run: bad arguments"); return B200_ERR_INVALID; }
  if (!e->impl.cfg.manual_step) { set_error("engine was not created with manual_step"); return B200_ERR_INVALID; }
  cudaSetDevice(e->impl.cfg.device);
  int done = 0;
  int rc = e->impl.run(max_steps, idle_timeout_us, infos, &done);
  if (n_done) *n_done = done;
  return rc;
}

int b200_engine_replay(b200_engine* e, int32_t n, int32_t repeat, double* ms_total, int64_t* tokens, int64_t* sampled,
                       int64_t* kv_tokens_read, int64_t* launches) {
  if (!e || n <= 0 || repeat <= 0) { set_error("b200_engine_replay: bad arguments"); return B200_ERR_INVALID; }
  Engine& g = e->impl;
  if (!g.cfg.manual_step) { set_error("replay needs manual_step"); return B200_ERR_INVALID; }
  if (n > g.ring_n - 1 || n > g.recorded) { set_error("only %lld steps recorded (ring %d)", static_cast<long long>(g.recorded), g.ring_n); return B200_ERR_INVALID; }
  cudaSetDevice(g.cfg.device);
  int64_t tk = 0, sm = 0, kvt = 0;
  const int64_t l0 = g.stats.kernel_launches;
  CK(cudaEventRecord(g.ev0, g.stream));
  for (int r = 0; r < repeat; ++r) {
    for (int i = n; i >= 1; --i) {
      const int rn = g.ring_n - 1;
      const int slot = ((g.ring_pos - i) % rn + rn) % rn;
      const StepMeta& m = g.ring_meta[slot];
      if (int rc = g.forward(m, g.stage_dev[slot], false, nullptr)) return rc;
      tk += m.T; sm += m.S; kvt += m.kv_tokens;
    }
  }
  CK(cudaEventRecord(g.ev1, g.stream));
  CK(cudaStreamSynchronize(g.stream));
  float ms = 0.f;
  cudaEventElapsedTime(&ms, g.ev0, g.ev1);
  if (ms_total) *ms_total = ms;
  if (tokens) *tokens = tk;
  if (sampled) *sampled = sm;
  if (kv_tokens_read) *kv_tokens_read = kvt;
  if (launches) *launches = g.stats.kernel_launches - l0;
  return 0;
}

int b200_engine_set_skip_mask(b200_engine* e, uint32_t mask) {
  if (!e) { set_error("null engine"); return B200_ERR_INVALID; }
  e->impl.skip_mask = mask;
  return 0;
}

int b200_engine_set_recording(b200_engine* e, int32_t on) {
  if (!e) { set_error("null engine"); return B200_ERR_INVALID; }
  e->impl.recording = on != 0;
  return 0;
}

int b200_engine_profile_range(b200_engine* e, int32_t n, int32_t min_tokens, int32_t max_tokens, double* class_us,
                              int64_t* class_launches, int32_t num_classes, int64_t* steps, int64_t* tokens,
                              int64_t* sampled, int64_t* kv_tokens_read) {
  if (!e || n <= 0 || !class_us || !class_launches || num_classes < B200_K_NUM) { set_error("b200_engine_profile: bad arguments"); return B200_ERR_INVALID; }
  Engine& g = e->impl;
  if (!g.cfg.manual_step) { set_error("profile needs manual_step"); return B200_ERR_INVALID; }
  if (n > g.ring_n - 1 || n > g.recorded) { set_error("only %lld steps recorded", static_cast<long long>(g.recorded)); return B200_ERR_INVALID; }
  cudaSetDevice(g.cfg.device);
  for (int i = 0; i < num_classes; ++i) { class_us[i] = 0; class_launches[i] = 0; }
  int64_t ns = 0, nt = 0, nsm = 0, nkv = 0;
  const int rn = g.ring_n - 1;
  for (int i = n; i >= 1; --i) {
    const int slot = ((g.ring_pos - i) % rn + rn) % rn;
    const StepMeta& m = g.ring_meta[slot];
    if (m.T < min_tokens || m.T > max_tokens) continue;
    g.profiling = true;
    g.prof_used = 0;
    int rc = g.forward(m, g.stage_dev[slot], false, nullptr);
    g.profiling = false;
    if (rc) return rc;
    CK(cudaStreamSynchronize(g.stream));
    for (size_t k = 0; k + 1 < g.prof_used; k += 2) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, g.prof_events[k].second, g.prof_events[k + 1].second);
      class_us[g.prof_events[k].first] += ms * 1000.0;
      class_launches[g.prof_events[k].first] += 1;
    }
    ++ns; nt += m.T; nsm += m.S; nkv += m.kv_tokens;
  }
  if (steps) *steps = ns;
  if (tokens) *tokens = nt;
  if (sampled) *sampled = nsm;
  if (kv_tokens_read) *kv_tokens_read = nkv;
  return 0;
}

int b200_engine_profile(b200_engine* e, int32_t n, double* class_us, int64_t* class_launches, int32_t num_classes) {
  return b200_engine_profile_range(e, n, 0, 1 << 30, class_us, class_launches, num_classes, nullptr, nullptr, nullptr,
                                   nullptr);
}

int b200_engine_reset_prefix_cache(b200_engine* e) {
  if (!e) { set_error("null engine"); return B200_ERR_INVALID; }
  if (!e->impl.cfg.manual_step) { set_error("reset needs manual_step"); return B200_ERR_INVALID; }
  e->impl.pool.reset_cache();
  return 0;
}

int b200_engine_tensor_info(b200_engine* e, const char* name, uint64_t* num_bytes, void** device_ptr) {
  if (!e || !name) { set_error("null argument"); return B200_ERR_INVALID; }
  auto it = e->impl.tensors.find(name);
  if (it == e->impl.tensors.end()) { set_error("unknown tensor %s", name); return B200_ERR_NOT_FOUND; }
  if (num_bytes) *num_bytes = it->second.second;
  if (device_ptr) *device_ptr = it->second.first;
  return 0;
}

static bool is_gate_up(const char* name) {
  const size_t n = strlen(name);
  return n > 4 && strcmp(name + n - 4, ".wgu") == 0;
}

int b200_engine_tensor_read(b200_engine* e, const char* name, void* host_dst, uint64_t cap) {
  uint64_t nb = 0; void* p = nullptr;
  if (int rc = b200_engine_tensor_info(e, name, &nb, &p)) return rc;
  if (!host_dst || cap < nb) { set_error("buffer too small (%llu < %llu)", (unsigned long long)cap, (unsigned long long)nb); return B200_ERR_INVALID; }
  Engine& g = e->impl;
  cudaSetDevice(g.cfg.device);
  CK(cudaStreamSynchronize(g.stream));
  if (is_gate_up(name)) {   // the ABI speaks the logical [gate | up] row order
    void* tmp = nullptr;
    CK(cudaMalloc(&tmp, nb));
    int rc = permute_gate_up(tmp, p, g.I, g.H, 0, g.stream);
    cudaError_t ce = rc ? cudaErrorUnknown : cudaStreamSynchronize(g.stream);
    if (ce == cudaSuccess) ce = cudaMemcpy(host_dst, tmp, nb, cudaMemcpyDeviceToHost);
    cudaFree(tmp);
    if (ce != cudaSuccess) { set_error("tensor_read(%s): %s", name, cudaGetErrorString(ce)); return B200_ERR_CUDA; }
    return 0;
  }
  CK(cudaMemcpy(host_dst, p, nb, cudaMemcpyDeviceToHost));
  return 0;
}

int b200_engine_tensor_write(b200_engine* e, const char* name, const void* host_src, uint64_t n) {
  uint64_t nb = 0; void* p = nullptr;
  if (int rc = b200_engine_tensor_info(e, name, &nb, &p)) return rc;
  if (!host_src || n != nb) { set_error("size mismatch (%llu != %llu)", (unsigned long long)n, (unsigned long long)nb); return B200_ERR_INVALID; }
  Engine& g = e->impl;
  cudaSetDevice(g.cfg.device);
  CK(cudaStreamSynchronize(g.stream));
  CK(cudaMemcpy(p, host_src, nb, cudaMemcpyHostToDevice));
  if (is_gate_up(name)) return b200::engine_relayout_gate_up(e, name);
  return 0;
}

int b200_engine_set_keep_logits(b200_engine* e, int32_t keep) {
  if (!e) { set_error("null engine"); return B200_ERR_INVALID; }
  if (!e->impl.cfg.manual_step) { set_error("keep_logits needs manual_step"); return B200_ERR_INVALID; }
  e->impl.keep_logits = keep != 0;
  return 0;
}

int b200_engine_read_logits(b200_engine* e, void* host_logits_bf16, int32_t rows) {
  if (!e || !host_logits_bf16 || rows <= 0) { set_error("bad arguments"); return B200_ERR_INVALID; }
  Engine& g = e->impl;
  if (!g.keep_logits) { set_error("logits are only kept after b200_engine_set_keep_logits(e, 1)"); return B200_ERR_INVALID; }
  if (rows > g.last_S) { set_error("the last step sampled %d rows", g.last_S); return B200_ERR_INVALID; }
  cudaSetDevice(g.cfg.device);
  CK(cudaStreamSynchronize(g.stream));
  CK(cudaMemcpy(host_logits_bf16, g.logits, static_cast<size_t>(rows) * g.V * 2, cudaMemcpyDeviceToHost));
  return 0;
}

}  // extern "C"

int b200::engine_runner(const b200_engine* e) { return e->impl.pooling ? B200_RUNNER_POOLING : B200_RUNNER_GENERATE; }
int b200::engine_num_labels(const b200_engine* e) { return e->impl.num_labels; }
int b200::engine_score_join_pair(const b200_engine* e) { return e->impl.cfg.score_join_pair; }
int b200::engine_hidden(const b200_engine* e) { return e->impl.H; }

int b200::engine_relayout_gate_up(b200_engine* e, const char* name) {
  uint64_t nb = 0; void* p = nullptr;
  if (int rc = b200_engine_tensor_info(e, name, &nb, &p)) return rc;
  Engine& g = e->impl;
  cudaSetDevice(g.cfg.device);
  void* tmp = nullptr;
  CK(cudaMalloc(&tmp, nb));
  cudaError_t ce = cudaMemcpyAsync(tmp, p, nb, cudaMemcpyDeviceToDevice, g.stream);
  if (ce == cudaSuccess && permute_gate_up(p, tmp, g.I, g.H, 1, g.stream)) ce = cudaErrorUnknown;
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(g.stream);
  cudaFree(tmp);
  if (ce != cudaSuccess) { set_error("relayout(%s): %s", name, cudaGetErrorString(ce)); return B200_ERR_CUDA; }
  return 0;
}

extern "C" {

int b200_engine_forward_logits(b200_engine* e, const int32_t* ids, int32_t n, void* host_logits_bf16) {
  if (!e || !ids || n <= 0 || !host_logits_bf16) { set_error("bad arguments"); return B200_ERR_INVALID; }
  Engine& g = e->impl;
  if (!g.cfg.manual_step) { set_error("forward_logits needs manual_step"); return B200_ERR_INVALID; }
  if (g.pooling) { set_error("forward_logits needs the lm_head, which a pooling engine does not have"); return B200_ERR_INVALID; }
  if (n > g.Tcap || n > g.cfg.max_model_len) { set_error("too many tokens"); return B200_ERR_INVALID; }
  cudaSetDevice(g.cfg.device);
  // one greedy prompt from position 0, packed as a step and staged in the scratch ring slot: the recorded steps stay
  // replayable
  auto s = std::make_shared<Seq>();
  s->toks.assign(ids, ids + n);
  s->n_prompt = n;
  if (!g.ensure_blocks(*s, n)) { set_error("KV pool exhausted"); return B200_ERR_OOM; }
  const std::vector<Sched> sched = {{s, n}};
  StepMeta m;
  int rc = g.pack(sched, &m);
  bf16* dl = nullptr;
  if (!rc && cudaMalloc(&dl, static_cast<size_t>(n) * g.V * 2) != cudaSuccess) { set_error("forward_logits: no memory for the logits"); rc = B200_ERR_OOM; }
  if (!rc) {
    int32_t* dbuf = g.stage_dev[g.ring_n - 1];
    cudaError_t ce = cudaMemcpyAsync(dbuf, g.stage_host, static_cast<size_t>(m.words) * 4, cudaMemcpyHostToDevice, g.stream);
    rc = ce == cudaSuccess ? g.forward(m, dbuf, true, dl) : B200_ERR_CUDA;
    if (!rc) {
      ce = cudaMemcpyAsync(host_logits_bf16, dl, static_cast<size_t>(n) * g.V * 2, cudaMemcpyDeviceToHost, g.stream);
      if (ce == cudaSuccess) ce = cudaStreamSynchronize(g.stream);
      if (ce != cudaSuccess) { set_error("forward_logits: %s", cudaGetErrorString(ce)); rc = B200_ERR_CUDA; }
    }
  }
  cudaFree(dl);
  for (auto it = s->blocks.rbegin(); it != s->blocks.rend(); ++it) g.pool.unref(*it);
  return rc;
}

}  // extern "C"
