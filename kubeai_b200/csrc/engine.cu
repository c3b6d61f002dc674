// In-process inference engine: one instance per GPU replica (SURVEY.md §8a K1-K11, §8b).
// It stands where the reference launches a backend pod (internal/modelcontroller/engine_vllm.go:82-100)
// and is reached through the C ABI in include/b200engine.h instead of the HTTP hop at
// internal/modelproxy/handler.go:158.
//
// Host side (this file): paged-KV block pool with hash-chained prefix cache, continuous-batching
// scheduler with chunked prefill under a per-step token budget (semantics of vLLM's
// v1/core/sched/scheduler.py: running first, then waiting; preempt-by-recompute on KV exhaustion;
// 16-token blocks; a prefix hit covers at most len-1 tokens), the Llama forward as a fixed kernel
// sequence on one CUDA stream, greedy sampling, thread-safe submit/poll/wait/abort.
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

constexpr int kD = 128;
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
  int n_generated = 0;
  std::atomic<int> n_cached{-1};  // prefix-hit tokens at first admission
  bool admitted = false;
  bool leaving = false;  // finished in the step being completed: swept out of the running list
  // shared with API threads: guarded by m (one lock per request, so a step's 128 wake-ups do not convoy on one mutex)
  std::mutex m;
  std::condition_variable cv;
  std::vector<int32_t> out;
  size_t drained = 0;
  int finished = 0;
  uint64_t arrival_key = 0;   // xxh64 of the prompt: admission order among requests that arrive between two steps
  std::atomic<bool> abort_requested{false};
};

struct Sched {
  std::shared_ptr<Seq> s;
  int n;
};
// a launched, not yet completed step
struct InFlight {
  std::vector<Sched> sched;
  int words = 0, ndec_seq = 0, npre_seq = 0;
  double t_enter = 0, t_packed = 0, t_launched = 0;
};
// a result not yet visible to the API threads (published while the next step runs on the GPU)
struct Pub {
  std::shared_ptr<Seq> s;
  int32_t tok;
  bool has_tok;
  int code;
};

struct StepMeta {
  int T = 0, nd = 0, np = 0, S = 0, nseq = 0;
  int off_ids = 0, off_pos = 0, off_slots = 0, off_rows = 0, off_dwork = 0, off_pwork = 0, off_btab = 0;
  int words = 0;
  int64_t kv_tokens = 0;
  int out_tokens = 0;  // sampled rows that produce a generated token
  int dmax_ctx = 0;    // longest context among the decode work items (split-KV decision)
};

struct XMaps {
  CUtensorMap m[kGemmNumBlockN];  // token tiles 32, 64, 128, 256, 512
};

}  // namespace

// ------------------------------------------------------------------ engine
struct Engine {
  b200_config cfg;
  int L, H, Hq, Hkv, I, V, QKV;
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
  GemmPlan p_lm;
  bf16* weights_blob = nullptr;
  size_t weights_bytes = 0;
  std::unordered_map<std::string, std::pair<void*, size_t>> tensors;

  // activations
  bf16 *res = nullptr, *x = nullptr, *normed = nullptr, *qkv = nullptr, *attn = nullptr, *gu = nullptr, *act = nullptr,
       *last_hidden = nullptr, *logits = nullptr;
  int* sampled = nullptr;
  int32_t* sampled_host = nullptr;  // pinned
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
    return paged_attention(qkv, QKV, attn, Hq * kD, kv_l, btab, max_blocks_per_seq, dwork, m.nd, Hq, Hkv, scale, 1, stream, attn_ws, split);
  }
  int prefill_attention(bf16* kv_l, const int* btab, const AttnWork* pwork, int np, float scale) {
    return paged_attention_prefill_tc(qkv, Tcap, QKV, attn, Hq * kD, kv_l, btab, max_blocks_per_seq, pwork, np, Hq, Hkv, scale, stream);
  }
  // one scheduler iteration = launch (schedule, pack, H2D, kernels, D2H enqueue) + complete (sync, apply) + publish
  int launch(InFlight* f, StepMeta* m);
  int complete(InFlight& f, const StepMeta& m, b200_step_info* info);
  void publish();
  int step(b200_step_info* info);
  int run(int max_steps, int64_t idle_timeout_us, b200_step_info* infos, int* n_done);
  void fail_all();
  void loop();
  std::vector<Pub> pending_pub;
  InFlight inflight_;
  std::vector<AttnWork> dwork_, pwork_;  // packing scratch (kept across steps: no per-step allocation)
  std::vector<int> rows_;
  bool ensure_blocks(Seq& s, int upto);
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
  void* frees[] = {weights_blob, res, x, normed, qkv, attn, gu, act, last_hidden, logits, sampled, gemm_ws,
                   gemm_counters, kv, cand, attn_ws};
  for (void* p : frees)
    if (p) cudaFree(p);
  for (auto p : stage_dev)
    if (p) cudaFree(p);
  if (stage_host) cudaFreeHost(stage_host);
  if (sampled_host) cudaFreeHost(sampled_host);
  if (ev0) cudaEventDestroy(ev0);
  if (ev1) cudaEventDestroy(ev1);
  if (stream) cudaStreamDestroy(stream);
}

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

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
              s_a = 1.0f / sqrtf(static_cast<float>(Hq * kD));
  items.push_back({"embed", static_cast<size_t>(V) * H, &embed, 1.0f, 0.f});
  for (int l = 0; l < L; ++l) {
    std::string p = "layers." + std::to_string(l) + ".";
    items.push_back({p + "wqkv", static_cast<size_t>(QKV) * H, &layers[l].wqkv, s_h, 0.f});
    items.push_back({p + "wo", static_cast<size_t>(H) * Hq * kD, &layers[l].wo, s_a, 0.f});
    items.push_back({p + "wgu", static_cast<size_t>(2) * I * H, &layers[l].wgu, s_h, 0.f});
    items.push_back({p + "wdown", static_cast<size_t>(H) * I, &layers[l].wdown, s_i, 0.f});
    items.push_back({p + "norm1", static_cast<size_t>(H), &layers[l].norm1, 0.1f, 1.0f});
    items.push_back({p + "norm2", static_cast<size_t>(H), &layers[l].norm2, 0.1f, 1.0f});
  }
  items.push_back({"final_norm", static_cast<size_t>(H), &final_norm, 0.1f, 1.0f});
  items.push_back({"lm_head", static_cast<size_t>(V) * H, &lm_head, s_h * (cfg.init_scale > 0 ? cfg.init_scale : 4.0f), 0.f});
  size_t total = 0;
  std::vector<size_t> offs;
  for (auto& it : items) {
    offs.push_back(total);
    total += align_up(it.elems * 2, 1024);
  }
  const size_t cs_elems = static_cast<size_t>(cfg.max_model_len) * kD;
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
    std::vector<float> inv(kD / 2);
    for (int i = 0; i < kD / 2; ++i)
      inv[i] = 1.0f / powf(cfg.rope_theta, static_cast<float>(2 * i) / static_cast<float>(kD));
    float pos_div = 1.0f;
    if (cfg.rope_scaling_type == 1) {
      // LinearScalingRotaryEmbedding (rotary_embedding/linear_scaling_rope.py): t / factor
      pos_div = cfg.rope_factor;
    } else if (cfg.rope_scaling_type == 2) {
      // Llama3RotaryEmbedding._compute_inv_freq (rotary_embedding/llama3_rope.py:37-54)
      const float orig = static_cast<float>(cfg.rope_original_max_pos);
      const float low_wl = orig / cfg.rope_low_freq_factor, high_wl = orig / cfg.rope_high_freq_factor;
      for (int i = 0; i < kD / 2; ++i) {
        const float wl = 2.0f * static_cast<float>(M_PI) / inv[i];
        if (wl < high_wl) continue;
        if (wl > low_wl || cfg.rope_low_freq_factor == cfg.rope_high_freq_factor) { inv[i] = inv[i] / cfg.rope_factor; continue; }
        const float smooth = (orig / wl - cfg.rope_low_freq_factor) / (cfg.rope_high_freq_factor - cfg.rope_low_freq_factor);
        inv[i] = (1.0f - smooth) * inv[i] / cfg.rope_factor + smooth * inv[i];
      }
    }
    for (int t = 0; t < cfg.max_model_len; ++t)
      for (int i = 0; i < kD / 2; ++i) {
        const float f = static_cast<float>(t) / pos_div * inv[i];
        h[static_cast<size_t>(t) * kD + i] = __float2bfloat16_rn(cosf(f));
        h[static_cast<size_t>(t) * kD + kD / 2 + i] = __float2bfloat16_rn(sinf(f));
      }
    CK(cudaMemcpyAsync(cos_sin, h.data(), cs_elems * 2, cudaMemcpyHostToDevice, stream));
    CK(cudaStreamSynchronize(stream));
  }

  // ---- activations
  CK(cudaMalloc(&res, static_cast<size_t>(Tcap) * H * 2));
  CK(cudaMalloc(&x, static_cast<size_t>(Tcap) * H * 2));
  CK(cudaMalloc(&normed, static_cast<size_t>(Tcap) * H * 2));
  CK(cudaMalloc(&qkv, static_cast<size_t>(Tcap) * QKV * 2));
  CK(cudaMalloc(&attn, static_cast<size_t>(Tcap) * Hq * kD * 2));
  CK(cudaMalloc(&gu, static_cast<size_t>(Tcap) * 2 * I * 2));
  CK(cudaMalloc(&act, static_cast<size_t>(Tcap) * I * 2));
  CK(cudaMalloc(&last_hidden, static_cast<size_t>(Scap) * H * 2));
  CK(cudaMalloc(&logits, static_cast<size_t>(Scap) * V * 2));
  CK(cudaMalloc(&sampled, static_cast<size_t>(Scap) * 4));
  CK(cudaMemset(normed, 0, static_cast<size_t>(Tcap) * H * 2));
  CK(cudaMemset(attn, 0, static_cast<size_t>(Tcap) * Hq * kD * 2));
  CK(cudaMemset(act, 0, static_cast<size_t>(Tcap) * I * 2));
  CK(cudaMemset(last_hidden, 0, static_cast<size_t>(Scap) * H * 2));
  CK(cudaMallocHost(&sampled_host, static_cast<size_t>(Scap) * 4));
  CK(cudaMalloc(&cand, static_cast<size_t>(std::min(Scap, 128)) * ((V + 127) / 128) * sizeof(float2)));
  // outputs of the last step, readable by name (b200_engine_tensor_read): sampled ids int32 [S]; the lm_head's per-slab
  // {best logit, index} candidates float2 [S][ceil(V / 128)] when the step sampled through them, else bf16 logits [S][V]
  tensors["step.sampled"] = {sampled, static_cast<size_t>(Scap) * 4};
  tensors["step.argmax_candidates"] = {cand, static_cast<size_t>(std::min(Scap, 128)) * ((V + 127) / 128) * sizeof(float2)};
  tensors["step.logits"] = {logits, static_cast<size_t>(Scap) * V * 2};
  CK(cudaMalloc(&attn_ws, attn_split_ws_bytes(kSplitMaxWork, Hkv, kSplitMaxParts)));
  { const char* e = getenv("B200_ATTN_SPLIT"); attn_split_force = e ? atoi(e) : 0; }
  // split-K workspace and arrival counters: the largest need of any projection at any step size up to Tcap
  {
    const int shapes[5][2] = {{QKV, H}, {H, Hq * kD}, {2 * I, H}, {H, I}, {V, H}};
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
    if (plan(&layers[l].p_qkv, layers[l].wqkv, QKV, H) || plan(&layers[l].p_o, layers[l].wo, H, Hq * kD) ||
        plan(&layers[l].p_gu, layers[l].wgu, 2 * I, H) || plan(&layers[l].p_down, layers[l].wdown, H, I))
      return cuda_fail("gemm_plan_init", -2);
  }
  if (plan(&p_lm, lm_head, V, H)) return cuda_fail("gemm_plan_init(lm_head)", -2);
  const int bns[kGemmNumBlockN] = {64, 128, 256};
  for (int i = 0; i < kGemmNumBlockN; ++i) {
    if (gemm_make_x_map(&xm_normed.m[i], normed, Tcap, H, H, bns[i]) ||
        gemm_make_x_map(&xm_attn.m[i], attn, Tcap, Hq * kD, Hq * kD, bns[i]) ||
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
  const size_t block_bytes_layer = static_cast<size_t>(2) * Hkv * kPage * kD * 2;
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
  kv_layer_elems = static_cast<size_t>(nblocks) * 2 * Hkv * kPage * kD;
  CK(cudaMalloc(&kv, kv_layer_elems * 2 * L));
  // the attention kernel gathers whole pages and masks the rows past a sequence's end: those rows must be finite
  CK(cudaMemsetAsync(kv, 0, kv_layer_elems * 2 * L, stream));
  pool.init(nblocks, cfg.enable_prefix_caching != 0);

  // ---- step input ring
  max_blocks_per_seq = (cfg.max_model_len + kPage - 1) / kPage;
  step_words_cap = 3 * Tcap + Scap + 4 * Scap + 4 * (Tcap / 16 + Scap + 1) + Scap * max_blocks_per_seq + 64;
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
  QKV = (Hq + 2 * Hkv) * kD;
  // the constraints of every kernel the forward launches, checked here so that a bad shape fails at create time with a
  // message instead of poisoning the replica at its first step: RMSNorm rows are 256-element multiples up to 8192,
  // argmax and the partial readers use 8-element vectors, GEMM K dims are 64-element TMA boxes
  if (L < 1 || H % 256 || H > 8192 || Hq != 4 * Hkv || Hkv < 1 || I % 64 || V < 8 || V % 8 || c.max_model_len < 16 ||
      c.max_num_seqs < 1 || c.max_batched_tokens < 16) {
    set_error("unsupported model/config (need q_heads == 4*kv_heads, hidden %% 256 == 0 and <= 8192, intermediate %% 64 == 0, "
              "vocab %% 8 == 0, max_model_len >= 16)");
    return B200_ERR_INVALID;
  }
  if (c.rope_scaling_type < 0 || c.rope_scaling_type > 2 ||
      (c.rope_scaling_type != 0 && !(c.rope_factor > 0.f)) ||
      (c.rope_scaling_type == 2 && (!(c.rope_low_freq_factor > 0.f) || !(c.rope_high_freq_factor > 0.f) || c.rope_original_max_pos < 1))) {
    set_error("bad rope scaling parameters (type %d)", c.rope_scaling_type);
    return B200_ERR_INVALID;
  }
  Tcap = (c.max_batched_tokens + 15) / 16 * 16;
  Scap = c.max_num_seqs;
  memset(&stats, 0, sizeof(stats));
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
  const float scale = 1.0f / sqrtf(static_cast<float>(kD));
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
      p.positions = pos; p.slots = slots; p.cos_sin = cos_sin; p.kv_layer = kv_l; p.Hq = Hq; p.Hkv = Hkv; p.max_pos = cfg.max_model_len;
      rc |= launch_proj(p, xm_normed, T);
    }
    Q();
    if (!fused) { P(B200_K_ROPE); if (on(B200_K_ROPE)) rc |= rope_kv_write(qkv, pos, slots, cos_sin, kv_l, T, Hq, Hkv, cfg.max_model_len, stream); Q(); launched(1); }
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
    if (!fused) { P(B200_K_SILU); if (on(B200_K_SILU)) rc |= silu_mul(gu, act, T, I, stream, no_partials(), 1); Q(); launched(1); }
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
    // argmax candidates per 128-row slab in the lm_head epilogue (the candidate buffer holds 128 rows), or bf16 logits
    const bool cand_ok = fused && !keep_logits && m.S <= 128;
    Gemm3Params p = proj(p_lm, cand_ok ? GEMM3_EPI_ARGMAX : GEMM3_EPI_PLAIN);
    p.out = logits; p.ldo = V; p.cand = cand;
    P(B200_K_GEMM_LM); rc |= launch_proj(p, xm_last, m.S); Q();
    last_S = m.S;
    P(B200_K_ARGMAX);
    if (cand_ok) rc |= argmax_candidates(cand, sampled, m.S, (V + 127) / 128, stream);
    else rc |= argmax_rows(logits, sampled, m.S, V, V, stream);
    Q();
    launched(1);
  }
  if (rc) return cuda_fail("forward(head)", -2);
  return 0;
}

// ------------------------------------------------------------------ scheduler helpers
bool Engine::ensure_blocks(Seq& s, int upto) {
  const int need = (upto + kPage - 1) / kPage - static_cast<int>(s.blocks.size());
  if (need <= 0) return true;
  if (pool.free_count() < need) return false;
  for (int i = 0; i < need; ++i) s.blocks.push_back(pool.alloc());
  return true;
}

void Engine::release_blocks(Seq& s) {
  // tail blocks go to the front of the LRU free queue order first (vLLM frees in reverse)
  for (auto it = s.blocks.rbegin(); it != s.blocks.rend(); ++it) pool.unref(*it);
  s.blocks.clear();
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
      if (p.has_tok) p.s->out.push_back(p.tok);
      if (p.code) p.s->finished = p.code;
    }
    p.s->cv.notify_all();
  }
  pending_pub.clear();
}

void Engine::admit_prefix(Seq& s) {
  // hash-chained full-block lookup; a hit may cover at most len-1 tokens (kv_cache_manager.py:210-222)
  const int len = static_cast<int>(s.toks.size());
  const int nfull = (len - 1) / kPage;
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

// ------------------------------------------------------------------ one scheduler iteration + forward
// launch(): schedule (running first, then admissions, vLLM v1 order), pack the step's device inputs, enqueue the
// H2D copy, the kernels and the D2H of the sampled ids.  Returns 0 when there is nothing to run, 1 when a step is
// in flight, negative on error.
int Engine::launch(InFlight* f, StepMeta* mp) {
  static const bool timing = [] { const char* e = getenv("B200_STEP_TIMING"); return e && atoi(e) != 0; }();
  f->t_enter = timing ? now_s() : 0.0;
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
  // aborted requests leave first
  {
    size_t k = 0;
    for (size_t i = 0; i < running.size(); ++i) {
      if (running[i]->abort_requested.load(std::memory_order_relaxed)) finish(running[i], B200_FINISH_ABORTED);
      else running[k++] = running[i];
    }
    running.resize(k);
    for (auto it = waiting.begin(); it != waiting.end();) {
      if ((*it)->abort_requested.load(std::memory_order_relaxed)) {
        finish(*it, B200_FINISH_ABORTED);
        it = waiting.erase(it);
      } else {
        ++it;
      }
    }
  }

  std::vector<Sched>& sched = f->sched;
  sched.clear();
  int budget = cfg.max_batched_tokens;
  bool preempted = false;
  // 1. running requests first (decodes and in-progress prefills)
  for (size_t i = 0; i < running.size() && budget > 0;) {
    auto s = running[i];  // a copy: the preemption loop below pops elements of `running`, possibly this one
    int n = std::min(static_cast<int>(s->toks.size()) - s->n_computed, budget);
    if (n <= 0) { ++i; continue; }
    bool ok = true;
    while (!ensure_blocks(*s, s->n_computed + n)) {
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
  // 2. admit waiting requests
  while (!preempted && budget > 0 && !waiting.empty() && static_cast<int>(running.size()) < cfg.max_num_seqs) {
    auto s = waiting.front();
    if (!s->admitted) admit_prefix(*s);
    int n = std::min(static_cast<int>(s->toks.size()) - s->n_computed, budget);
    if (!ensure_blocks(*s, s->n_computed + n)) {
      release_blocks(*s);
      if (running.empty() && sched.empty()) {
        // nothing else holds pages and it still does not fit: it never will (cannot happen while the pool holds one
        // max_model_len sequence, which init() enforces) — fail it instead of blocking the queue behind it forever
        waiting.pop_front();
        finish(s, B200_FINISH_ERROR);
        continue;
      }
      break;
    }
    s->admitted = true;
    waiting.pop_front();
    running.push_back(s);
    sched.push_back({s, n});
    budget -= n;
  }
  {
    std::lock_guard<std::mutex> lk(mu_);
    stats.running = static_cast<int>(running.size());
    stats.waiting = static_cast<int>(waiting.size());
    stats.kv_blocks_free = pool.free_count();
  }
  if (sched.empty()) return 0;

  // ---- pack the step's device inputs
  StepMeta m;
  m.nseq = static_cast<int>(sched.size());
  for (auto& sc : sched) m.T += sc.n;
  dwork_.clear();
  pwork_.clear();
  rows_.clear();
  int32_t* h = stage_host;
  m.off_ids = 0; m.off_pos = m.T; m.off_slots = 2 * m.T;
  int tok = 0;
  f->ndec_seq = f->npre_seq = 0;
  for (int si = 0; si < m.nseq; ++si) {
    Seq& s = *sched[si].s;
    const int n = sched[si].n, p0 = s.n_computed;
    for (int j = 0; j < n; ++j) {
      const int p = p0 + j;
      h[m.off_ids + tok + j] = s.toks[p];
      h[m.off_pos + tok + j] = p;
      h[m.off_slots + tok + j] = s.blocks[p / kPage] * kPage + (p % kPage);
    }
    if (n == 1) {
      dwork_.push_back({tok, 1, p0, si});
      m.kv_tokens += p0 + 1;
      ++f->ndec_seq;
    } else {
      const int qb = kPrefillQueryBlock;
      for (int j = 0; j < n; j += qb) pwork_.push_back({tok + j, std::min(qb, n - j), p0 + j, si});
      m.kv_tokens += p0 + n;  // unique K/V tokens this sequence streams from HBM (query tiles re-read them from L2)
      ++f->npre_seq;
    }
    if (p0 + n == static_cast<int>(s.toks.size())) rows_.push_back(tok + n - 1);
    tok += n;
  }
  // longest-context work first: CTAs are dispatched in blockIdx order, so the tail of the attention grid is made of
  // the shortest sequences (LPT scheduling) instead of whatever happened to be last
  auto longer = [](const AttnWork& a, const AttnWork& b) { return a.q_pos0 + a.q_count > b.q_pos0 + b.q_count; };
  std::stable_sort(dwork_.begin(), dwork_.end(), longer);
  std::stable_sort(pwork_.begin(), pwork_.end(), longer);
  m.nd = static_cast<int>(dwork_.size());
  m.dmax_ctx = m.nd ? dwork_[0].q_pos0 + 1 : 0;   // sorted longest-first
  m.np = static_cast<int>(pwork_.size());
  m.S = static_cast<int>(rows_.size());
  m.out_tokens = m.S;
  int w = 3 * m.T;
  m.off_rows = w; memcpy(h + w, rows_.data(), rows_.size() * 4); w += m.S;
  w = (w + 3) & ~3;
  m.off_dwork = w; memcpy(h + w, dwork_.data(), dwork_.size() * 16); w += 4 * m.nd;
  m.off_pwork = w; memcpy(h + w, pwork_.data(), pwork_.size() * 16); w += 4 * m.np;
  m.off_btab = w;
  for (int si = 0; si < m.nseq; ++si) {
    Seq& s = *sched[si].s;
    memcpy(h + w + static_cast<size_t>(si) * max_blocks_per_seq, s.blocks.data(), s.blocks.size() * 4);
  }
  w += m.nseq * max_blocks_per_seq;
  m.words = w;
  if (w > step_words_cap) {
    set_error("step staging overflow (%d > %d words)", w, step_words_cap);
    return B200_ERR_INVALID;
  }

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
  snprintf(nv, sizeof(nv), "step T=%d dec=%d pre=%d", m.T, f->ndec_seq, f->npre_seq);
  nvtxRangePushA(nv);
  CK(cudaMemcpyAsync(dbuf, h, static_cast<size_t>(w) * 4, cudaMemcpyHostToDevice, stream));
  CK(cudaEventRecord(ev0, stream));
  const int frc = forward(m, dbuf, false, nullptr);
  nvtxRangePop();
  if (frc) return frc;
  CK(cudaEventRecord(ev1, stream));
  if (m.S) CK(cudaMemcpyAsync(sampled_host, sampled, static_cast<size_t>(m.S) * 4, cudaMemcpyDeviceToHost, stream));
  f->t_launched = timing ? now_s() : 0.0;
  f->words = w;
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

  int ri = 0;
  int64_t gen = 0;
  bool any_done = false;
  for (int si = 0; si < m.nseq; ++si) {
    const std::shared_ptr<Seq>& sp = f.sched[si].s;
    Seq& s = *sp;
    const int n = f.sched[si].n;
    const bool samples = (s.n_computed + n == static_cast<int>(s.toks.size()));
    s.n_computed += n;
    // publish newly full blocks to the prefix cache
    while ((s.n_published + 1) * kPage <= s.n_computed) {
      const int b = s.n_published;
      s.chain_uid = pool.publish(s.blocks[b], s.chain_uid, &s.toks[static_cast<size_t>(b) * kPage]);
      ++s.n_published;
    }
    if (!samples) continue;
    const int32_t t = sampled_host[ri++];
    s.toks.push_back(t);
    ++s.n_generated;
    ++gen;
    int code = 0;
    if (!s.ignore_eos && cfg.eos_token_id >= 0 && t == cfg.eos_token_id) code = B200_FINISH_STOP;
    for (int sid : s.stop_ids) if (t == sid) code = B200_FINISH_STOP;
    if (!code && s.n_generated >= s.max_tokens) code = B200_FINISH_LENGTH;
    if (!code && static_cast<int>(s.toks.size()) >= cfg.max_model_len) code = B200_FINISH_LENGTH;
    pending_pub.push_back({sp, t, true, code});
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
    stats.last_step_device_us = ms * 1000.0;
    stats.total_device_us += ms * 1000.0;
    stats.last_step_tokens = m.T;
    stats.h2d_bytes += static_cast<int64_t>(f.words) * 4;
    stats.d2h_bytes += static_cast<int64_t>(m.S) * 4;
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
    info->decode_seqs = f.ndec_seq;
    info->prefill_seqs = f.npre_seq;
    info->sampled = m.S;
    info->kv_tokens_read = m.kv_tokens;
    info->device_us = ms * 1000.0;
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
  for (auto& s : all) {
    { std::lock_guard<std::mutex> lk(s->m); s->finished = B200_FINISH_ERROR; }
    s->cv.notify_all();
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
  if (int rc = require_device()) return rc;
  b200_engine* e = new (std::nothrow) b200_engine();
  if (!e) { set_error("host OOM"); return B200_ERR_OOM; }
  int rc = e->impl.init(*cfg);
  if (rc) { delete e; return rc; }
  *out = e;
  return 0;
}

void b200_engine_destroy(b200_engine* e) { delete e; }

int b200_submit(b200_engine* e, const int32_t* prompt_ids, int32_t n, const b200_sampling* sp, uint64_t* req_id) {
  if (!e || !prompt_ids || n <= 0 || !req_id) { set_error("b200_submit: bad arguments"); return B200_ERR_INVALID; }
  Engine& g = e->impl;
  const int max_tokens = sp && sp->max_tokens > 0 ? sp->max_tokens : 16;
  if (n + 1 > g.cfg.max_model_len) { set_error("prompt (%d tokens) exceeds max_model_len %d", n, g.cfg.max_model_len); return B200_ERR_INVALID; }
  if (sp && sp->temperature >= 1e-5f) { set_error("only greedy sampling (temperature < 1e-5) is implemented"); return B200_ERR_INVALID; }
  for (int i = 0; i < n; ++i) if (prompt_ids[i] < 0 || prompt_ids[i] >= g.V) { set_error("token id out of range"); return B200_ERR_INVALID; }
  auto s = std::make_shared<Seq>();
  s->toks.assign(prompt_ids, prompt_ids + n);
  s->n_prompt = n;
  s->arrival_key = xxh64(prompt_ids, static_cast<size_t>(n) * sizeof(int32_t), 0);
  s->max_tokens = max_tokens;
  s->ignore_eos = sp && sp->ignore_eos;
  if (sp && sp->num_stop_ids > 0 && sp->stop_ids) s->stop_ids.assign(sp->stop_ids, sp->stop_ids + sp->num_stop_ids);
  {
    std::lock_guard<std::mutex> lk(g.mu_);
    if (g.fatal) { set_error("engine is in a failed state"); return B200_ERR_CUDA; }
    s->id = g.next_id++;
    g.requests[s->id] = s;
    g.incoming.push_back(s);
    *req_id = s->id;
  }
  g.cv_work_.notify_one();
  return 0;
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

int b200_poll(b200_engine* e, uint64_t req_id, int32_t* out_ids, int32_t cap, int32_t* n_out, int32_t* finished,
              b200_usage* usage) {
  if (!e || !n_out) { set_error("b200_poll: bad arguments"); return B200_ERR_INVALID; }
  Engine& g = e->impl;
  std::shared_ptr<Seq> s;
  {
    std::lock_guard<std::mutex> lk(g.mu_);
    s = find_req(g, req_id);
  }
  if (!s) { set_error("unknown request %llu", static_cast<unsigned long long>(req_id)); return B200_ERR_NOT_FOUND; }
  std::lock_guard<std::mutex> lk(s->m);
  int n = static_cast<int>(std::min<size_t>(s->out.size() - s->drained, cap > 0 && out_ids ? cap : 0));
  if (n > 0) memcpy(out_ids, s->out.data() + s->drained, static_cast<size_t>(n) * 4);
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
  if (n > g.Tcap || n > g.cfg.max_model_len) { set_error("too many tokens"); return B200_ERR_INVALID; }
  cudaSetDevice(g.cfg.device);
  Seq s;
  s.toks.assign(ids, ids + n);
  if (!g.ensure_blocks(s, n)) { set_error("KV pool exhausted"); return B200_ERR_OOM; }
  StepMeta m;
  m.T = n; m.nseq = 1;
  int32_t* h = g.stage_host;
  m.off_ids = 0; m.off_pos = n; m.off_slots = 2 * n;
  for (int j = 0; j < n; ++j) {
    h[j] = ids[j];
    h[n + j] = j;
    h[2 * n + j] = s.blocks[j / kPage] * kPage + j % kPage;
  }
  int w = (3 * n + 3) & ~3;
  m.off_rows = w;
  m.off_dwork = w;
  std::vector<AttnWork> pw;
  if (n == 1) { m.nd = 1; h[w] = 0; h[w + 1] = 1; h[w + 2] = 0; h[w + 3] = 0; w += 4; m.off_pwork = w; }
  else {
    m.off_pwork = w;
    const int qb = kPrefillQueryBlock;
    for (int j = 0; j < n; j += qb) { h[w] = j; h[w + 1] = std::min(qb, n - j); h[w + 2] = j; h[w + 3] = 0; w += 4; ++m.np; }
  }
  m.off_btab = w;
  memcpy(h + w, s.blocks.data(), s.blocks.size() * 4);
  w += g.max_blocks_per_seq;
  m.words = w;
  bf16* dl = nullptr;
  CK(cudaMalloc(&dl, static_cast<size_t>(n) * g.V * 2));
  int32_t* dbuf = g.stage_dev[0];
  cudaError_t ce = cudaMemcpyAsync(dbuf, h, static_cast<size_t>(w) * 4, cudaMemcpyHostToDevice, g.stream);
  int rc = ce == cudaSuccess ? g.forward(m, dbuf, true, dl) : B200_ERR_CUDA;
  if (!rc) {
    ce = cudaMemcpyAsync(host_logits_bf16, dl, static_cast<size_t>(n) * g.V * 2, cudaMemcpyDeviceToHost, g.stream);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(g.stream);
    if (ce != cudaSuccess) { set_error("forward_logits: %s", cudaGetErrorString(ce)); rc = B200_ERR_CUDA; }
  }
  cudaFree(dl);
  for (auto it = s.blocks.rbegin(); it != s.blocks.rend(); ++it) g.pool.unref(*it);
  return rc;
}

}  // extern "C"
