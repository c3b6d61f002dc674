// Op-level C-ABI entry points (include/b200engine.h "op-level entry points") + error plumbing.
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <mutex>

#include "../../include/b200engine.h"
#include "errors.h"
#include "gemm.h"
#include "gemm3.h"
#include "kernels.h"

namespace b200 {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int require_device() {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0) {
    set_error("no CUDA device available (%s): the engine has no CPU fallback",
              e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    return B200_ERR_NO_DEVICE;
  }
  return 0;
}

int cuda_fail(const char* what, int rc) {
  cudaError_t e = cudaGetLastError();
  set_error("%s failed (rc=%d, cuda=%s)", what, rc, cudaGetErrorString(e));
  return rc == -1 ? B200_ERR_INVALID : B200_ERR_CUDA;
}

namespace {
// scratch for b200_op_gemm (the engine owns its own)
std::mutex g_mu;
float* g_ws = nullptr;
size_t g_ws_bytes = 0;
int* g_counters = nullptr;
constexpr int kCounterInts = 1 << 20;

int ensure_scratch() {
  std::lock_guard<std::mutex> lk(g_mu);
  if (g_ws) return 0;
  g_ws_bytes = 256ull << 20;
  if (cudaMalloc(&g_ws, g_ws_bytes) != cudaSuccess) return -1;
  if (cudaMalloc(&g_counters, kCounterInts * sizeof(int)) != cudaSuccess) return -1;
  cudaMemset(g_counters, 0, kCounterInts * sizeof(int));
  return 0;
}
}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

const char* b200_last_error(void) { return g_err; }
const char* b200_version(void) { return "kubeai-b200 0.1.0 sm_90a"; }

int b200_op_gemm(const void* w, const void* x, void* out, int32_t N, int32_t T, int32_t K, void* stream) {
  if (int rc = require_device()) return rc;
  if (!w || !x || !out || N <= 0 || T < 0 || K <= 0 || K % 8) {
    set_error("b200_op_gemm: bad arguments N=%d T=%d K=%d", N, T, K);
    return B200_ERR_INVALID;
  }
  if (T == 0) return 0;
  if (ensure_scratch()) {
    set_error("b200_op_gemm: workspace allocation failed");
    return B200_ERR_OOM;
  }
  GemmPlan plan;
  int rc = gemm_plan_init(&plan, w, N, K, K, g_ws, g_ws_bytes, g_counters, kCounterInts);
  if (rc) return cuda_fail("gemm_plan_init", rc);
  const int bn = gemm_block_n_for(T);
  CUtensorMap tmx;
  rc = gemm_make_x_map(&tmx, x, T, K, K, bn);
  if (rc) return cuda_fail("gemm_make_x_map", rc);
  rc = gemm_run(plan, tmx, bn, out, N, T, static_cast<cudaStream_t>(stream));
  if (rc == -9) {
    set_error("b200_op_gemm: problem too large for the op-level scratch");
    return B200_ERR_INVALID;
  }
  if (rc) return cuda_fail("gemm_run", rc);
  return 0;
}

int b200_op_gemm_deferred(const void* w, const void* x, void* out, int32_t N, int32_t T, int32_t K, void* stream) {
  // the engine's form of the product: split-K sized to the device whatever the variant, output rows 16-byte aligned for
  // the vectorised elementwise consumers
  if (int rc = require_device()) return rc;
  if (!w || !x || !out || N <= 0 || T <= 0 || K <= 0 || K % 8 || N % 8) {
    set_error("b200_op_gemm_deferred: bad arguments N=%d T=%d K=%d (N %% 8 == 0 required)", N, T, K);
    return B200_ERR_INVALID;
  }
  if (ensure_scratch()) { set_error("workspace allocation failed"); return B200_ERR_OOM; }
  std::lock_guard<std::mutex> lk(g_mu);
  const int v = gemm_variant();
  gemm_set_variant(2);
  int rc = 0;
  {
    GemmPlan plan;
    rc = gemm_plan_init(&plan, w, N, K, K, g_ws, g_ws_bytes, g_counters, kCounterInts);
    const int bn = gemm_block_n_for(T);
    CUtensorMap tmx;
    if (!rc) rc = gemm_make_x_map(&tmx, x, T, K, K, bn);
    if (!rc) rc = gemm_run(plan, tmx, bn, out, N, T, static_cast<cudaStream_t>(stream));
  }
  gemm_set_variant(v);
  return rc ? cuda_fail("gemm_deferred", rc) : 0;
}

int b200_op_gemm3(const b200_gemm3_args* a, void* stream, int32_t* schedule_out) {
  if (int rc = require_device()) return rc;
  if (!a || !a->w || !a->x || a->N <= 0 || a->T <= 0 || a->K <= 0 || a->x_rows < a->T) {
    set_error("b200_op_gemm3: bad arguments");
    return B200_ERR_INVALID;
  }
  if (ensure_scratch()) { set_error("workspace allocation failed"); return B200_ERR_OOM; }
  static float2* cand = nullptr;          // [128 tokens][slabs]
  static std::mutex mu;
  std::lock_guard<std::mutex> lk(mu);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  constexpr int kMaxCandSlabs = 4096;
  if (!cand && cudaMalloc(&cand, sizeof(float2) * 128 * kMaxCandSlabs) != cudaSuccess) return B200_ERR_OOM;
  const int slabs = (a->N + 127) / 128;
  if (a->epi == GEMM3_EPI_ARGMAX && (slabs > kMaxCandSlabs || !a->argmax_out || a->T > 128)) {
    set_error("b200_op_gemm3: argmax needs argmax_out, T <= 128 and N <= 524288");
    return B200_ERR_INVALID;
  }
  if (a->T > 128 && (a->pro != GEMM3_PRO_NONE || a->normed_out)) {
    set_error("b200_op_gemm3: T > 128 serves PRO_NONE without the fused norm");
    return B200_ERR_INVALID;
  }
  Gemm3Schedule sch;
  int rc = gemm3_schedule(a->N, a->K, a->T, a->force, &sch);
  if (rc) { set_error("b200_op_gemm3: shape / schedule not served (rc=%d, N=%d K=%d T=%d force=%d)", rc, a->N, a->K, a->T, a->force); return B200_ERR_INVALID; }
  GemmPlan plan;
  rc = gemm_plan_init(&plan, a->w, a->N, a->K, a->K, g_ws, g_ws_bytes, g_counters, kCounterInts);
  if (rc) return cuda_fail("gemm_plan_init", rc);
  Gemm3Params p;
  memset(&p, 0, sizeof(p));
  p.tm_w = plan.tm_w;
  rc = gemm_make_x_map(&p.tm_x, a->x, a->x_rows, a->K, a->K, sch.block_n);
  if (rc) return cuda_fail("gemm_make_x_map", rc);
  p.N = a->N; p.T = a->T; p.K = a->K; p.pro = a->pro; p.epi = a->epi;
  p.ssq_in = a->ssq_in; p.ssq_slabs = a->ssq_slabs; p.norm_w = static_cast<const __nv_bfloat16*>(a->norm_w); p.eps = a->eps;
  p.out = static_cast<__nv_bfloat16*>(a->out); p.ldo = a->ldo; p.ssq_out = a->ssq_out;
  p.positions = a->positions; p.slots = a->slots; p.cos_sin = static_cast<const __nv_bfloat16*>(a->cos_sin);
  p.kv_layer = static_cast<__nv_bfloat16*>(a->kv_layer); p.Hq = a->q_heads; p.Hkv = a->kv_heads; p.max_pos = a->max_pos;
  p.head_dim = a->head_dim ? a->head_dim : 128;
  if (a->epi == GEMM3_EPI_ROPE_KV && !attn_head_dim_ok(p.head_dim)) {
    set_error("b200_op_gemm3: head_dim=%d; 64 and 128 are served", a->head_dim);
    return B200_ERR_INVALID;
  }
  p.cand = cand; p.n_valid = a->n_valid > 0 ? a->n_valid : a->N;
  if (a->epi == GEMM3_EPI_RESADD && a->normed_out) {
    if (!a->norm_w_out || !a->ssq_out) { set_error("b200_op_gemm3: the fused norm needs norm_w_out and ssq_out"); return B200_ERR_INVALID; }
    p.normed_out = static_cast<__nv_bfloat16*>(a->normed_out);
    p.norm_w_out = static_cast<const __nv_bfloat16*>(a->norm_w_out);
  }
  p.ws = g_ws; p.ws_bytes = g_ws_bytes;
  p.counters = g_counters; p.counters_cap = kCounterInts;
  if (schedule_out) { schedule_out[0] = sch.S; schedule_out[1] = sch.rule; schedule_out[2] = sch.grid; }
  rc = gemm3_launch(p, sch, st);
  if (rc) return cuda_fail("gemm3_launch", rc);
  if (a->epi == GEMM3_EPI_ARGMAX) {
    rc = argmax_candidates(cand, a->argmax_out, a->T, slabs, st);
    if (rc) return cuda_fail("argmax_candidates", rc);
    cudaStreamSynchronize(st);   // the shared candidate buffer is reused by the next call
  }
  return 0;
}

int b200_schedule_query(int32_t N, int32_t K, int32_t T, int32_t sms, int32_t* out8) {
  if (N <= 0 || K <= 0 || T <= 0 || sms < 2 || !out8) { set_error("b200_schedule_query: bad arguments"); return B200_ERR_INVALID; }
  Gemm3Schedule sch;
  if (gemm3_schedule_for(N, K, T, 0, sms, &sch)) { set_error("b200_schedule_query: shape not served"); return B200_ERR_INVALID; }
  const int ntt = (T + sch.block_n - 1) / sch.block_n;
  const int vals[8] = {sch.block_n, ntt, ((N + 127) / 128) * ntt, sch.S, sch.grid, sch.rule, 0, 0};
  for (int i = 0; i < 8; ++i) out8[i] = vals[i];
  return 0;
}

int b200_attn_split_query(int32_t num_work, int32_t kv_heads, int32_t max_ctx, int32_t sms) {
  if (num_work <= 0 || kv_heads <= 0 || max_ctx <= 0 || sms <= 0) return 1;
  return attn_decode_split(num_work, kv_heads, max_ctx, sms);
}

int b200_set_gemm_variant(int32_t v) {
  gemm_set_variant(v);
  return gemm_variant();
}

int b200_op_gemm_trace(void* trace_dev) {
  if (!trace_dev) return 0;   // tracing off: the only state the GEMM kernels support
  set_error("b200_op_gemm_trace: the GEMM kernels record no timestamps");
  return B200_ERR_INVALID;
}

int b200_op_embed(const void* table, const int32_t* ids, void* out, int32_t T, int32_t H, int32_t vocab,
                  void* stream) {
  if (int rc = require_device()) return rc;
  int rc = embed_gather(table, ids, out, T, H, vocab, static_cast<cudaStream_t>(stream));
  return rc ? cuda_fail("embed_gather", rc) : 0;
}

int b200_op_rmsnorm(const void* x, void* residual, const void* w, void* out, const int32_t* row_index,
                    int32_t rows, int32_t H, float eps, void* stream) {
  if (int rc = require_device()) return rc;
  int rc = rmsnorm(x, residual, w, out, row_index, rows, H, eps, static_cast<cudaStream_t>(stream));
  return rc ? cuda_fail("rmsnorm", rc) : 0;
}

int b200_op_pool_rows(const void* hidden, const void* w, const int32_t* row_index, const int32_t* flags, int32_t rows,
                      int32_t H, float eps, float* out, void* stream) {
  if (int rc = require_device()) return rc;
  if (rows < 0 || H % 256 || H <= 0 || H > 8192 || (rows > 0 && (!hidden || !w || !row_index || !flags || !out))) {
    set_error("b200_op_pool_rows: bad arguments (rows %d, H %d: H %% 256 == 0 and <= 8192)", rows, H);
    return B200_ERR_INVALID;
  }
  int rc = pool_rows(hidden, nullptr, w, row_index, flags, rows, H, eps, out, static_cast<cudaStream_t>(stream));
  return rc ? cuda_fail("pool_rows", rc) : 0;
}

int b200_op_score_rows(const void* hidden, const void* norm_w, const void* score_w, const int32_t* row_index,
                       const int32_t* flags, int32_t rows, int32_t H, int32_t num_labels, int32_t activation, float eps,
                       float* out, void* stream) {
  if (int rc = require_device()) return rc;
  if (rows < 0 || H % 256 || H <= 0 || H > 8192 || num_labels < 1 || num_labels > kMaxScoreLabels || activation < 0 ||
      activation > kScoreNone || (rows > 0 && (!hidden || !norm_w || !score_w || !row_index || !flags || !out))) {
    set_error("b200_op_score_rows: bad arguments (rows %d, H %d, num_labels %d, activation %d: H %% 256 == 0 and <= 8192, "
              "1 <= num_labels <= %d, activation 0..3)", rows, H, num_labels, activation, kMaxScoreLabels);
    return B200_ERR_INVALID;
  }
  const int act = activation ? activation : (num_labels == 1 ? kScoreSigmoid : kScoreSoftmax);
  int rc = score_rows(hidden, nullptr, norm_w, score_w, row_index, flags, rows, H, num_labels, act, eps, out,
                      static_cast<cudaStream_t>(stream));
  return rc ? cuda_fail("score_rows", rc) : 0;
}

int b200_op_rope_kvwrite(void* qkv, const int32_t* positions, const int32_t* slots, const void* cos_sin,
                         void* kv_layer, int32_t T, int32_t q_heads, int32_t kv_heads, int32_t max_pos,
                         void* stream) {
  return b200_op_rope_kvwrite_hd(qkv, positions, slots, cos_sin, kv_layer, T, q_heads, kv_heads, max_pos, 128, stream);
}

int b200_op_rope_kvwrite_hd(void* qkv, const int32_t* positions, const int32_t* slots, const void* cos_sin,
                            void* kv_layer, int32_t T, int32_t q_heads, int32_t kv_heads, int32_t max_pos, int32_t head_dim,
                            void* stream) {
  if (int rc = require_device()) return rc;
  if (!attn_head_dim_ok(head_dim)) {
    set_error("b200_op_rope_kvwrite_hd: head_dim=%d; 64 and 128 are served", head_dim);
    return B200_ERR_INVALID;
  }
  int rc = rope_kv_write(qkv, positions, slots, cos_sin, kv_layer, T, q_heads, kv_heads, max_pos,
                         static_cast<cudaStream_t>(stream), head_dim);
  return rc ? cuda_fail("rope_kv_write", rc) : 0;
}

int b200_op_silu_mul(const void* gate_up, void* out, int32_t T, int32_t I, void* stream) {
  return b200_op_silu_mul_il(gate_up, out, T, I, 0, stream);
}

int b200_op_silu_mul_il(const void* gate_up, void* out, int32_t T, int32_t I, int32_t interleaved, void* stream) {
  if (int rc = require_device()) return rc;
  if (interleaved && I % 64) {
    set_error("b200_op_silu_mul_il: the interleaved layout needs I %% 64 == 0 (I = %d)", I);
    return B200_ERR_INVALID;
  }
  int rc = silu_mul(gate_up, out, T, I, static_cast<cudaStream_t>(stream), interleaved);
  return rc ? cuda_fail("silu_mul", rc) : 0;
}

int b200_op_argmax(const void* logits, int32_t* out, int32_t S, int32_t V, int32_t ld, void* stream) {
  if (int rc = require_device()) return rc;
  int rc = argmax_rows(logits, out, S, V, ld, static_cast<cudaStream_t>(stream));
  return rc ? cuda_fail("argmax_rows", rc) : 0;
}

int b200_op_sample(const void* logits, int32_t ld, const b200_sample_row* rows, int32_t S, int32_t V, int32_t* out, void* stream) {
  if (int rc = require_device()) return rc;
  static_assert(sizeof(b200_sample_row) == sizeof(SampleRow), "b200_sample_row is SampleRow on the wire");
  if (!logits || !rows || !out || S < 0 || V < 1 || ld < V || ld % 8) {
    set_error("b200_op_sample: bad arguments (S=%d V=%d ld=%d; ld %% 8 == 0 and V <= ld required)", S, V, ld);
    return B200_ERR_INVALID;
  }
  int rc = sample_rows(logits, ld, rows, 7, S, V, out, static_cast<cudaStream_t>(stream));
  return rc ? cuda_fail("sample_rows", rc) : 0;
}

namespace {
// One request's record list as the engine builds it at admission (the prompt and output only when a penalty is on, the
// stop ids only while fewer than min_tokens tokens exist) and its PenaltyRow for logits row and list `s`.  False when an
// id is outside [0, V) or a list is malformed.
bool penalty_list_of(const b200_penalty_row& r, int V, int s, std::vector<PenaltyRec>* list, PenaltyRow* prow) {
  auto ids_ok = [&](const int32_t* p, int n) {
    if (n < 0 || (n > 0 && !p)) return false;
    for (int i = 0; i < n; ++i) if (p[i] < 0 || p[i] >= V) return false;
    return true;
  };
  if (!ids_ok(r.prompt, r.num_prompt) || !ids_ok(r.output, r.num_output) || !ids_ok(r.logit_bias_ids, r.num_logit_bias) ||
      !ids_ok(r.stop_ids, r.num_stop_ids) || (r.num_logit_bias > 0 && !r.logit_bias_values) || !(r.repetition_penalty >= 0.f))
    return false;
  const float rp = r.repetition_penalty > 0.f ? r.repetition_penalty : 1.f;
  const bool history = r.presence_penalty != 0.f || r.frequency_penalty != 0.f || rp != 1.f;
  *prow = PenaltyRow{s, s, r.presence_penalty, r.frequency_penalty, rp, r.num_output, r.min_tokens, history ? 1 : 0};
  penalty_records(r.prompt, r.num_prompt, r.output, r.num_output, history, r.logit_bias_ids, r.logit_bias_values,
                  r.num_logit_bias, r.stop_ids, r.num_output < r.min_tokens ? r.num_stop_ids : 0, list);
  return true;
}

// The rows of a slot-addressed launch (host memory) as PenaltyRows, checked against the caller's lists: every row in
// [0, S) and every slot in [0, n_slots), each at most once where `unique_rows` / `unique_slots` ask it (two CTAs on one
// logits row or one list would race), and lens[slot] in [0, cap].  ids_V > 0: every id below lens[slot] of a named list
// is in [0, ids_V) as well (the edit writes logits[row][id]).  Copies lens (and those lists) to the host.
int slot_rows_of(const char* what, const b200_penalty_slot_row* rows, int n, int S, const void* recs, const int32_t* lens,
                 int n_slots, int cap, bool unique_rows, bool unique_slots, int ids_V, std::vector<PenaltyRow>* out) {
  static_assert(sizeof(b200_penalty_slot_row) == sizeof(PenaltyRow), "b200_penalty_slot_row is PenaltyRow on the wire");
  if (n < 0 || (n > 0 && !rows) || S < 1 || !recs || !lens || n_slots < 1 || cap < 1) {
    set_error("%s: bad arguments (n=%d S=%d n_slots=%d cap=%d)", what, n, S, n_slots, cap);
    return B200_ERR_INVALID;
  }
  std::vector<int> h_lens(n_slots);
  if (cudaMemcpy(h_lens.data(), lens, h_lens.size() * sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess)
    return cuda_fail(what, -2);
  std::vector<char> row_seen(S, 0), slot_seen(n_slots, 0);
  out->resize(n);
  for (int i = 0; i < n; ++i) {
    const b200_penalty_slot_row& r = rows[i];
    if (r.row < 0 || r.row >= S || r.slot < 0 || r.slot >= n_slots) {
      set_error("%s: row %d names logits row %d of %d, list %d of %d", what, i, r.row, S, r.slot, n_slots);
      return B200_ERR_INVALID;
    }
    if ((unique_rows && row_seen[r.row]) || (unique_slots && slot_seen[r.slot])) {
      set_error("%s: row %d repeats logits row %d or list %d", what, i, r.row, r.slot);
      return B200_ERR_INVALID;
    }
    if (!(r.repetition_penalty >= 0.f) || h_lens[r.slot] < 0 || h_lens[r.slot] > cap) {
      set_error("%s: row %d has repetition %g or list %d of length %d (cap %d)", what, i, r.repetition_penalty, r.slot,
                h_lens[r.slot], cap);
      return B200_ERR_INVALID;
    }
    if (ids_V > 0 && !slot_seen[r.slot]) {
      std::vector<PenaltyRec> list(h_lens[r.slot]);
      if (cudaMemcpy(list.data(), static_cast<const PenaltyRec*>(recs) + static_cast<size_t>(r.slot) * cap,
                     list.size() * sizeof(PenaltyRec), cudaMemcpyDeviceToHost) != cudaSuccess)
        return cuda_fail(what, -2);
      for (const PenaltyRec& e : list)
        if (e.id < 0 || e.id >= ids_V) {
          set_error("%s: list %d holds id %d outside [0, %d)", what, r.slot, e.id, ids_V);
          return B200_ERR_INVALID;
        }
    }
    row_seen[r.row] = slot_seen[r.slot] = 1;
    (*out)[i] = PenaltyRow{r.row, r.slot, r.presence_penalty, r.frequency_penalty,
                           r.repetition_penalty > 0.f ? r.repetition_penalty : 1.f, r.n_generated, r.min_tokens, r.history};
  }
  return 0;
}
}  // namespace

int b200_op_penalty_list(const b200_penalty_row* row, int32_t V, void* recs, int32_t* lens, int32_t n_slots, int32_t cap,
                         int32_t slot, void* stream) {
  if (int rc = require_device()) return rc;
  std::vector<PenaltyRec> list;
  PenaltyRow prow;
  if (!row || !recs || !lens || V < 1 || cap < 1 || slot < 0 || slot >= n_slots || !penalty_list_of(*row, V, slot, &list, &prow)) {
    set_error("b200_op_penalty_list: bad arguments (V=%d slot=%d n_slots=%d cap=%d) or a token id outside [0, V)", V, slot,
              n_slots, cap);
    return B200_ERR_INVALID;
  }
  const int n = static_cast<int>(list.size());
  if (n > cap) {
    set_error("b200_op_penalty_list: record list of %d entries exceeds %d", n, cap);
    return B200_ERR_INVALID;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t ce = cudaMemcpyAsync(static_cast<PenaltyRec*>(recs) + static_cast<size_t>(slot) * cap, list.data(),
                                   static_cast<size_t>(n) * sizeof(PenaltyRec), cudaMemcpyHostToDevice, st);
  if (ce == cudaSuccess) ce = cudaMemcpyAsync(lens + slot, &n, sizeof(int), cudaMemcpyHostToDevice, st);
  if (cudaStreamSynchronize(st) != cudaSuccess || ce != cudaSuccess) return cuda_fail("b200_op_penalty_list", -2);
  return 0;
}

int b200_op_penalize_update(const b200_penalty_slot_row* rows, int32_t n, const int32_t* sampled, int32_t S, int32_t V,
                            void* recs, int32_t* lens, int32_t n_slots, int32_t cap, void* stream) {
  if (int rc = require_device()) return rc;
  std::vector<PenaltyRow> prow;
  if (int rc = slot_rows_of("b200_op_penalize_update", rows, n, S, recs, lens, n_slots, cap, true, true, 0, &prow)) return rc;
  if (!sampled || V < 1) {
    set_error("b200_op_penalize_update: bad arguments (V=%d)", V);
    return B200_ERR_INVALID;
  }
  for (int s = 0; s < S; ++s)
    if (sampled[s] < 0 || sampled[s] >= V) {
      set_error("b200_op_penalize_update: sampled[%d] = %d is outside [0, %d)", s, sampled[s], V);
      return B200_ERR_INVALID;
    }
  if (n == 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PenaltyRow* d_rows = nullptr;
  int* d_sampled = nullptr;
  cudaError_t ce = cudaMalloc(&d_rows, prow.size() * sizeof(PenaltyRow));
  if (ce == cudaSuccess) ce = cudaMalloc(&d_sampled, static_cast<size_t>(S) * sizeof(int));
  if (ce == cudaSuccess) ce = cudaMemcpyAsync(d_rows, prow.data(), prow.size() * sizeof(PenaltyRow), cudaMemcpyHostToDevice, st);
  if (ce == cudaSuccess) ce = cudaMemcpyAsync(d_sampled, sampled, static_cast<size_t>(S) * sizeof(int), cudaMemcpyHostToDevice, st);
  int rc = ce == cudaSuccess ? 0 : -2;
  if (!rc) rc = penalize_update(d_rows, n, d_sampled, static_cast<PenaltyRec*>(recs), lens, cap, st);
  if (cudaStreamSynchronize(st) != cudaSuccess) rc = -2;   // before the host rows and the scratch go away
  cudaFree(d_rows);
  cudaFree(d_sampled);
  return rc ? cuda_fail("penalize_update", rc) : 0;
}

// penalize_rows, then (edited given) the copy and penalize_restore, on S rows of logits; `lists` holds cap records per
// row's slot, the lengths in `lens`.  Device memory throughout; frees its own scratch.
static int penalize_launch(void* logits, int ld, int S, const std::vector<PenaltyRow>& prow, const PenaltyRec* recs,
                           const int* lens, int cap, void* edited, cudaStream_t st) {
  const int n = static_cast<int>(prow.size());
  PenaltyRow* d_rows = nullptr;
  uint16_t* d_save = nullptr;
  cudaError_t ce = cudaMalloc(&d_rows, prow.size() * sizeof(PenaltyRow));
  if (ce == cudaSuccess) ce = cudaMalloc(&d_save, static_cast<size_t>(n) * cap * sizeof(uint16_t));
  if (ce == cudaSuccess) ce = cudaMemcpyAsync(d_rows, prow.data(), prow.size() * sizeof(PenaltyRow), cudaMemcpyHostToDevice, st);
  int rc = ce == cudaSuccess ? 0 : -2;
  if (!rc) rc = penalize_rows(logits, ld, d_rows, n, recs, lens, cap, d_save, st);
  if (!rc && edited) {
    ce = cudaMemcpyAsync(edited, logits, static_cast<size_t>(S) * ld * 2, cudaMemcpyDeviceToDevice, st);
    rc = ce == cudaSuccess ? penalize_restore(logits, ld, d_rows, n, recs, lens, cap, d_save, st) : -2;
  }
  if (cudaStreamSynchronize(st) != cudaSuccess) rc = -2;   // before the host rows and the scratch go away
  cudaFree(d_rows);
  cudaFree(d_save);
  return rc;
}

int b200_op_penalize_slots(void* logits, int32_t ld, int32_t S, int32_t V, const b200_penalty_slot_row* rows, int32_t n,
                           const void* recs, const int32_t* lens, int32_t n_slots, int32_t cap, void* edited, void* stream) {
  if (int rc = require_device()) return rc;
  if (!logits || V < 1 || ld < V) {
    set_error("b200_op_penalize_slots: bad arguments (S=%d V=%d ld=%d)", S, V, ld);
    return B200_ERR_INVALID;
  }
  std::vector<PenaltyRow> prow;
  if (int rc = slot_rows_of("b200_op_penalize_slots", rows, n, S, recs, lens, n_slots, cap, true, false, V, &prow)) return rc;
  if (n == 0) return 0;
  int rc = penalize_launch(logits, ld, S, prow, static_cast<const PenaltyRec*>(recs), lens, cap, edited,
                           static_cast<cudaStream_t>(stream));
  return rc ? cuda_fail("penalize_rows", rc) : 0;
}

int b200_op_penalize(void* logits, int32_t ld, int32_t S, int32_t V, const b200_penalty_row* rows, void* edited, void* stream) {
  if (int rc = require_device()) return rc;
  if (!logits || (S > 0 && !rows) || S < 0 || V < 1 || ld < V) {
    set_error("b200_op_penalize: bad arguments (S=%d V=%d ld=%d)", S, V, ld);
    return B200_ERR_INVALID;
  }
  if (S == 0) return 0;
  // the engine's lists, one slot per row, built by the engine's host code
  std::vector<std::vector<PenaltyRec>> lists(S);
  std::vector<PenaltyRow> prow(S);
  int cap = 1;
  for (int s = 0; s < S; ++s) {
    if (!penalty_list_of(rows[s], V, s, &lists[s], &prow[s])) {
      set_error("b200_op_penalize: row %d has a token id outside [0, %d) or a bad list", s, V);
      return B200_ERR_INVALID;
    }
    cap = std::max(cap, static_cast<int>(lists[s].size()));
  }
  std::vector<PenaltyRec> recs(static_cast<size_t>(S) * cap);
  std::vector<int> lens(S);
  for (int s = 0; s < S; ++s) {
    std::copy(lists[s].begin(), lists[s].end(), recs.begin() + static_cast<size_t>(s) * cap);
    lens[s] = static_cast<int>(lists[s].size());
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PenaltyRec* d_recs = nullptr;
  int* d_lens = nullptr;
  cudaError_t ce = cudaMalloc(&d_recs, recs.size() * sizeof(PenaltyRec));
  if (ce == cudaSuccess) ce = cudaMalloc(&d_lens, lens.size() * sizeof(int));
  if (ce == cudaSuccess) ce = cudaMemcpyAsync(d_recs, recs.data(), recs.size() * sizeof(PenaltyRec), cudaMemcpyHostToDevice, st);
  if (ce == cudaSuccess) ce = cudaMemcpyAsync(d_lens, lens.data(), lens.size() * sizeof(int), cudaMemcpyHostToDevice, st);
  int rc = ce == cudaSuccess ? penalize_launch(logits, ld, S, prow, d_recs, d_lens, cap, edited, st) : -2;
  if (cudaStreamSynchronize(st) != cudaSuccess) rc = -2;   // before the host lists and the scratch go away
  cudaFree(d_recs);
  cudaFree(d_lens);
  return rc ? cuda_fail("penalize_rows", rc) : 0;
}

int b200_op_logprobs(const void* logits, int32_t ld, int32_t S, int32_t V, const int32_t* tokens, const int32_t* top_n,
                     float* out_logprob, int32_t* out_top_ids, float* out_top_logprob, void* stream) {
  if (int rc = require_device()) return rc;
  static_assert(kMaxLogprobs == B200_MAX_LOGPROBS, "one logprobs limit");
  if (!logits || !tokens || !top_n || !out_logprob || !out_top_ids || !out_top_logprob || S < 0 || V < 1 || ld < V || ld % 8) {
    set_error("b200_op_logprobs: bad arguments (S=%d V=%d ld=%d; ld %% 8 == 0 and V <= ld required)", S, V, ld);
    return B200_ERR_INVALID;
  }
  int rc = logprobs_rows(logits, ld, V, nullptr, top_n, S, tokens, out_logprob, 1, out_top_logprob, kMaxLogprobs, out_top_ids,
                         static_cast<cudaStream_t>(stream));
  return rc ? cuda_fail("logprobs_rows", rc) : 0;
}

int b200_op_logprobs_rank(const void* logits, int32_t ld, int32_t S, int32_t V, const int32_t* tokens, const int32_t* top_n,
                          float* out_logprob, int32_t* out_rank, int32_t* out_top_ids, float* out_top_logprob, void* stream) {
  if (int rc = require_device()) return rc;
  if (!logits || !tokens || !top_n || !out_logprob || !out_rank || !out_top_ids || !out_top_logprob || S < 0 || V < 1 ||
      ld < V || ld % 8) {
    set_error("b200_op_logprobs_rank: bad arguments (S=%d V=%d ld=%d; ld %% 8 == 0 and V <= ld required)", S, V, ld);
    return B200_ERR_INVALID;
  }
  int rc = logprobs_rows(logits, ld, V, nullptr, top_n, S, tokens, out_logprob, 1, out_top_logprob, kMaxLogprobs, out_top_ids,
                         static_cast<cudaStream_t>(stream), out_rank);
  return rc ? cuda_fail("logprobs_rows", rc) : 0;
}

int b200_op_paged_attn(const void* q, int32_t ldq, void* out, int32_t ldo, const void* kv_layer,
                       const int32_t* block_tables, int32_t max_blocks, const int32_t* work, int32_t num_work,
                       int32_t q_heads, int32_t kv_heads, float scale, int32_t decode, void* stream) {
  return b200_op_paged_attn_hd(q, ldq, out, ldo, kv_layer, block_tables, max_blocks, work, num_work, q_heads, kv_heads, scale,
                               decode, 128, stream);
}

int b200_op_paged_attn_hd(const void* q, int32_t ldq, void* out, int32_t ldo, const void* kv_layer,
                          const int32_t* block_tables, int32_t max_blocks, const int32_t* work, int32_t num_work,
                          int32_t q_heads, int32_t kv_heads, float scale, int32_t decode, int32_t head_dim, void* stream) {
  if (int rc = require_device()) return rc;
  static_assert(sizeof(AttnWork) == 16, "AttnWork is int32[4] on the wire");
  if (!decode) {
    set_error("b200_op_paged_attn: decode = 0 is not served; chunked prefill is b200_op_paged_attn_prefill_tc[_hd]");
    return B200_ERR_INVALID;
  }
  if (!attn_head_dim_ok(head_dim)) {
    set_error("b200_op_paged_attn: head_dim=%d; 64 and 128 are served", head_dim);
    return B200_ERR_INVALID;
  }
  if (!attn_group_ok(q_heads, kv_heads)) {
    set_error("b200_op_paged_attn: q_heads=%d kv_heads=%d: kv_heads must divide q_heads with 1..16 query heads per KV head",
              q_heads, kv_heads);
    return B200_ERR_INVALID;
  }
  int rc = paged_attention(q, ldq, out, ldo, kv_layer, block_tables, max_blocks,
                           reinterpret_cast<const AttnWork*>(work), num_work, q_heads, kv_heads, scale,
                           static_cast<cudaStream_t>(stream), nullptr, 1, head_dim);
  return rc ? cuda_fail("paged_attention", rc) : 0;
}

int b200_op_paged_attn_decode_split(const void* q, int32_t ldq, void* out, int32_t ldo, const void* kv_layer,
                                    const int32_t* block_tables, int32_t max_blocks, const int32_t* work, int32_t num_work,
                                    int32_t q_heads, int32_t kv_heads, float scale, int32_t split, void* stream) {
  return b200_op_paged_attn_decode_split_hd(q, ldq, out, ldo, kv_layer, block_tables, max_blocks, work, num_work, q_heads,
                                            kv_heads, scale, split, 128, stream);
}

int b200_op_paged_attn_decode_split_hd(const void* q, int32_t ldq, void* out, int32_t ldo, const void* kv_layer,
                                       const int32_t* block_tables, int32_t max_blocks, const int32_t* work, int32_t num_work,
                                       int32_t q_heads, int32_t kv_heads, float scale, int32_t split, int32_t head_dim,
                                       void* stream) {
  if (int rc = require_device()) return rc;
  if (split < 1 || split > 64 || num_work <= 0 || !attn_group_ok(q_heads, kv_heads) || !attn_head_dim_ok(head_dim)) {
    set_error("b200_op_paged_attn_decode_split: bad arguments");
    return B200_ERR_INVALID;
  }
  static float* ws = nullptr;
  static size_t ws_bytes = 0;
  static std::mutex mu;
  std::lock_guard<std::mutex> lk(mu);
  const size_t need = attn_split_ws_bytes(num_work, q_heads, split, kDecodeRows / (q_heads / kv_heads), head_dim);
  if (need > ws_bytes) {
    cudaDeviceSynchronize();
    if (ws) cudaFree(ws);
    ws = nullptr;
    ws_bytes = 0;
    if (cudaMalloc(&ws, need) != cudaSuccess) { set_error("workspace allocation failed"); return B200_ERR_OOM; }
    ws_bytes = need;
  }
  int rc = paged_attention(q, ldq, out, ldo, kv_layer, block_tables, max_blocks, reinterpret_cast<const AttnWork*>(work), num_work,
                           q_heads, kv_heads, scale, static_cast<cudaStream_t>(stream), ws, split, head_dim);
  return rc ? cuda_fail("paged_attention(split)", rc) : 0;
}

int b200_op_paged_attn_prefill_tc(const void* qkv, int32_t q_rows, int32_t ldq, void* out, int32_t ldo, const void* kv_layer,
                                  const int32_t* block_tables, int32_t max_blocks, const int32_t* work, int32_t num_work,
                                  int32_t q_heads, int32_t kv_heads, float scale, void* stream) {
  return b200_op_paged_attn_prefill_tc_hd(qkv, q_rows, ldq, out, ldo, kv_layer, block_tables, max_blocks, work, num_work, q_heads,
                                          kv_heads, scale, 128, stream);
}

int b200_op_paged_attn_prefill_tc_hd(const void* qkv, int32_t q_rows, int32_t ldq, void* out, int32_t ldo, const void* kv_layer,
                                     const int32_t* block_tables, int32_t max_blocks, const int32_t* work, int32_t num_work,
                                     int32_t q_heads, int32_t kv_heads, float scale, int32_t head_dim, void* stream) {
  if (int rc = require_device()) return rc;
  int rc = paged_attention_prefill_tc(qkv, q_rows, ldq, out, ldo, kv_layer, block_tables, max_blocks,
                                      reinterpret_cast<const AttnWork*>(work), num_work, q_heads, kv_heads, scale,
                                      static_cast<cudaStream_t>(stream), head_dim);
  return rc ? cuda_fail("paged_attention_prefill_tc", rc) : 0;
}

int b200_op_kv_copy_blocks(void* kv, int32_t num_layers, int64_t layer_stride_bytes, int64_t block_bytes, const int32_t* src,
                           const int32_t* dst, int32_t n_pairs, void* stream) {
  if (int rc = require_device()) return rc;
  int rc = kv_copy_blocks(kv, num_layers, layer_stride_bytes, block_bytes, src, dst, n_pairs, static_cast<cudaStream_t>(stream));
  if (rc == -1) {
    set_error("b200_op_kv_copy_blocks: bad arguments (n_pairs=%d num_layers=%d block_bytes=%lld layer_stride_bytes=%lld; "
              "16-byte multiples and a 16-byte aligned kv required)", n_pairs, num_layers, static_cast<long long>(block_bytes),
              static_cast<long long>(layer_stride_bytes));
    return B200_ERR_INVALID;
  }
  return rc ? cuda_fail("kv_copy_blocks", rc) : 0;
}

int b200_op_init_uniform(void* p, uint64_t n, uint32_t seed, float scale, float offset, void* stream) {
  if (int rc = require_device()) return rc;
  int rc = init_uniform(p, n, seed, scale, offset, static_cast<cudaStream_t>(stream));
  return rc ? cuda_fail("init_uniform", rc) : 0;
}

}  // extern "C"
