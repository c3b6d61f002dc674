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

int b200_op_rope_kvwrite(void* qkv, const int32_t* positions, const int32_t* slots, const void* cos_sin,
                         void* kv_layer, int32_t T, int32_t q_heads, int32_t kv_heads, int32_t max_pos,
                         void* stream) {
  if (int rc = require_device()) return rc;
  int rc = rope_kv_write(qkv, positions, slots, cos_sin, kv_layer, T, q_heads, kv_heads, max_pos,
                         static_cast<cudaStream_t>(stream));
  return rc ? cuda_fail("rope_kv_write", rc) : 0;
}

int b200_op_silu_mul(const void* gate_up, void* out, int32_t T, int32_t I, void* stream) {
  if (int rc = require_device()) return rc;
  int rc = silu_mul(gate_up, out, T, I, static_cast<cudaStream_t>(stream));
  return rc ? cuda_fail("silu_mul", rc) : 0;
}

int b200_op_argmax(const void* logits, int32_t* out, int32_t S, int32_t V, int32_t ld, void* stream) {
  if (int rc = require_device()) return rc;
  int rc = argmax_rows(logits, out, S, V, ld, static_cast<cudaStream_t>(stream));
  return rc ? cuda_fail("argmax_rows", rc) : 0;
}

int b200_op_paged_attn(const void* q, int32_t ldq, void* out, int32_t ldo, const void* kv_layer,
                       const int32_t* block_tables, int32_t max_blocks, const int32_t* work, int32_t num_work,
                       int32_t q_heads, int32_t kv_heads, float scale, int32_t decode, void* stream) {
  if (int rc = require_device()) return rc;
  static_assert(sizeof(AttnWork) == 16, "AttnWork is int32[4] on the wire");
  int rc = paged_attention(q, ldq, out, ldo, kv_layer, block_tables, max_blocks,
                           reinterpret_cast<const AttnWork*>(work), num_work, q_heads, kv_heads, scale, decode,
                           static_cast<cudaStream_t>(stream));
  return rc ? cuda_fail("paged_attention", rc) : 0;
}

int b200_op_paged_attn_decode_split(const void* q, int32_t ldq, void* out, int32_t ldo, const void* kv_layer,
                                    const int32_t* block_tables, int32_t max_blocks, const int32_t* work, int32_t num_work,
                                    int32_t q_heads, int32_t kv_heads, float scale, int32_t split, void* stream) {
  if (int rc = require_device()) return rc;
  if (split < 1 || split > 64 || num_work <= 0) { set_error("b200_op_paged_attn_decode_split: bad arguments"); return B200_ERR_INVALID; }
  static float* ws = nullptr;
  static size_t ws_bytes = 0;
  static std::mutex mu;
  std::lock_guard<std::mutex> lk(mu);
  const size_t need = attn_split_ws_bytes(num_work, kv_heads, split);
  if (need > ws_bytes) {
    cudaDeviceSynchronize();
    if (ws) cudaFree(ws);
    ws = nullptr;
    ws_bytes = 0;
    if (cudaMalloc(&ws, need) != cudaSuccess) { set_error("workspace allocation failed"); return B200_ERR_OOM; }
    ws_bytes = need;
  }
  int rc = paged_attention(q, ldq, out, ldo, kv_layer, block_tables, max_blocks, reinterpret_cast<const AttnWork*>(work), num_work,
                           q_heads, kv_heads, scale, 1, static_cast<cudaStream_t>(stream), ws, split);
  return rc ? cuda_fail("paged_attention(split)", rc) : 0;
}

int b200_op_paged_attn_prefill_tc(const void* qkv, int32_t q_rows, int32_t ldq, void* out, int32_t ldo, const void* kv_layer,
                                  const int32_t* block_tables, int32_t max_blocks, const int32_t* work, int32_t num_work,
                                  int32_t q_heads, int32_t kv_heads, float scale, void* stream) {
  if (int rc = require_device()) return rc;
  int rc = paged_attention_prefill_tc(qkv, q_rows, ldq, out, ldo, kv_layer, block_tables, max_blocks,
                                      reinterpret_cast<const AttnWork*>(work), num_work, q_heads, kv_heads, scale,
                                      static_cast<cudaStream_t>(stream));
  return rc ? cuda_fail("paged_attention_prefill_tc", rc) : 0;
}

int b200_op_init_uniform(void* p, uint64_t n, uint32_t seed, float scale, float offset, void* stream) {
  if (int rc = require_device()) return rc;
  int rc = init_uniform(p, n, seed, scale, offset, static_cast<cudaStream_t>(stream));
  return rc ? cuda_fail("init_uniform", rc) : 0;
}

}  // extern "C"
