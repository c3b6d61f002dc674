// Sparse logits edits for vLLM V1's logits processors (vllm/v1/sample/sampler.py apply_logits_processors,
// v1/sample/logits_processor/builtin.py, model_executor/layers/utils.py apply_penalties), in its order and in fp32:
//   l = float(bf16 logit);  l += bias  (logit_bias);  l = -inf  (a stop id while fewer than min_tokens tokens exist);
//   l *= (l > 0 ? 1/r : r)  (repetition r, for tokens in the prompt or the output; 1/r is rounded to fp32);
//   l -= fp32(frequency * count);  l -= presence * (count > 0);
// and the result is written back rounded to bf16 (RNE), so the token selection kernels read the row they always read.
// Only the entries a request's record list names are touched: for every other token vLLM's arithmetic is the identity.
//
// The lists stay on the device for as long as the request runs.  penalize_rows (one CTA per edited row) edits in place
// and saves the raw bf16 values; after the token selection penalize_restore puts them back, so logprobs and the kept
// logits see the raw row; penalize_update then adds each sampled token to its list, which is sorted by id: a binary
// search, then a count + 1 or a shift of the records above it.  Each costs O(list) per row, and none depends on the batch.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <atomic>
#include <map>

#include "kernels.h"
#include "launch.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ float bf16_bits_to_f32(uint32_t b) { return __uint_as_float(b << 16); }

__global__ void __launch_bounds__(kThreads) penalize_kernel(uint16_t* __restrict__ logits, int ld,
                                                            const PenaltyRow* __restrict__ rows,
                                                            const PenaltyRec* __restrict__ recs,
                                                            const int* __restrict__ lens, int cap,
                                                            uint16_t* __restrict__ save) {
  griddep_enter();
  const PenaltyRow P = rows[blockIdx.x];
  uint16_t* row = logits + static_cast<size_t>(P.row) * ld;
  const PenaltyRec* list = recs + static_cast<size_t>(P.slot) * cap;
  uint16_t* sv = save + static_cast<size_t>(blockIdx.x) * cap;
  const int n = min(lens[P.slot], cap);
  const bool stops_on = P.n_generated < P.min_tokens;
  const float r = P.repetition, inv_r = __fdiv_rn(1.0f, P.repetition);
  for (int i = threadIdx.x; i < n; i += kThreads) {
    const PenaltyRec e = list[i];
    const uint16_t raw = row[e.id];
    sv[i] = raw;
    float l = bf16_bits_to_f32(raw);
    if (e.flags & kPenBias) l = __fadd_rn(l, e.bias);
    if ((e.flags & kPenStop) && stops_on) l = -INFINITY;
    if ((e.flags & kPenPrompt) || e.count > 0) l = __fmul_rn(l, l > 0.f ? inv_r : r);
    l = __fsub_rn(l, __fmul_rn(P.frequency, static_cast<float>(e.count)));
    l = __fsub_rn(l, __fmul_rn(P.presence, e.count > 0 ? 1.0f : 0.0f));
    row[e.id] = __bfloat16_as_ushort(__float2bfloat16_rn(l));
  }
}

__global__ void __launch_bounds__(kThreads) restore_kernel(uint16_t* __restrict__ logits, int ld,
                                                           const PenaltyRow* __restrict__ rows,
                                                           const PenaltyRec* __restrict__ recs,
                                                           const int* __restrict__ lens, int cap,
                                                           const uint16_t* __restrict__ save) {
  griddep_enter();
  const PenaltyRow P = rows[blockIdx.x];
  uint16_t* row = logits + static_cast<size_t>(P.row) * ld;
  const PenaltyRec* list = recs + static_cast<size_t>(P.slot) * cap;
  const uint16_t* sv = save + static_cast<size_t>(blockIdx.x) * cap;
  const int n = min(lens[P.slot], cap);
  for (int i = threadIdx.x; i < n; i += kThreads) row[list[i].id] = sv[i];
}

__global__ void __launch_bounds__(kThreads) update_kernel(const PenaltyRow* __restrict__ rows,
                                                          const int* __restrict__ sampled, PenaltyRec* __restrict__ recs,
                                                          int* __restrict__ lens, int cap) {
  __shared__ int s_pos, s_found;
  griddep_enter();
  const PenaltyRow P = rows[blockIdx.x];
  if (!P.history) return;
  PenaltyRec* list = recs + static_cast<size_t>(P.slot) * cap;
  const int n = lens[P.slot];
  const int t = sampled[P.row];
  if (threadIdx.x == 0) {
    int lo = 0, hi = n;   // first record with id >= t
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (list[mid].id < t) lo = mid + 1;
      else hi = mid;
    }
    s_pos = lo;
    s_found = lo < n && list[lo].id == t;
    if (s_found) ++list[lo].count;
  }
  __syncthreads();
  if (s_found || n >= cap) return;   // a list holds every distinct id it can meet: n < cap here
  const int pos = s_pos;
  // shift [pos, n) up by one, highest chunk first: each chunk is read before the chunk below overwrites its first entry
  for (int hi = n; hi > pos; hi -= kThreads) {
    const int i = hi - kThreads + static_cast<int>(threadIdx.x);
    PenaltyRec e;
    const bool mine = i >= pos && i < hi;
    if (mine) e = list[i];
    __syncthreads();
    if (mine) list[i + 1] = e;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    list[pos] = PenaltyRec{t, 1, 0.f, 0u};
    lens[P.slot] = n + 1;
  }
}

}  // namespace

void penalty_records(const int32_t* prompt, int n_prompt, const int32_t* output, int n_output, bool history,
                     const int32_t* bias_ids, const float* bias_values, int n_bias, const int32_t* stops, int n_stops,
                     std::vector<PenaltyRec>* out) {
  std::map<int, PenaltyRec> m;
  auto at = [&](int id) -> PenaltyRec& {
    auto it = m.find(id);
    if (it == m.end()) it = m.emplace(id, PenaltyRec{id, 0, 0.f, 0u}).first;
    return it->second;
  };
  if (history) {
    for (int i = 0; i < n_prompt; ++i) at(prompt[i]).flags |= kPenPrompt;
    for (int i = 0; i < n_output; ++i) ++at(output[i]).count;
  }
  for (int i = 0; i < n_bias; ++i) {   // a later entry for the same id replaces an earlier one, as in a JSON object
    PenaltyRec& r = at(bias_ids[i]);
    r.flags |= kPenBias;
    r.bias = std::min(100.0f, std::max(-100.0f, bias_values[i]));
  }
  for (int i = 0; i < n_stops; ++i) at(stops[i]).flags |= kPenStop;
  out->clear();
  out->reserve(m.size());
  for (auto& kv : m) out->push_back(kv.second);
}

int penalize_rows(void* logits, int ld, const PenaltyRow* rows, int n, const PenaltyRec* recs, const int* lens, int cap,
                  uint16_t* save, cudaStream_t st) {
  if (n <= 0) return 0;
  if (ld < 1 || cap < 1) return -1;
  launch_pdl(penalize_kernel, dim3(n), dim3(kThreads), 0, st, static_cast<uint16_t*>(logits), ld, rows, recs, lens, cap, save);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int penalize_restore(void* logits, int ld, const PenaltyRow* rows, int n, const PenaltyRec* recs, const int* lens, int cap,
                     const uint16_t* save, cudaStream_t st) {
  if (n <= 0) return 0;
  if (ld < 1 || cap < 1) return -1;
  launch_pdl(restore_kernel, dim3(n), dim3(kThreads), 0, st, static_cast<uint16_t*>(logits), ld, rows, recs, lens, cap, save);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int penalize_update(const PenaltyRow* rows, int n, const int* sampled, PenaltyRec* recs, int* lens, int cap, cudaStream_t st) {
  if (n <= 0) return 0;
  if (cap < 1) return -1;
  launch_pdl(update_kernel, dim3(n), dim3(kThreads), 0, st, rows, sampled, recs, lens, cap);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

}  // namespace b200
