// Last-token pooling of a pooling runner's step (vLLM's LastPool + PoolerNormalize, pooler/ in vLLM 0.22): the final RMSNorm
// of each pooled row, then, per row, its L2 normalisation in fp32 (torch.nn.functional.normalize: x / max(||x||, 1e-12)),
// or, on a score head (a *ForSequenceClassification checkpoint), its fp32 score logits and their activation.
#include <cuda_bf16.h>
#include <math.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"
#include "launch.h"
#include "ptx.cuh"

namespace b200 {

namespace {

union Vec8 {
  uint4 u;
  __nv_bfloat16 h[8];
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The block-wide sum of one float per thread in a fixed order: xor-shuffle within each warp, then the warp sums in warp
// order through shared memory, again by xor-shuffle.  red: 32 floats of shared memory, free on entry.
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) red[0] = t;
  }
  __syncthreads();
  return red[0];
}

// The final RMSNorm of one row, shared by pool_rows_kernel and score_rows_kernel.  Row r of x (+ residual, added in bf16
// as the fused-add RMSNorm does, residual not written back) is normed with w exactly as rmsnorm_kernel<VPT> in
// elementwise.cu does with the same block size (same per-thread order, same reduction, same rounding points), so the bf16
// normed row is bit-identical to the gathered final norm.  xin and res are the row of x and of residual (null: none).
// norm_row_prologue issues the loads that do not depend on the previous kernel (the caller runs it before
// griddep_enter()); norm_row then leaves the bf16 normed values, widened to fp32, in y.  red: 32 floats of shared memory,
// free on entry; red[0] is read by every thread on return.
template <int VPT>
__device__ __forceinline__ void norm_row_prologue(const uint4* res, const __nv_bfloat16* __restrict__ w, Vec8 (&rb)[VPT],
                                                  Vec8 (&ww)[VPT]) {
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int idx = threadIdx.x + i * blockDim.x;
    ww[i].u = __ldg(reinterpret_cast<const uint4*>(w) + idx);
    if (res) rb[i].u = res[idx];
  }
}

template <int VPT>
__device__ __forceinline__ void norm_row(const uint4* xin, const uint4* res, int H, float eps, const Vec8 (&rb)[VPT],
                                         const Vec8 (&ww)[VPT], float (&y)[VPT][8], float* red) {
  float v[VPT][8];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    Vec8 xa;
    xa.u = xin[threadIdx.x + i * blockDim.x];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float f = __bfloat162float(xa.h[j]);
      v[i][j] = res ? __bfloat162float(__float2bfloat16_rn(f + __bfloat162float(rb[i].h[j]))) : f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) ss += v[i][j] * v[i][j];
  }
  const float inv = rsqrtf(block_sum(ss, red) / static_cast<float>(H) + eps);
#pragma unroll
  for (int i = 0; i < VPT; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const __nv_bfloat16 nb = __float2bfloat16_rn(v[i][j] * inv);
      y[i][j] = __bfloat162float(__float2bfloat16_rn(__bfloat162float(nb) * __bfloat162float(ww[i].h[j])));
    }
}

// One CTA per pooled row s: row r = row_index[s] of x (+ residual), normed by norm_row.  flags[s] != 0: out[s] = y /
// max(sqrt(sum y^2), 1e-12) with the sum of squares of the bf16 values y taken in fp32 in a fixed order (each thread's
// values in visit order, then block_sum), IEEE sqrt and division; else out[s] = y.
template <int VPT>
__global__ void pool_rows_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ residual,
                                 const __nv_bfloat16* __restrict__ w, const int* __restrict__ row_index,
                                 const int* __restrict__ flags, int H, float eps, float* __restrict__ out) {
  const int s = blockIdx.x;
  const int r = row_index[s];
  const bool normalize = flags[s] != 0;
  const uint4* xin = reinterpret_cast<const uint4*>(x + static_cast<size_t>(r) * H);
  const uint4* res = residual ? reinterpret_cast<const uint4*>(residual + static_cast<size_t>(r) * H) : nullptr;
  Vec8 rb[VPT], ww[VPT];
  norm_row_prologue<VPT>(res, w, rb, ww);
  griddep_enter();
  __shared__ float red[32];
  float y[VPT][8];
  norm_row<VPT>(xin, res, H, eps, rb, ww, y, red);
  float yy = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) yy = __fmaf_rn(y[i][j], y[i][j], yy);
  if (normalize) {   // uniform across the CTA: one row per CTA
    __syncthreads();   // red[0] has been read by every thread
    const float denom = fmaxf(__fsqrt_rn(block_sum(yy, red)), 1e-12f);
#pragma unroll
    for (int i = 0; i < VPT; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) y[i][j] = __fdiv_rn(y[i][j], denom);
  }
  float4* o4 = reinterpret_cast<float4*>(out + static_cast<size_t>(s) * H);
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int idx = threadIdx.x + i * blockDim.x;
    o4[2 * idx] = make_float4(y[i][0], y[i][1], y[i][2], y[i][3]);
    o4[2 * idx + 1] = make_float4(y[i][4], y[i][5], y[i][6], y[i][7]);
  }
}

// One CTA per pooled row s of a score head (vLLM's LastPool -> fp32 score linear -> PoolerClassify): the row normed by
// norm_row, then logit[l] = sum_h y_h * sw[l, h] in fp32 for l < L (y the bf16 normed values, sw the bf16 score weight
// [L, H], both widened): per label, each thread's FMAs in visit order (its vectors i, their elements j), then warp_sum,
// then the warp sums added one after another in warp order.  flags[s] != 0 applies the activation (act: 1 sigmoid
// 1 / (1 + expf(-x)), 2 softmax: expf(x - max), summed in label order, then divided; 3 none) in warp 0, lane l holding
// logit l; else out[s, l] = logit[l].  The score weights are not registers' worth at L = 32 (up to 512 KB), so the CTA's
// slice of them is prefetched into L2 before griddep_enter() and read with __ldg after.
template <int VPT>
__global__ void score_rows_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ residual,
                                  const __nv_bfloat16* __restrict__ w, const __nv_bfloat16* __restrict__ sw,
                                  const int* __restrict__ row_index, const int* __restrict__ flags, int H, int L, int act,
                                  float eps, float* __restrict__ out) {
  const int s = blockIdx.x;
  const int r = row_index[s];
  const bool activate = flags[s] != 0;
  const uint4* xin = reinterpret_cast<const uint4*>(x + static_cast<size_t>(r) * H);
  const uint4* res = residual ? reinterpret_cast<const uint4*>(residual + static_cast<size_t>(r) * H) : nullptr;
  Vec8 rb[VPT], ww[VPT];
  norm_row_prologue<VPT>(res, w, rb, ww);
  for (int l = 0; l < L; ++l)
#pragma unroll
    for (int i = 0; i < VPT; ++i)
      asm volatile("prefetch.global.L2::evict_last [%0];" ::"l"(reinterpret_cast<const uint4*>(sw + static_cast<size_t>(l) * H) +
                                                                  threadIdx.x + i * blockDim.x));
  griddep_enter();
  __shared__ float red[32];
  __shared__ float part[32][kMaxScoreLabels];   // [warp][label]
  float y[VPT][8];
  norm_row<VPT>(xin, res, H, eps, rb, ww, y, red);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int l = 0; l < L; ++l) {
    const uint4* wl = reinterpret_cast<const uint4*>(sw + static_cast<size_t>(l) * H);
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      Vec8 wv;
      wv.u = __ldg(wl + threadIdx.x + i * blockDim.x);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc = __fmaf_rn(y[i][j], __bfloat162float(wv.h[j]), acc);
    }
    acc = warp_sum(acc);
    if (lane == 0) part[warp][l] = acc;
  }
  __syncthreads();
  if (warp != 0) return;
  float logit = 0.f;
  if (lane < L) {
    logit = part[0][lane];
    for (int k = 1; k < nwarps; ++k) logit += part[k][lane];
  }
  float o = logit;
  if (activate && act == kScoreSigmoid) {
    o = __fdiv_rn(1.f, 1.f + expf(-logit));
  } else if (activate && act == kScoreSoftmax) {
    float m = lane < L ? logit : -INFINITY;
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, k));
    const float e = lane < L ? expf(logit - m) : 0.f;
    red[lane] = e;   // every thread has read red[0] in norm_row before the __syncthreads above
    __syncwarp();
    float sum = red[0];
    for (int k = 1; k < L; ++k) sum += red[k];
    o = __fdiv_rn(e, sum);
  }
  if (lane < L) out[static_cast<size_t>(s) * L + lane] = o;
}

}  // namespace

int pool_rows(const void* x, const void* residual, const void* w, const int* row_index, const int* flags, int rows, int H,
              float eps, float* out, cudaStream_t st) {
  if (rows <= 0) return 0;
  if (H % 256 || H > 8192 || !row_index || !flags) return -1;
  const __nv_bfloat16* xx = static_cast<const __nv_bfloat16*>(x);
  const __nv_bfloat16* rr = static_cast<const __nv_bfloat16*>(residual);
  const __nv_bfloat16* ww = static_cast<const __nv_bfloat16*>(w);
  const int vecs = H / 8;
  // rmsnorm()'s choice of block size for the same rows and H: the normed row depends on the reduction order
  if (rows < 512 || vecs % 256 != 0) {
    launch_pdl(pool_rows_kernel<1>, dim3(rows), dim3(vecs), 0, st, xx, rr, ww, row_index, flags, H, eps, out);
  } else {
    switch (vecs / 256) {
      case 1: launch_pdl(pool_rows_kernel<1>, dim3(rows), dim3(256), 0, st, xx, rr, ww, row_index, flags, H, eps, out); break;
      case 2: launch_pdl(pool_rows_kernel<2>, dim3(rows), dim3(256), 0, st, xx, rr, ww, row_index, flags, H, eps, out); break;
      case 3: launch_pdl(pool_rows_kernel<3>, dim3(rows), dim3(256), 0, st, xx, rr, ww, row_index, flags, H, eps, out); break;
      default: launch_pdl(pool_rows_kernel<4>, dim3(rows), dim3(256), 0, st, xx, rr, ww, row_index, flags, H, eps, out); break;
    }
  }
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int score_rows(const void* x, const void* residual, const void* w, const void* sw, const int* row_index, const int* flags,
               int rows, int H, int L, int act, float eps, float* out, cudaStream_t st) {
  if (rows <= 0) return 0;
  if (H % 256 || H > 8192 || L < 1 || L > kMaxScoreLabels || act < kScoreSigmoid || act > kScoreNone || !sw || !row_index ||
      !flags)
    return -1;
  const __nv_bfloat16* xx = static_cast<const __nv_bfloat16*>(x);
  const __nv_bfloat16* rr = static_cast<const __nv_bfloat16*>(residual);
  const __nv_bfloat16* ww = static_cast<const __nv_bfloat16*>(w);
  const __nv_bfloat16* ss = static_cast<const __nv_bfloat16*>(sw);
  const int vecs = H / 8;
  // pool_rows' (and so rmsnorm()'s) choice of block size: the normed row depends on the reduction order
  if (rows < 512 || vecs % 256 != 0) {
    launch_pdl(score_rows_kernel<1>, dim3(rows), dim3(vecs), 0, st, xx, rr, ww, ss, row_index, flags, H, L, act, eps, out);
  } else {
    switch (vecs / 256) {
      case 1: launch_pdl(score_rows_kernel<1>, dim3(rows), dim3(256), 0, st, xx, rr, ww, ss, row_index, flags, H, L, act, eps, out); break;
      case 2: launch_pdl(score_rows_kernel<2>, dim3(rows), dim3(256), 0, st, xx, rr, ww, ss, row_index, flags, H, L, act, eps, out); break;
      case 3: launch_pdl(score_rows_kernel<3>, dim3(rows), dim3(256), 0, st, xx, rr, ww, ss, row_index, flags, H, L, act, eps, out); break;
      default: launch_pdl(score_rows_kernel<4>, dim3(rows), dim3(256), 0, st, xx, rr, ww, ss, row_index, flags, H, L, act, eps, out); break;
    }
  }
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

}  // namespace b200
