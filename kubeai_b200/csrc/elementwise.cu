// Bandwidth-bound per-step ops of the Llama forward (SURVEY.md §8a K2, K3, K5, K9-act, K11-argmax).
// Rounding points follow the reference backend so greedy tokens match:
//   RMSNorm:              vllm/ir/ops/layernorm.py:9-21;  fused add: vllm/_custom_ops.py:323-327 (_C op: bf16 sum, norm of it)
//   RoPE (neox):          vllm/model_executor/layers/rotary_embedding/base.py:140-198 (bf16 cos/sin cache)
//   SiLU*mul:             vllm/model_executor/layers/activation.py:138-148 (silu in fp32, rounded, then * up)
//   greedy sampling:      vllm/v1/sample/sampler.py:91,235-236 (argmax, lowest index wins ties)
// All kernels: 16-byte vectorised, coalesced, one warp-shuffle + one smem hop for reductions.
#include <cuda_bf16.h>
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

__device__ __forceinline__ void unpack8_bf16(const uint4& u, float (&o)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = __bfloat1622float2(h[j]);
    o[2 * j] = f.x;
    o[2 * j + 1] = f.y;
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------ embedding gather
__global__ void embed_kernel(const __nv_bfloat16* __restrict__ table, const int* __restrict__ ids,
                             __nv_bfloat16* __restrict__ out, int H, int vocab) {
  griddep_enter();
  const int t = blockIdx.x;
  int id = ids[t];
  if (id < 0 || id >= vocab) id = 0;
  const uint4* src = reinterpret_cast<const uint4*>(table + static_cast<size_t>(id) * H);
  uint4* dst = reinterpret_cast<uint4*>(out + static_cast<size_t>(t) * H);
  for (int i = threadIdx.x; i < H / 8; i += blockDim.x) dst[i] = __ldg(src + i);
}

// ------------------------------------------------------------------ (fused add) RMSNorm
// x: [rows_in, H] GEMM output (or hidden), residual: in/out [rows_in, H] or null.
// row_index (optional): output row s reads input row row_index[s]; residual is then NOT written back.
template <int VPT>  // uint4 vectors per thread (H = VPT * 8 * blockDim)
__global__ void rmsnorm_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ residual,
                               const __nv_bfloat16* __restrict__ w, __nv_bfloat16* __restrict__ out,
                               const int* __restrict__ row_index, int H, float eps) {
  // ---- before the dependency wait (ptx.cuh griddep_enter): everything that does not come from the producer GEMM —
  // the row index (step input), the residual (written four or more launches upstream) and the norm weight
  const int s = blockIdx.x;
  const int r = row_index ? row_index[s] : s;
  const uint4* xin = reinterpret_cast<const uint4*>(x + static_cast<size_t>(r) * H);
  uint4* res = residual ? reinterpret_cast<uint4*>(residual + static_cast<size_t>(r) * H) : nullptr;
  float v[VPT][8];
  float ss = 0.f;
  Vec8 rb[VPT], ww[VPT];
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int idx = threadIdx.x + i * blockDim.x;
    ww[i].u = __ldg(reinterpret_cast<const uint4*>(w) + idx);
    if (res) rb[i].u = res[idx];
  }
  griddep_enter();
  float xa[VPT][8];
  uint4 raw[VPT];
#pragma unroll
  for (int i = 0; i < VPT; ++i) raw[i] = xin[threadIdx.x + i * blockDim.x];
#pragma unroll
  for (int i = 0; i < VPT; ++i) unpack8_bf16(raw[i], xa[i]);
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int idx = threadIdx.x + i * blockDim.x;
    if (res) {
      Vec8 o;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        // residual += x in bf16; variance and normalisation use the ROUNDED sum (vLLM _C fused_add_rms_norm, HF
        // modeling_llama.py:325 + :62-67) — the GEMM residual-add epilogue stores exactly this bf16 sum (gemm_wgmma.cu)
        o.h[j] = __float2bfloat16_rn(xa[i][j] + __bfloat162float(rb[i].h[j]));
        v[i][j] = __bfloat162float(o.h[j]);
      }
      if (!row_index) res[idx] = o.u;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[i][j] = xa[i][j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) ss += v[i][j] * v[i][j];
  }
  __shared__ float red[32];
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) red[0] = t;
  }
  __syncthreads();
  const float inv = rsqrtf(red[0] / static_cast<float>(H) + eps);
  uint4* o4 = reinterpret_cast<uint4*>(out + static_cast<size_t>(s) * H);
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int idx = threadIdx.x + i * blockDim.x;
    Vec8 o;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      // normalised value rounded to bf16 BEFORE the weight multiply (layernorm.py:19)
      __nv_bfloat16 nb = __float2bfloat16_rn(v[i][j] * inv);
      o.h[j] = __float2bfloat16_rn(__bfloat162float(nb) * __bfloat162float(ww[i].h[j]));
    }
    o4[idx] = o.u;
  }
}

// ------------------------------------------------------------------ RoPE (neox) + paged KV write
// qkv: [T, (Hq + 2*Hkv) * D], q and k rotated in place; k,v rows scattered to the paged cache; D = 64 or 128
// kv layout per layer: [block][2][Hkv][16][D]  (head-major inside a page: one (page,head) = 32 * D bytes contiguous)
template <int D>
__global__ void rope_kv_kernel(__nv_bfloat16* __restrict__ qkv, const int* __restrict__ positions,
                               const int* __restrict__ slots, const __nv_bfloat16* __restrict__ cos_sin,
                               __nv_bfloat16* __restrict__ kv, int Hq, int Hkv, int max_pos) {
  constexpr int HALF = D / 2, RT = HALF / 8, VT = D / 8;  // rotation / V-copy tasks per head
  constexpr int RTL = D == 128 ? 3 : 2, VTL = RTL + 1;     // their log2
  const int t = blockIdx.x;
  // ---- before the dependency wait: step inputs (positions, slots) and cos/sin rows.  The first task of every thread is
  // prepared here; later tasks (only when blockDim < tasks) load theirs afterwards.
  int pos = positions[t];
  pos = pos < 0 ? 0 : (pos >= max_pos ? max_pos - 1 : pos);
  const int slot = slots[t];
  const int ld = (Hq + 2 * Hkv) * D;
  __nv_bfloat16* row = qkv + static_cast<size_t>(t) * ld;
  const __nv_bfloat16* cs = cos_sin + static_cast<size_t>(pos) * D;  // cos[0:D/2] | sin[0:D/2]
  const int blk = slot >> 4, off = slot & 15;
  const size_t page_stride = static_cast<size_t>(Hkv) * 16 * D;  // elements per K (or V) page over all heads
  __nv_bfloat16* kbase = kv + static_cast<size_t>(blk) * 2 * page_stride;
  __nv_bfloat16* vbase = kbase + page_stride;

  const int rot_tasks = (Hq + Hkv) * RT;  // 8 elements of x1 (and the matching 8 of x2) per task
  const int v_tasks = Hkv * VT;
  Vec8 co0, si0;
  if (static_cast<int>(threadIdx.x) < rot_tasks) {
    const int c = threadIdx.x & (RT - 1);
    co0.u = __ldg(reinterpret_cast<const uint4*>(cs + c * 8));
    si0.u = __ldg(reinterpret_cast<const uint4*>(cs + HALF + c * 8));
  }
  griddep_enter();
  // rotation tasks and V-copy tasks share one index space so that a 512-thread CTA gives every thread one task
  for (int task = threadIdx.x; task < rot_tasks; task += blockDim.x) {
    const int head = task >> RTL, c = task & (RT - 1);
    const bool first = task == static_cast<int>(threadIdx.x);
    __nv_bfloat16* hp = row + head * D;
    Vec8 x1, x2, co, si, o1, o2;
    x1.u = *reinterpret_cast<const uint4*>(hp + c * 8);
    x2.u = *reinterpret_cast<const uint4*>(hp + HALF + c * 8);
    if (first) {
      co = co0;
      si = si0;
    } else {
      co.u = __ldg(reinterpret_cast<const uint4*>(cs + c * 8));
      si.u = __ldg(reinterpret_cast<const uint4*>(cs + HALF + c * 8));
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float a = __bfloat162float(x1.h[j]), b = __bfloat162float(x2.h[j]);
      const float cc = __bfloat162float(co.h[j]), sn = __bfloat162float(si.h[j]);
      // every bf16 op rounds, exactly like the reference kernel's scalar_t arithmetic
      // (x * cos - y * sin with c10::BFloat16 operators == rotary_embedding/common.py:173-174)
      const float ac = __bfloat162float(__float2bfloat16_rn(__fmul_rn(a, cc)));
      const float bs = __bfloat162float(__float2bfloat16_rn(__fmul_rn(b, sn)));
      const float bc = __bfloat162float(__float2bfloat16_rn(__fmul_rn(b, cc)));
      const float as = __bfloat162float(__float2bfloat16_rn(__fmul_rn(a, sn)));
      o1.h[j] = __float2bfloat16_rn(ac - bs);
      o2.h[j] = __float2bfloat16_rn(bc + as);
    }
    *reinterpret_cast<uint4*>(hp + c * 8) = o1.u;
    *reinterpret_cast<uint4*>(hp + HALF + c * 8) = o2.u;
    if (head >= Hq && slot >= 0) {
      __nv_bfloat16* dst = kbase + (static_cast<size_t>(head - Hq) * 16 + off) * D;
      *reinterpret_cast<uint4*>(dst + c * 8) = o1.u;
      *reinterpret_cast<uint4*>(dst + HALF + c * 8) = o2.u;
    }
  }
  if (slot >= 0) {
    const __nv_bfloat16* vrow = row + (Hq + Hkv) * D;
    // start the V tasks where the rotation tasks ended so idle threads of the first pass take them
    for (int task = static_cast<int>((threadIdx.x + blockDim.x - rot_tasks % blockDim.x) % blockDim.x); task < v_tasks;
         task += blockDim.x) {
      const int head = task >> VTL, c = task & (VT - 1);
      *reinterpret_cast<uint4*>(vbase + (static_cast<size_t>(head) * 16 + off) * D + c * 8) =
          *reinterpret_cast<const uint4*>(vrow + head * D + c * 8);
    }
  }
}

// ------------------------------------------------------------------ SiLU(gate) * up
template <int VPT>  // uint4 output vectors per thread
// interleaved != 0: gate and up columns alternate in 64-column blocks (the engine's gate_up weight rows are laid out
// that way so that the decode GEMM's epilogue finds a gate row and its up row in one 128-row slab)
// Tokens are on gridDim.x (up to 2^31 - 1): gridDim.y stops at 65535, fewer than a large prefill step can hold.
__global__ void silu_mul_kernel(const __nv_bfloat16* __restrict__ gu, __nv_bfloat16* __restrict__ out, int I,
                                int ldi, int interleaved) {
  const int t = blockIdx.x;
  const uint4* g = reinterpret_cast<const uint4*>(gu + static_cast<size_t>(t) * ldi);
  uint4* o = reinterpret_cast<uint4*>(out + static_cast<size_t>(t) * I);
  const int nvec = I / 8;
  const int i0 = blockIdx.y * blockDim.x * VPT + threadIdx.x;
  float x[2 * VPT][8];  // gate vectors, then up vectors
  int n0[2 * VPT];
#pragma unroll
  for (int k = 0; k < VPT; ++k) {
    const int i = min(i0 + k * static_cast<int>(blockDim.x), nvec - 1);
    const int c = i * 8;
    n0[k] = interleaved ? ((c >> 6) << 7) + (c & 63) : c;
    n0[VPT + k] = interleaved ? n0[k] + 64 : I + c;
  }
  griddep_enter();
  uint4 raw[2 * VPT];
#pragma unroll
  for (int k = 0; k < VPT; ++k) {
    raw[k] = g[n0[k] >> 3];
    raw[VPT + k] = g[n0[VPT + k] >> 3];
  }
#pragma unroll
  for (int k = 0; k < 2 * VPT; ++k) unpack8_bf16(raw[k], x[k]);
#pragma unroll
  for (int k = 0; k < VPT; ++k) {
    const int i = i0 + k * blockDim.x;
    if (i >= nvec) continue;
    Vec8 r;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float gv = x[k][j];
      const __nv_bfloat16 s = silu_bf16(gv);
      r.h[j] = __float2bfloat16_rn(__bfloat162float(s) * x[VPT + k][j]);
    }
    o[i] = r.u;
  }
}

// ------------------------------------------------------------------ greedy argmax over bf16 logits
__global__ void argmax_kernel(const __nv_bfloat16* __restrict__ logits, int* __restrict__ out, int V, int ld) {
  griddep_enter();
  const int s = blockIdx.x;
  const __nv_bfloat16* row = logits + static_cast<size_t>(s) * ld;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  const int nvec = V / 8;
  const uint4* r4 = reinterpret_cast<const uint4*>(row);
  for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
    Vec8 a;
    a.u = r4[i];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float f = __bfloat162float(a.h[j]);
      const int idx = i * 8 + j;
      if (f > best || (f == best && idx < bi)) {
        best = f;
        bi = idx;
      }
    }
  }
  for (int idx = nvec * 8 + threadIdx.x; idx < V; idx += blockDim.x) {
    const float f = __bfloat162float(row[idx]);
    if (f > best || (f == best && idx < bi)) {
      best = f;
      bi = idx;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) {
      best = ob;
      bi = oi;
    }
  }
  __shared__ float sb[32];
  __shared__ int si[32];
  if ((threadIdx.x & 31) == 0) {
    sb[threadIdx.x >> 5] = best;
    si[threadIdx.x >> 5] = bi;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    const int nw = blockDim.x >> 5;
    best = threadIdx.x < nw ? sb[threadIdx.x] : -INFINITY;
    bi = threadIdx.x < nw ? si[threadIdx.x] : 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) {
        best = ob;
        bi = oi;
      }
    }
    if (threadIdx.x == 0) out[s] = bi == 0x7fffffff ? 0 : bi;
  }
}

// ------------------------------------------------------------------ gate_up row layout
// logical [gate rows 0..I) | up rows 0..I)]  <->  physical 64 gate rows, the 64 matching up rows, next 64 gate rows, ...
__global__ void permute_gu_kernel(__nv_bfloat16* __restrict__ dst, const __nv_bfloat16* __restrict__ src, int I, int H,
                                  int to_physical) {
  const int r = blockIdx.x;  // logical row
  const int i = r < I ? r : r - I;
  const int pr = ((i >> 6) << 7) + (r < I ? 0 : 64) + (i & 63);
  const uint4* s = reinterpret_cast<const uint4*>(src + static_cast<size_t>(to_physical ? r : pr) * H);
  uint4* d = reinterpret_cast<uint4*>(dst + static_cast<size_t>(to_physical ? pr : r) * H);
  for (int k = threadIdx.x; k < H / 8; k += blockDim.x) d[k] = s[k];
}

// ------------------------------------------------------------------ seeded weight init (device side)
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x7feb352du;
  x ^= x >> 15;
  x *= 0x846ca68bu;
  x ^= x >> 16;
  return x;
}
// value(i) = scale * u, u uniform in [-sqrt(3), sqrt(3)) (unit variance), from a counter hash.
__global__ void init_uniform_kernel(__nv_bfloat16* __restrict__ p, size_t n, uint32_t seed, float scale,
                                    float offset) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    uint32_t h = mix32(static_cast<uint32_t>(i) ^ mix32(seed + static_cast<uint32_t>(i >> 32) * 0x9e3779b9u));
    // explicit _rn intrinsics: no FMA contraction, so a numpy replica is bit-exact
    const float u = __fmul_rn(__fadd_rn(__fmul_rn(static_cast<float>(h >> 8), 1.0f / 16777216.0f), -0.5f),
                              3.4641016151f);
    p[i] = __float2bfloat16_rn(__fadd_rn(offset, __fmul_rn(scale, u)));
  }
}

}  // namespace

int embed_gather(const void* table, const int* ids, void* out, int T, int H, int vocab, cudaStream_t st) {
  if (T <= 0) return 0;
  if (H % 8) return -1;
  launch_pdl(embed_kernel, dim3(T), dim3(256), 0, st, static_cast<const __nv_bfloat16*>(table), ids,
             static_cast<__nv_bfloat16*>(out), H, vocab);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int rmsnorm(const void* x, void* residual, const void* w, void* out, const int* row_index, int rows, int H,
            float eps, cudaStream_t st) {
  if (rows <= 0) return 0;
  const __nv_bfloat16* xx = static_cast<const __nv_bfloat16*>(x);
  __nv_bfloat16* rr = static_cast<__nv_bfloat16*>(residual);
  const __nv_bfloat16* ww = static_cast<const __nv_bfloat16*>(w);
  __nv_bfloat16* oo = static_cast<__nv_bfloat16*>(out);
  if (H % 8) return -1;
  const int vecs = H / 8;
  // few rows (decode): one vector per thread so each row has the most loads in flight; many rows (prefill bursts):
  // 256-thread CTAs with 2-4 vectors each (measured: 24 us vs 29 us per call at T=2048, H=4096)
  if (vecs % 32 == 0 && vecs <= 1024 && (rows < 512 || vecs % 256 != 0 || vecs / 256 > 4)) {
    launch_pdl(rmsnorm_kernel<1>, dim3(rows), dim3(vecs), 0, st, xx, rr, ww, oo, row_index, H, eps);
  } else if (vecs % 256 == 0 && vecs / 256 <= 4) {
    switch (vecs / 256) {
      case 1: launch_pdl(rmsnorm_kernel<1>, dim3(rows), dim3(256), 0, st, xx, rr, ww, oo, row_index, H, eps); break;
      case 2: launch_pdl(rmsnorm_kernel<2>, dim3(rows), dim3(256), 0, st, xx, rr, ww, oo, row_index, H, eps); break;
      case 3: launch_pdl(rmsnorm_kernel<3>, dim3(rows), dim3(256), 0, st, xx, rr, ww, oo, row_index, H, eps); break;
      default: launch_pdl(rmsnorm_kernel<4>, dim3(rows), dim3(256), 0, st, xx, rr, ww, oo, row_index, H, eps); break;
    }
  } else {
    return -1;
  }
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int rope_kv_write(void* qkv, const int* positions, const int* slots, const void* cos_sin, void* kv_layer,
                  int T, int Hq, int Hkv, int max_pos, cudaStream_t st, int head_dim) {
  if (T <= 0) return 0;
  if (head_dim != 64 && head_dim != 128) return -1;
  const int tasks = ((Hq + Hkv) * 8 + Hkv * 16) * head_dim / 128;
  // decode: one task per thread (latency); prefill bursts: 128-thread CTAs (throughput; measured 21 vs 31 us at T=2048)
  const int threads = T >= 512 ? 128 : tasks >= 512 ? 512 : tasks >= 256 ? 256 : 128;
  launch_pdl(head_dim == 64 ? rope_kv_kernel<64> : rope_kv_kernel<128>, dim3(T), dim3(threads), 0, st,
             static_cast<__nv_bfloat16*>(qkv), positions, slots, static_cast<const __nv_bfloat16*>(cos_sin),
             static_cast<__nv_bfloat16*>(kv_layer), Hq, Hkv, max_pos);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int silu_mul(const void* gate_up, void* out, int T, int I, cudaStream_t st, int interleaved) {
  if (T <= 0) return 0;
  if (I % 8) return -1;
  const __nv_bfloat16* gu = static_cast<const __nv_bfloat16*>(gate_up);
  __nv_bfloat16* o = static_cast<__nv_bfloat16*>(out);
  // decode: one output vector per thread (2 loads in flight); prefill bursts: two (4 batched loads in flight)
  if (T >= 512)
    launch_pdl(silu_mul_kernel<2>, dim3(T, (I / 8 + 511) / 512), dim3(256), 0, st, gu, o, I, 2 * I, interleaved);
  else
    launch_pdl(silu_mul_kernel<1>, dim3(T, (I / 8 + 255) / 256), dim3(256), 0, st, gu, o, I, 2 * I, interleaved);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int argmax_rows(const void* logits, int* out, int S, int V, int ld, cudaStream_t st) {
  if (S <= 0) return 0;
  if (ld % 8) return -1;
  launch_pdl(argmax_kernel, dim3(S), dim3(1024), 0, st, static_cast<const __nv_bfloat16*>(logits), out, V, ld);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int permute_gate_up(void* dst, const void* src, int I, int H, int to_physical, cudaStream_t st) {
  if (I % 64 || H % 8) return -1;
  permute_gu_kernel<<<2 * I, 128, 0, st>>>(static_cast<__nv_bfloat16*>(dst), static_cast<const __nv_bfloat16*>(src), I, H, to_physical);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int init_uniform(void* p, size_t n, uint32_t seed, float scale, float offset, cudaStream_t st) {
  if (n == 0) return 0;
  init_uniform_kernel<<<148 * 8, 256, 0, st>>>(static_cast<__nv_bfloat16*>(p), n, seed, scale, offset);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

}  // namespace b200
