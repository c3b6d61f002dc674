// Deferred split-K reduction: a GEMM may leave split tiles unreduced for its consumer kernel.
// A tile computed entirely by one CTA pair is written as bf16 to the output tensor; a tile whose
// k-range is shared by several pairs is left as one fp32 segment per pair in an L2-resident
// workspace.  The consumer kernel (RMSNorm, RoPE, SiLU*mul, argmax, or the generic reducer) sums the
// segments while it loads its input, so the kernel boundary is the only synchronisation of the
// split-K reduction: no flags, fences, spin-waits or extra round trips inside the GEMM.
//   table:     per output tile (256 weight rows x block_n tokens) {first segment, #segments};
//              #segments == 1 means "complete: read the bf16 tensor"
//   workspace: [segment][rank 0|1][token in tile][128 weight rows] fp32
// Segments are summed in index order in fp32 and rounded to bf16 once — the same rounding point as
// a GEMM that writes bf16 (vllm linear output), so downstream numerics are unchanged.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

struct PartialView {
  const float* ws;               // nullptr => the op reads its ordinary bf16 input tensor
  const int2* table;             // [slab2 * ntt + tt]
  const __nv_bfloat16* dense;    // output tensor holding the complete tiles
  int ld_dense;
  int slot;                      // floats per (segment, rank) slot = block_n * 128
  int ntt;                       // token tiles
  int block_n;                   // tokens per tile (power of two)
  int bn_shift;                  // log2(block_n)
};

inline PartialView no_partials() { return PartialView{nullptr, nullptr, nullptr, 0, 0, 1, 512, 9}; }

__device__ __forceinline__ int2 partial_entry(const PartialView& v, int t, int n0) {
  return __ldg(v.table + (n0 >> 8) * v.ntt + (t >> v.bn_shift));
}
__device__ __forceinline__ void unpack8_bf16(const uint4& u, float (&o)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = __bfloat1622float2(h[j]);
    o[2 * j] = f.x;
    o[2 * j + 1] = f.y;
  }
}

// Value of the GEMM output for token t, weight rows [n0, n0+8) (n0 % 8 == 0), as bf16-representable floats, given the
// tile's table entry e.
__device__ __forceinline__ void load8_entry(const PartialView& v, const int2 e, int t, int n0, float (&o)[8]) {
  if (e.y == 1) {  // complete tile: already bf16 in the output tensor
    unpack8_bf16(__ldcg(reinterpret_cast<const uint4*>(v.dense + static_cast<size_t>(t) * v.ld_dense + n0)), o);
    return;
  }
  const int rank = (n0 >> 7) & 1, row = n0 & 127;
  const int tl = t & (v.block_n - 1);
  const size_t stride = 2 * static_cast<size_t>(v.slot);
  const float* p = v.ws + (static_cast<size_t>(e.x) * 2 + rank) * v.slot + static_cast<size_t>(tl) * 128 + row;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
  // eight segments' loads are issued before the first add (independent L2 round trips: the o_proj / down_proj tiles of a
  // decode step have 5-6 segments, one round instead of two), the adds stay in segment order so the result does not
  // depend on the unrolling
  for (int s = 0; s < e.y; s += 8, p += 8 * stride) {
    float4 x[8], y[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      if (s + u < e.y) {
        x[u] = __ldcg(reinterpret_cast<const float4*>(p + u * stride));
        y[u] = __ldcg(reinterpret_cast<const float4*>(p + u * stride + 4));
      } else {
        x[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        y[u] = x[u];
      }
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      a.x += x[u].x; a.y += x[u].y; a.z += x[u].z; a.w += x[u].w;
      b.x += y[u].x; b.y += y[u].y; b.z += y[u].z; b.w += y[u].w;
    }
  }
  o[0] = __bfloat162float(__float2bfloat16_rn(a.x));
  o[1] = __bfloat162float(__float2bfloat16_rn(a.y));
  o[2] = __bfloat162float(__float2bfloat16_rn(a.z));
  o[3] = __bfloat162float(__float2bfloat16_rn(a.w));
  o[4] = __bfloat162float(__float2bfloat16_rn(b.x));
  o[5] = __bfloat162float(__float2bfloat16_rn(b.y));
  o[6] = __bfloat162float(__float2bfloat16_rn(b.z));
  o[7] = __bfloat162float(__float2bfloat16_rn(b.w));
}

__device__ __forceinline__ void load8_partials(const PartialView& v, int t, int n0, float (&o)[8]) {
  load8_entry(v, partial_entry(v, t, n0), t, n0, o);
}

// M vectors of one token at once.  The table entries are static per (plan, token-tile count), so a kernel looks them
// up BEFORE its dependency wait (partial_entries) and only the data loads follow it (load8xM_entries).  When every tile
// involved is complete (the common case at large T) the M 16-byte loads are issued back to back — M memory round
// trips overlap instead of chaining lookup -> branch -> load per vector.
template <int M>
__device__ __forceinline__ void partial_entries(const PartialView& v, int t, const int (&n0)[M], int2 (&e)[M]) {
#pragma unroll
  for (int i = 0; i < M; ++i) e[i] = partial_entry(v, t, n0[i]);
}

template <int M>
__device__ __forceinline__ void load8xM_entries(const PartialView& v, const int2 (&e)[M], int t, const int (&n0)[M],
                                                float (&o)[M][8]) {
  bool dense = true;
#pragma unroll
  for (int i = 0; i < M; ++i) dense = dense && e[i].y == 1;
  if (dense) {
    uint4 u[M];
#pragma unroll
    for (int i = 0; i < M; ++i)
      u[i] = __ldcg(reinterpret_cast<const uint4*>(v.dense + static_cast<size_t>(t) * v.ld_dense + n0[i]));
#pragma unroll
    for (int i = 0; i < M; ++i) unpack8_bf16(u[i], o[i]);
    return;
  }
#pragma unroll
  for (int i = 0; i < M; ++i) load8_entry(v, e[i], t, n0[i], o[i]);
}

template <int M>
__device__ __forceinline__ void load8xM_partials(const PartialView& v, int t, const int (&n0)[M], float (&o)[M][8]) {
  int2 e[M];
  partial_entries<M>(v, t, n0, e);
  load8xM_entries<M>(v, e, t, n0, o);
}

}  // namespace b200
