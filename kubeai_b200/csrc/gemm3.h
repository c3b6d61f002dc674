// Host interface of the projection GEMM (gemm_wgmma.cu): out[t, n] = sum_k X[t, k] * W[n, k], one 128-row weight slab x
// block_n-token tile per CTA, optional split-K reduced in-kernel in a fixed order, prologue/epilogue modes that absorb the
// elementwise kernels around the projections.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace b200 {

enum { GEMM3_PRO_NONE = 0, GEMM3_PRO_NORM = 1 };
enum { GEMM3_EPI_PLAIN = 0, GEMM3_EPI_RESADD = 1, GEMM3_EPI_SILU = 2, GEMM3_EPI_ROPE_KV = 3, GEMM3_EPI_ARGMAX = 4 };

struct Gemm3Params {
  CUtensorMap tm_w;   // weight [N, K] bf16, box 128 rows x 64 cols, 128B swizzle (GemmPlan::tm_w)
  CUtensorMap tm_x;   // token tile source [rows, K] bf16, box block_n rows x 64 cols: activations, or the residual for PRO_NORM
  int N, T, K;
  int pro, epi;
  // PRO_NORM: per (token, slab) sums of squares of the residual, norm weight [K], eps
  const float* ssq_in;
  int ssq_slabs;
  const __nv_bfloat16* norm_w;
  float eps;
  // epilogue destination: PLAIN out [T, N]; RESADD residual in/out [T, N]; SILU act [T, N/2]; ROPE_KV the fused qkv buffer
  __nv_bfloat16* out;
  int ldo;
  float* ssq_out;     // RESADD (optional): [T, ceil(N/128)] sums of squares of the new residual per 128-column slab
  // RESADD (optional): normed_out [T, N] (leading dimension ldo) = RMSNorm(new residual) * norm_w_out, written by the last CTA
  // of each token tile once every slab's sums are out
  __nv_bfloat16* normed_out;
  const __nv_bfloat16* norm_w_out;
  // ROPE_KV
  const int* positions;
  const int* slots;
  const __nv_bfloat16* cos_sin;
  __nv_bfloat16* kv_layer;
  int Hq, Hkv, max_pos;
  // ARGMAX: per (token, 128-row slab) {best logit, index as int bits}; columns >= n_valid are ignored
  float2* cand;
  int n_valid;
  // split-K partials [tile][split][block_n tokens][128 rows] fp32, and one arrival counter per tile plus one per token tile
  // (zero-initialised, reset by the kernel that uses them)
  float* ws;
  size_t ws_bytes;
  int* counters;
  int counters_cap;
};

struct Gemm3Schedule {
  int block_n;  // tokens per tile: 64, 128 or 256
  int S;        // K-splits per tile
  int rule;     // which rule chose S: 0 the caller's split count, 1 the device-filling rule for one token tile (T <= 128),
                // 2 the device-filling rule over several token tiles (T > 128)
  int grid;     // CTAs
};

// force (T <= 128): 0 automatic; 1..8 that many K-splits; -1 splits sized to the device; -n (n >= 2) n K-splits.
// force (T > 128): 0 automatic; >= 64 the requested token-tile size: the kernel uses the largest of 64 / 128 / 256 that
// does not exceed it (wgmma N is at most 256).  <0: shape or force not served.
int gemm3_schedule(int N, int K, int T, int force, Gemm3Schedule* out);
int gemm3_schedule_for(int N, int K, int T, int force, int sms, Gemm3Schedule* out);   // host-only: for a device of `sms` SMs
int gemm3_launch(const Gemm3Params& p, const Gemm3Schedule& sch, cudaStream_t st);
// fp32 workspace and counters a launch of this schedule needs
size_t gemm3_ws_bytes(int N, const Gemm3Schedule& sch, int T);
int gemm3_counters_needed(int N, const Gemm3Schedule& sch, int T);
// out[s] = best index over the candidates of row s
int argmax_candidates(const void* cand, int* out, int S, int slabs, cudaStream_t st);

}  // namespace b200
