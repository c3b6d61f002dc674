// Host-side plan of the projection GEMM (gemm_wgmma.cu) and the tensor-map helpers shared with the attention kernels.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace b200 {

struct GemmPlan {
  CUtensorMap tm_w;  // weight [N, K] bf16, box 128 x 64, 128B swizzle
  int N, K;
  const void* w_ptr;  // same tensor, raw pointer
  int ldw;
  float* ws;          // fp32 split-K workspace
  size_t ws_bytes;
  int* counters;      // zero-initialised, self-resetting
  int counters_cap;
};

// variant 2 (default): split-K sized to the device; variant 1: every tile over its whole K (no split)
void gemm_set_variant(int v);
int gemm_variant();
constexpr int kGemmNumBlockN = 3;         // token-tile sizes 64, 128, 256
int gemm_block_n_for(int T);              // token-tile size for T tokens
int gemm_block_n_index(int block_n);      // 0..2
int num_sms();
// W row-major [N, K] with leading dimension ldw (elements).
int gemm_plan_init(GemmPlan* p, const void* W, int N, int K, int ldw, float* ws, size_t ws_bytes, int* counters, int counters_cap);
// Activation map over X row-major [rows, K] (rows = buffer capacity), for a given token-tile size.
int gemm_make_x_map(CUtensorMap* tm, const void* X, int rows, int K, int ldx, int block_n);
// Generic 2-D bf16 tensor map (used by the attention kernel for the paged KV cache).
int tmap_encode_bf16_2d(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, int box_rows,
                        int box_cols, int swizzle128);
// out[t, n] (bf16, leading dimension ldo) for t < T.
int gemm_run(const GemmPlan& p, const CUtensorMap& tm_x, int block_n, void* out, int ldo, int T, cudaStream_t st);

}  // namespace b200
