// Copy whole KV pages across every layer (parallel sampling: the children of an n > 1 request get their own copy of the
// prompt's partly filled tail page; the full pages are shared by reference).  The pool is [layer][block][K|V][kv_head][16][128]
// bf16, so one page of one layer is one contiguous run of block_bytes.  A bit-exact 16-byte copy: no arithmetic.
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"

namespace b200 {

namespace {

constexpr int kCopyThreads = 256;
constexpr int kCopyVecs = 4;   // 16-byte vectors per thread per CTA: a CTA moves 16 KiB of one page of one layer
constexpr int64_t kCopyChunk = static_cast<int64_t>(kCopyThreads) * kCopyVecs * 16;

// grid (pair * num_layers + layer, chunk of the page): all loads of a thread are issued before its stores
__global__ void __launch_bounds__(kCopyThreads) kv_copy_kernel(uint8_t* __restrict__ kv, int num_layers, int64_t layer_stride,
                                                               int64_t block_bytes, const int* __restrict__ src,
                                                               const int* __restrict__ dst) {
  const int pair = blockIdx.x / num_layers, layer = blockIdx.x % num_layers;
  const int64_t base = static_cast<int64_t>(layer) * layer_stride;
  const uint4* s = reinterpret_cast<const uint4*>(kv + base + static_cast<int64_t>(src[pair]) * block_bytes);
  uint4* d = reinterpret_cast<uint4*>(kv + base + static_cast<int64_t>(dst[pair]) * block_bytes);
  const int64_t nvec = block_bytes / 16;
  const int64_t v0 = static_cast<int64_t>(blockIdx.y) * (kCopyChunk / 16) + threadIdx.x;
  uint4 r[kCopyVecs];
#pragma unroll
  for (int i = 0; i < kCopyVecs; ++i) {
    const int64_t v = v0 + static_cast<int64_t>(i) * kCopyThreads;
    if (v < nvec) r[i] = __ldcs(s + v);
  }
#pragma unroll
  for (int i = 0; i < kCopyVecs; ++i) {
    const int64_t v = v0 + static_cast<int64_t>(i) * kCopyThreads;
    if (v < nvec) __stcs(d + v, r[i]);
  }
}

}  // namespace

int kv_copy_blocks(void* kv, int num_layers, int64_t layer_stride_bytes, int64_t block_bytes, const int* src, const int* dst,
                   int n_pairs, cudaStream_t st) {
  if (n_pairs == 0) return 0;
  if (!kv || !src || !dst || n_pairs < 0 || num_layers < 1 || block_bytes <= 0 || block_bytes % 16 ||
      layer_stride_bytes % 16 || reinterpret_cast<uintptr_t>(kv) % 16 ||
      static_cast<int64_t>(n_pairs) * num_layers > 0x7fffffff)
    return -1;
  const dim3 grid(static_cast<unsigned>(n_pairs * num_layers), static_cast<unsigned>((block_bytes + kCopyChunk - 1) / kCopyChunk));
  kv_copy_kernel<<<grid, kCopyThreads, 0, st>>>(static_cast<uint8_t*>(kv), num_layers, layer_stride_bytes, block_bytes, src, dst);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

}  // namespace b200
