// Chunked-prefill paged attention on the Hopper tensor cores (SURVEY.md §8a K7): for every query token of a work item,
// softmax(q . K^T / sqrt(128)) . V over the causal prefix gathered through the sequence's block table, GQA 4:1 — the
// operation the reference backend delegates to FlashInfer/FlashAttention (vllm/model_executor/models/llama.py:223-233).
//
// H100 design: one CTA = one warpgroup = (work item of up to 64 query tokens, one query head).
//   * Q [64 tokens][128] sits in shared memory as two 64-column halves in the 128-byte-swizzled K-major layout wgmma reads;
//     each 64-token K tile goes to the same layout, V is transposed into [128 dims][64 tokens] (K-major for P . V).
//   * S = Q K^T: wgmma m64n64k16 with both operands from shared-memory descriptors, fp32 accumulators in registers.
//   * online softmax in registers (row max / sum over the 4 threads of a quad), P rounded to bf16 and fed to O += P V as
//     the register A operand of wgmma (the accumulator fragment of S is the A fragment of P V), O in registers.
// Tokens past the context are not read: their K / V rows are zero and their scores masked.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <atomic>

#include "kernels.h"
#include "launch.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kD = 128;
constexpr int kQ = kPrefillQueryBlock;   // 64 query tokens per work item = the wgmma M tile
constexpr int kKv = 64;                  // kv tokens per tile
constexpr int kHalf = 64 * 128;          // [64 rows][64 bf16] swizzled: 8 KB
constexpr int kSmem = 1024 + 3 * 2 * kHalf;   // Q, K, V^T

// byte offset of 16-byte chunk c of row r in a 128B-swizzled tile (base 1024-B aligned)
__device__ __forceinline__ uint32_t swz(int r, int c) { return r * 128 + ((c ^ (r & 7)) << 4); }

__global__ void __launch_bounds__(128) prefill_attn_wgmma_kernel(const __nv_bfloat16* __restrict__ qkv, int qkv_rows, int ldq,
                                                                 __nv_bfloat16* __restrict__ out, int ldo,
                                                                 const __nv_bfloat16* __restrict__ kv_layer,
                                                                 const int* __restrict__ block_tables, int max_blocks,
                                                                 const AttnWork* __restrict__ work, int Hkv, float scale_log2) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (sbase - smem_u32(smem_raw));
  uint8_t* sq = smem;                 // two halves: dims 0..63, 64..127
  uint8_t* sk = smem + 2 * kHalf;
  uint8_t* sv = smem + 4 * kHalf;     // V^T: rows = dims 0..127, 64 tokens each
  const uint32_t aq = sbase, ak = sbase + 2 * kHalf, av = sbase + 4 * kHalf;

  // work[] and block_tables were uploaded before the first kernel of the step: readable ahead of the dependency wait
  const AttnWork wk = work[blockIdx.y];
  const int h = blockIdx.x, kvh = h >> 2;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int* btab = block_tables + static_cast<size_t>(wk.seq) * max_blocks;
  const int kv_end = wk.q_pos0 + wk.q_count;
  const size_t head_stride = 16 * kD, kind_stride = static_cast<size_t>(Hkv) * head_stride;
  griddep_enter();

  // ---- Q tile (rows past the work item read as zero)
  for (int i = tid; i < kQ * 16; i += 128) {
    const int r = i >> 4, c = i & 15;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r < wk.q_count && wk.q_tok0 + r < qkv_rows)
      v = *reinterpret_cast<const uint4*>(qkv + static_cast<size_t>(wk.q_tok0 + r) * ldq + h * kD + c * 8);
    *reinterpret_cast<uint4*>(sq + (c >> 3) * kHalf + swz(r, c & 7)) = v;
  }

  // this thread's accumulator rows (wgmma D fragment): r0 and r0 + 8
  const int r0 = warp * 16 + (lane >> 2);
  const int qpos0 = wk.q_pos0 + r0, qpos1 = qpos0 + 8;
  float o[2][32];
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[j][i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

  const int ntiles = (kv_end + kKv - 1) / kKv;
  for (int t = 0; t < ntiles; ++t) {
    const int j0 = t * kKv;
    __syncthreads();   // the previous tile's wgmma reads are complete (wait_group 0 below) in every warp
    // ---- K tile [64 tokens][128 dims] and V^T [128 dims][64 tokens]
    for (int i = tid; i < kKv * 16; i += 128) {
      const int r = i >> 4, c = i & 15, j = j0 + r;
      uint4 kvec = make_uint4(0, 0, 0, 0), vvec = kvec;   // tokens past the context: no page to read, masked below
      if (j < kv_end) {
        const size_t base = static_cast<size_t>(__ldg(btab + (j >> 4))) * 2 * kind_stride + kvh * head_stride + (j & 15) * kD + c * 8;
        kvec = *reinterpret_cast<const uint4*>(kv_layer + base);
        vvec = *reinterpret_cast<const uint4*>(kv_layer + base + kind_stride);
      }
      *reinterpret_cast<uint4*>(sk + (c >> 3) * kHalf + swz(r, c & 7)) = kvec;
      const __nv_bfloat16* vh = reinterpret_cast<const __nv_bfloat16*>(&vvec);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int d = c * 8 + e;   // row d of V^T, column r (token)
        *reinterpret_cast<__nv_bfloat16*>(sv + swz(d, r >> 3) + (r & 7) * 2) = vh[e];
      }
    }
    fence_proxy_async();   // generic-proxy stores -> wgmma (async proxy) reads
    __syncthreads();

    // ---- S = Q K^T
    float s[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kD / 16; ++kk) {
      const uint32_t off = (kk >> 2) * kHalf + (kk & 3) * 32;
      wgmma_m64n64(s, gmma_desc(aq + off), gmma_desc(ak + off));
    }
    wgmma_commit();
    wgmma_wait0();

    // ---- causal mask + online softmax (scaled to log2 units)
    float mx0 = m0, mx1 = m1;
#pragma unroll
    for (int q = 0; q < 8; ++q)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int j = j0 + q * 8 + (lane & 3) * 2 + e;
        float& a = s[q * 4 + e];
        float& b = s[q * 4 + 2 + e];
        a = (j < kv_end && j <= qpos0) ? a * scale_log2 : -INFINITY;
        b = (j < kv_end && j <= qpos1) ? b * scale_log2 : -INFINITY;
        mx0 = fmaxf(mx0, a);
        mx1 = fmaxf(mx1, b);
      }
#pragma unroll
    for (int x = 1; x <= 2; x <<= 1) {
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, x));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, x));
    }
    const float b0 = mx0 == -INFINITY ? 0.f : mx0, b1 = mx1 == -INFINITY ? 0.f : mx1;
    const float c0 = exp2f(m0 - b0), c1 = exp2f(m1 - b1);   // m == -inf: 0 (nothing accumulated yet)
    m0 = mx0;
    m1 = mx1;
    float ps0 = 0.f, ps1 = 0.f;
    uint32_t pa[4][4];   // P as the A operand of P V: one m64 x k16 fragment per 16 kv tokens
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float p00 = exp2f(s[q * 4 + 0] - b0), p01 = exp2f(s[q * 4 + 1] - b0);
      const float p10 = exp2f(s[q * 4 + 2] - b1), p11 = exp2f(s[q * 4 + 3] - b1);
      ps0 += p00 + p01;
      ps1 += p10 + p11;
      pa[q >> 1][(q & 1) * 2 + 0] = pack_bf16x2(p00, p01);
      pa[q >> 1][(q & 1) * 2 + 1] = pack_bf16x2(p10, p11);
    }
    l0 = l0 * c0 + ps0;
    l1 = l1 * c1 + ps1;
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        o[j][q * 4 + 0] *= c0;
        o[j][q * 4 + 1] *= c0;
        o[j][q * 4 + 2] *= c1;
        o[j][q * 4 + 3] *= c1;
      }

    // ---- O += P V
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kKv / 16; ++kk)
#pragma unroll
      for (int j = 0; j < 2; ++j) wgmma_m64n64_rs(o[j], pa[kk], gmma_desc(av + j * kHalf + kk * 32));
    wgmma_commit();
    wgmma_wait0();
  }

  // ---- normalise and store
#pragma unroll
  for (int x = 1; x <= 2; x <<= 1) {
    l0 += __shfl_xor_sync(0xffffffffu, l0, x);
    l1 += __shfl_xor_sync(0xffffffffu, l1, x);
  }
  const float inv0 = l0 > 0.f ? 1.f / l0 : 0.f, inv1 = l1 > 0.f ? 1.f / l1 : 0.f;
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int d = j * 64 + q * 8 + (lane & 3) * 2;
      if (r0 < wk.q_count)
        *reinterpret_cast<uint32_t*>(out + static_cast<size_t>(wk.q_tok0 + r0) * ldo + h * kD + d) =
            pack_bf16x2(o[j][q * 4 + 0] * inv0, o[j][q * 4 + 1] * inv0);
      if (r0 + 8 < wk.q_count)
        *reinterpret_cast<uint32_t*>(out + static_cast<size_t>(wk.q_tok0 + r0 + 8) * ldo + h * kD + d) =
            pack_bf16x2(o[j][q * 4 + 2] * inv1, o[j][q * 4 + 3] * inv1);
    }
}

}  // namespace

int paged_attention_prefill_tc(const void* qkv, int qkv_rows, int ldq, void* out, int ldo, const void* kv_layer, const int* block_tables,
                               int max_blocks, const AttnWork* work, int num_work, int Hq, int Hkv, float scale, cudaStream_t st) {
  if (num_work <= 0) return 0;
  if (Hq != 4 * Hkv || qkv_rows <= 0 || ldq % 8 || ldo % 2) return -1;
  static std::atomic<unsigned long long> attr_done{0};
  if (!ensure_dynamic_smem(prefill_attn_wgmma_kernel, kSmem, &attr_done)) return -3;
  cudaError_t e = launch_pdl(prefill_attn_wgmma_kernel, dim3(Hq, num_work), dim3(128), kSmem, st,
                             static_cast<const __nv_bfloat16*>(qkv), qkv_rows, ldq, static_cast<__nv_bfloat16*>(out), ldo,
                             static_cast<const __nv_bfloat16*>(kv_layer), block_tables, max_blocks, work, Hkv,
                             scale * 1.4426950408889634f);
  return e == cudaSuccess ? 0 : -2;
}

}  // namespace b200
