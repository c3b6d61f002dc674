// Paged causal attention for the per-step hot path (SURVEY.md §8a K6 decode, K7 chunked prefill).
// Computes softmax(q . K^T / sqrt(128)) . V over the tokens reachable through a sequence's block
// table, GQA 4:1 — the operation the reference backend delegates to FlashInfer/FlashAttention
// (vllm/model_executor/models/llama.py:223-233, vllm/v1/attention/backends/flashinfer.py).
//
// Design: this op is an HBM stream (decode reads 4 KiB of K+V per context token per layer),
// so the kernel is organised around the page gather, not around the math:
//   * KV layout is [block][K|V][kv_head][16 tokens][128] so one (page, head) is a contiguous 4 KiB
//     run.  A layer is addressed as one 2-D tensor of 256-byte rows; ONE thread per CTA pulls a
//     64-token tile (4 pages x {K,V} x two 64-column halves = 16 TMA boxes of 2 KiB, 128-byte swizzle)
//     and signals an mbarrier.  The per-thread cp.async gather this replaces spent ~45% of the kernel's
//     issue slots on address arithmetic (ncu: issue-active 43% at 12 warps/SM, 4.8 TB/s).
//   * the 4 query heads of a KV head ride in one m16n8k16 tensor-core tile so K/V bytes are read
//     once per group (fp32 softmax, warp-shuffle row reductions, P rounded to bf16 for P.V).
//   * decode: the CTA's 4 warps each own a 16-token strip of every tile and merge their
//     (max, sum, acc) through smem at the end; prefill: a CTA owns 16 query tokens x 4 heads, one
//     head per warp, and walks the causal prefix.
// Rows of a page that lie beyond the sequence's last token are loaded as they are in HBM and masked; the pool is
// zero-initialised and only ever holds finite K/V values, so a masked probability of 0 never meets a NaN.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include <mutex>
#include <unordered_map>

#include "gemm.h"
#include "kernels.h"
#include "launch.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kD = 128;
constexpr int kTile = 64;                       // tokens per smem tile (4 pages)
constexpr int kHalfBytes = kTile * 128;         // [64 tokens][64 dims] bf16, 128-byte rows, 128B swizzle
constexpr int kTileBytes = 2 * kHalfBytes;      // 16 KiB for K, same for V
constexpr int kStageBytes = 2 * kTileBytes;     // K + V

template <int S>
constexpr int attn_smem_bytes() {
  return S * kStageBytes + 64 + 1024;  // stages + mbarriers + slack for the 1 KiB alignment the swizzle needs
}

template <bool DECODE, int S>  // S = tiles in flight per CTA
__global__ void __launch_bounds__(128)
paged_attn_kernel(const __grid_constant__ CUtensorMap tm_kv, const __nv_bfloat16* __restrict__ q, int ldq,
                  __nv_bfloat16* __restrict__ out, int ldo, const int* __restrict__ block_tables, int max_blocks,
                  const AttnWork* __restrict__ work, int Hkv, float scale_log2, float* __restrict__ split_ws) {
  constexpr int WT = DECODE ? 16 : 64;  // tokens of each tile handled by one warp
  constexpr int NT = WT / 8;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (sbase - smem_u32(smem_raw));
  const uint32_t bar_base = sbase + S * kStageBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };

  // work[] and block_tables were uploaded before the first kernel of the step: readable ahead of the dependency wait.
  const AttnWork wk = work[blockIdx.y];  // work items are sorted longest-first; heads are the fast grid dimension
  const int kvh = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, tq = lane & 3;

  const int kv_end = wk.q_pos0 + wk.q_count;  // tokens [0, kv_end) are visible to the last query
  const int ntiles = (kv_end + kTile - 1) / kTile;
  const int last_page = (kv_end - 1) >> 4;
  // split-KV (decode with few sequences: gridDim.z parts per work item so that the context streams on all SMs): this CTA
  // owns tiles [t_begin, t_end) and leaves an unnormalised (max, sum, acc) per head for attn_merge_kernel
  const int parts = DECODE ? static_cast<int>(gridDim.z) : 1;
  const int part = DECODE ? static_cast<int>(blockIdx.z) : 0;
  const int tpp = (ntiles + parts - 1) / parts;
  const int t_begin = part * tpp;
  const int t_end = min(ntiles, t_begin + tpp);
  const int* btab = block_tables + static_cast<size_t>(wk.seq) * max_blocks;

  if (tid == 0) {
    tma_prefetch_desc(&tm_kv);
#pragma unroll
    for (int s = 0; s < S; ++s) mbar_init(full_bar(s), 1);
    fence_mbar_init();
  }
  __syncthreads();

  // thread 0: gather tile `tile` into stage `stage` (pages past the sequence's last one repeat it; they are masked)
  const uint64_t hint = DECODE ? kEvictFirst : kEvictNormal;
  auto issue_tile = [&](int tile, int stage) {
    const uint32_t dst = sbase + stage * kStageBytes;
    mbar_arrive_expect_tx(full_bar(stage), kStageBytes);
#pragma unroll
    for (int pg = 0; pg < 4; ++pg) {
      int page = tile * 4 + pg;
      page = page > last_page ? last_page : page;
      const int blk = __ldg(btab + page);
      const int row_k = ((blk * 2) * Hkv + kvh) * 16;  // row of the layer's [rows][128] view
      const int row_v = row_k + Hkv * 16;
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        tma_load_2d(dst + half * kHalfBytes + pg * 2048, &tm_kv, full_bar(stage), half * 64, row_k, hint);
        tma_load_2d(dst + kTileBytes + half * kHalfBytes + pg * 2048, &tm_kv, full_bar(stage), half * 64, row_v, hint);
      }
    }
  };

  // All S stages are put in flight as early as the data allows.  Decode: every cached token except the newest was
  // written by an earlier step, so tiles that end before the newest token are gathered BEFORE the dependency wait
  // (ptx.cuh griddep_enter) and overlap the RoPE/KV-write kernel upstream.  Prefill tiles may hold rows written by
  // this step: wait first.
  const int safe_tiles = DECODE ? wk.q_pos0 / kTile : 0;
  bool waited = false;
#pragma unroll
  for (int i = 0; i < S; ++i) {
    if (!waited && safe_tiles < t_begin + i + 1) {
      griddep_enter();
      waited = true;
    }
    if (tid == 0 && t_begin + i < t_end) issue_tile(t_begin + i, i);
  }
  if (!waited) griddep_enter();

  // ---- Q fragments (A operand, 16 rows x 128 d as 8 k-steps)
  uint32_t qf[8][4];
  {
    const __nv_bfloat16* r0p = nullptr;
    const __nv_bfloat16* r1p = nullptr;
    if (DECODE) {
      if (g < 4) r0p = q + static_cast<size_t>(wk.q_tok0) * ldq + (kvh * 4 + g) * kD;
    } else {
      const int head = kvh * 4 + warp;
      if (g < wk.q_count) r0p = q + static_cast<size_t>(wk.q_tok0 + g) * ldq + head * kD;
      if (g + 8 < wk.q_count) r1p = q + static_cast<size_t>(wk.q_tok0 + g + 8) * ldq + head * kD;
    }
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const int d = ks * 16 + tq * 2;
      qf[ks][0] = r0p ? *reinterpret_cast<const uint32_t*>(r0p + d) : 0u;
      qf[ks][1] = r1p ? *reinterpret_cast<const uint32_t*>(r1p + d) : 0u;
      qf[ks][2] = r0p ? *reinterpret_cast<const uint32_t*>(r0p + d + 8) : 0u;
      qf[ks][3] = r1p ? *reinterpret_cast<const uint32_t*>(r1p + d + 8) : 0u;
    }
  }

  float o[16][4];
#pragma unroll
  for (int i = 0; i < 16; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  const int wo = DECODE ? warp * 16 : 0;  // this warp's token offset inside a tile

  for (int t = t_begin; t < t_end; ++t) {
    const int stage = (t - t_begin) % S;
    mbar_wait(full_bar(stage), static_cast<uint32_t>((t - t_begin) / S) & 1u);

    const int tok_base = t * kTile + wo;
    if (tok_base < kv_end) {
      const uint32_t kb = sbase + stage * kStageBytes;
      const uint32_t vb = kb + kTileBytes;
      float s[NT][4];
#pragma unroll
      for (int i = 0; i < NT; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
      const int mi = lane >> 3, ri = lane & 7;
      // smem address of 16-byte chunk `chunk` (0..15 over the 128 dims) of token row `tok` of a K or V tile
      auto chunk_addr = [&](uint32_t base, int tok, int chunk) {
        return base + (chunk >> 3) * kHalfBytes + tok * 128 + (((chunk & 7) ^ (tok & 7)) << 4);
      };
      // ---- S = Q K^T
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
#pragma unroll
        for (int tp = 0; tp < WT / 16; ++tp) {
          const int tok = wo + tp * 16 + (mi >> 1) * 8 + ri;
          const int chunk = ks * 2 + (mi & 1);
          uint32_t b0, b1, b2, b3;
          ldmatrix_x4(chunk_addr(kb, tok, chunk), b0, b1, b2, b3);
          mma_bf16_16816(s[tp * 2], qf[ks], b0, b1);
          mma_bf16_16816(s[tp * 2 + 1], qf[ks], b2, b3);
        }
      }
      // ---- causal mask, online softmax (fp32, base-2)
      const int qp0 = DECODE ? wk.q_pos0 : wk.q_pos0 + g;
      const int qp1 = DECODE ? wk.q_pos0 : wk.q_pos0 + g + 8;
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const int kp = tok_base + nt * 8 + tq * 2;
        if (kp > qp0) s[nt][0] = -INFINITY;
        if (kp + 1 > qp0) s[nt][1] = -INFINITY;
        if (kp > qp1) s[nt][2] = -INFINITY;
        if (kp + 1 > qp1) s[nt][3] = -INFINITY;
        mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
        mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      const float mn0 = fmaxf(m0, mx0 * scale_log2), mn1 = fmaxf(m1, mx1 * scale_log2);
      const float mu0 = mn0 == -INFINITY ? 0.f : mn0, mu1 = mn1 == -INFINITY ? 0.f : mn1;
      const float a0 = exp2f(m0 - mu0), a1 = exp2f(m1 - mu1);
      m0 = mn0;
      m1 = mn1;
      float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        s[nt][0] = exp2f(s[nt][0] * scale_log2 - mu0);
        s[nt][1] = exp2f(s[nt][1] * scale_log2 - mu0);
        s[nt][2] = exp2f(s[nt][2] * scale_log2 - mu1);
        s[nt][3] = exp2f(s[nt][3] * scale_log2 - mu1);
        ps0 += s[nt][0] + s[nt][1];
        ps1 += s[nt][2] + s[nt][3];
      }
      l0 = l0 * a0 + ps0;
      l1 = l1 * a1 + ps1;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        o[i][0] *= a0;
        o[i][1] *= a0;
        o[i][2] *= a1;
        o[i][3] *= a1;
      }
      // ---- O += P V
#pragma unroll
      for (int kk = 0; kk < WT / 16; ++kk) {
        uint32_t pa[4];
        pa[0] = pack_bf16x2(s[2 * kk][0], s[2 * kk][1]);
        pa[1] = pack_bf16x2(s[2 * kk][2], s[2 * kk][3]);
        pa[2] = pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
        pa[3] = pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
        for (int dp = 0; dp < 8; ++dp) {
          const int tok = wo + kk * 16 + (mi & 1) * 8 + ri;
          const int chunk = dp * 2 + (mi >> 1);
          uint32_t b0, b1, b2, b3;
          ldmatrix_x4_trans(chunk_addr(vb, tok, chunk), b0, b1, b2, b3);
          mma_bf16_16816(o[dp * 2], pa, b0, b1);
          mma_bf16_16816(o[dp * 2 + 1], pa, b2, b3);
        }
      }
    }
    __syncthreads();  // every warp is done reading this stage
    if (tid == 0 && t + S < t_end) issue_tile(t + S, stage);
  }

  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);

  if (!DECODE) {
    const int head = kvh * 4 + warp;
    const float i0 = l0 > 0.f ? 1.f / l0 : 0.f, i1 = l1 > 0.f ? 1.f / l1 : 0.f;
    if (g < wk.q_count) {
      __nv_bfloat16* dst = out + static_cast<size_t>(wk.q_tok0 + g) * ldo + head * kD + tq * 2;
#pragma unroll
      for (int dn = 0; dn < 16; ++dn)
        *reinterpret_cast<uint32_t*>(dst + dn * 8) = pack_bf16x2(o[dn][0] * i0, o[dn][1] * i0);
    }
    if (g + 8 < wk.q_count) {
      __nv_bfloat16* dst = out + static_cast<size_t>(wk.q_tok0 + g + 8) * ldo + head * kD + tq * 2;
#pragma unroll
      for (int dn = 0; dn < 16; ++dn)
        *reinterpret_cast<uint32_t*>(dst + dn * 8) = pack_bf16x2(o[dn][2] * i1, o[dn][3] * i1);
    }
  } else {
    // merge the 4 warps' partial softmax states: rows 0..3 of each warp tile are the 4 heads.  The stages are free
    // here (the loop's last barrier followed the last tile, and no gather is in flight).
    float* so = reinterpret_cast<float*>(smem);            // [4 warps][4 heads][128]
    float* sm = so + 4 * 4 * kD;                           // [4][4]
    float* sl = sm + 16;                                   // [4][4]
    if (g < 4) {
#pragma unroll
      for (int dn = 0; dn < 16; ++dn) {
        float2 v = make_float2(o[dn][0], o[dn][1]);
        *reinterpret_cast<float2*>(so + (warp * 4 + g) * kD + dn * 8 + tq * 2) = v;
      }
      if (tq == 0) {
        sm[warp * 4 + g] = m0;
        sl[warp * 4 + g] = l0;
      }
    }
    __syncthreads();
    const int d = tid;
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      float mm = -INFINITY;
#pragma unroll
      for (int w = 0; w < 4; ++w) mm = fmaxf(mm, sm[w * 4 + h]);
      float num = 0.f, den = 0.f;
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        const float mw = sm[w * 4 + h];
        const float wgt = (mw == -INFINITY) ? 0.f : exp2f(mw - mm);
        num += so[(w * 4 + h) * kD + d] * wgt;
        den += sl[w * 4 + h] * wgt;
      }
      if (parts == 1) {
        out[static_cast<size_t>(wk.q_tok0) * ldo + (kvh * 4 + h) * kD + d] = __float2bfloat16_rn(den > 0.f ? num / den : 0.f);
      } else {
        // [work][kv head][part][4 heads][128 acc | max | sum]
        float* dst = split_ws + ((static_cast<size_t>(blockIdx.y) * Hkv + kvh) * parts + part) * (4 * (kD + 2)) + h * (kD + 2);
        dst[d] = num;
        if (d == 0) {
          dst[kD] = mm;
          dst[kD + 1] = den;
        }
      }
    }
  }
}

// out[token, head, :] = sum_p acc_p 2^(m_p - M) / sum_p l_p 2^(m_p - M) over the parts of a split decode work item
__global__ void __launch_bounds__(128)
attn_merge_kernel(const float* __restrict__ split_ws, __nv_bfloat16* __restrict__ out, int ldo, const AttnWork* __restrict__ work,
                  int Hkv, int parts) {
  griddep_enter();
  const AttnWork wk = work[blockIdx.y];
  const int kvh = blockIdx.x, d = threadIdx.x;
  const float* base = split_ws + (static_cast<size_t>(blockIdx.y) * Hkv + kvh) * parts * (4 * (kD + 2));
#pragma unroll
  for (int h = 0; h < 4; ++h) {
    float mm = -INFINITY;
    for (int p = 0; p < parts; ++p) mm = fmaxf(mm, base[(p * 4 + h) * (kD + 2) + kD]);
    float num = 0.f, den = 0.f;
    for (int p = 0; p < parts; ++p) {
      const float* s = base + (p * 4 + h) * (kD + 2);
      const float wgt = (s[kD] == -INFINITY) ? 0.f : exp2f(s[kD] - mm);
      num += s[d] * wgt;
      den += s[kD + 1] * wgt;
    }
    out[static_cast<size_t>(wk.q_tok0) * ldo + (kvh * 4 + h) * kD + d] = __float2bfloat16_rn(den > 0.f ? num / den : 0.f);
  }
}

constexpr int kPrefillStages = 2;

int decode_stages() {  // B200_ATTN_STAGES=2|3|4 (tiles in flight per decode CTA)
  static const int v = [] {
    const char* e = getenv("B200_ATTN_STAGES");
    const int n = e ? atoi(e) : 2;
    return n == 3 || n == 4 ? n : 2;
  }();
  return v;
}

// One tensor map per KV-layer base pointer: the layer is viewed as [rows][128] bf16 with 256-byte rows, gathered in
// boxes of 16 rows x 64 columns (one page-head half).  The row count is an upper bound, not the allocation size: the
// kernel only ever addresses pages named by the block table.
}  // namespace

int kv_map_for(const void* kv_layer, CUtensorMap* out) {
  static std::unordered_map<const void*, CUtensorMap> cache;
  static std::mutex mu;
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(kv_layer);
  if (it == cache.end()) {
    CUtensorMap tm;
    if ((reinterpret_cast<uintptr_t>(kv_layer) & 255) != 0) return -5;
    if (int rc = tmap_encode_bf16_2d(&tm, kv_layer, 1ull << 30, kD, kD, 16, 64, 1)) return rc;
    if (cache.size() > 4096) cache.clear();
    it = cache.emplace(kv_layer, tm).first;
  }
  *out = it->second;
  return 0;
}

namespace {

template <bool DECODE, int S>
int launch_attn(const CUtensorMap& tm, dim3 grid, cudaStream_t st, const __nv_bfloat16* q, int ldq, __nv_bfloat16* out,
                int ldo, const int* block_tables, int max_blocks, const AttnWork* work, int Hkv, float scale_log2,
                float* split_ws = nullptr) {
  static std::atomic<unsigned long long> attr_done{0};
  if (!ensure_dynamic_smem(paged_attn_kernel<DECODE, S>, attn_smem_bytes<S>(), &attr_done)) return -3;
  launch_pdl(paged_attn_kernel<DECODE, S>, grid, dim3(128), attn_smem_bytes<S>(), st, tm, q, ldq, out, ldo, block_tables,
             max_blocks, work, Hkv, scale_log2, split_ws);
  if (cudaGetLastError() != cudaSuccess) return -2;
  if (DECODE && grid.z > 1) {
    launch_pdl(attn_merge_kernel, dim3(grid.x, grid.y), dim3(128), 0, st, static_cast<const float*>(split_ws), out, ldo, work, Hkv,
               static_cast<int>(grid.z));
    if (cudaGetLastError() != cudaSuccess) return -2;
  }
  return 0;
}

}  // namespace

size_t attn_split_ws_bytes(int num_work, int Hkv, int parts) {
  return static_cast<size_t>(num_work) * Hkv * parts * 4 * (kD + 2) * sizeof(float);
}

// Parts per decode work item such that the launch has about two CTAs per SM, each with at least two 64-token tiles.
int attn_decode_split(int num_work, int Hkv, int max_ctx, int sms) {
  const int ctas = num_work * Hkv;
  if (ctas <= 0 || ctas >= sms) return 1;
  int p = (2 * sms + ctas - 1) / ctas;
  const int by_ctx = (max_ctx + 2 * kTile - 1) / (2 * kTile);
  if (p > by_ctx) p = by_ctx;
  if (p > 32) p = 32;
  return p < 1 ? 1 : p;
}

int paged_attention(const void* q, int ldq, void* out, int ldo, const void* kv_layer, const int* block_tables,
                    int max_blocks, const AttnWork* work, int num_work, int Hq, int Hkv, float scale,
                    int decode, cudaStream_t st, float* split_ws, int split) {
  if (num_work <= 0) return 0;
  if (Hq != 4 * Hkv) return -1;
  if (split > 1 && (!decode || !split_ws)) return -1;
  CUtensorMap tm;
  if (int rc = kv_map_for(kv_layer, &tm)) return rc;
  const float scale_log2 = scale * 1.4426950408889634f;
  dim3 grid(Hkv, num_work, split > 1 ? split : 1);
  const __nv_bfloat16* qq = static_cast<const __nv_bfloat16*>(q);
  __nv_bfloat16* oo = static_cast<__nv_bfloat16*>(out);
  if (!decode)
    return launch_attn<false, kPrefillStages>(tm, grid, st, qq, ldq, oo, ldo, block_tables, max_blocks, work, Hkv, scale_log2);
  switch (decode_stages()) {
    case 3: return launch_attn<true, 3>(tm, grid, st, qq, ldq, oo, ldo, block_tables, max_blocks, work, Hkv, scale_log2, split_ws);
    case 4: return launch_attn<true, 4>(tm, grid, st, qq, ldq, oo, ldo, block_tables, max_blocks, work, Hkv, scale_log2, split_ws);
    default: return launch_attn<true, 2>(tm, grid, st, qq, ldq, oo, ldo, block_tables, max_blocks, work, Hkv, scale_log2, split_ws);
  }
}

}  // namespace b200
