// Paged causal decode attention for the per-step hot path (SURVEY.md §8a K6; chunked prefill is attention_wgmma.cu).
// Computes softmax(q . K^T / sqrt(D)) . V over the tokens reachable through a sequence's block
// table, with head size D = 64 or 128 and G = Hq / Hkv query heads per KV head — the operation the reference backend
// delegates to FlashInfer/FlashAttention
// (vllm/model_executor/models/llama.py:223-233, vllm/v1/attention/backends/flashinfer.py).
//
// Design: this op is an HBM stream (decode reads 4 KiB of K+V per context token per layer),
// so the kernel is organised around the page gather, not around the math:
//   * KV layout is [block][K|V][kv_head][16 tokens][D] so one (page, head) is a contiguous 2 * 16 * D-byte
//     run.  A layer is addressed as one 2-D tensor of 2 * D-byte rows; ONE thread per CTA pulls a
//     64-token tile (4 pages x {K,V} x D / 64 column halves = 8 * D / 64 TMA boxes of 2 KiB, 128-byte swizzle)
//     and signals an mbarrier.  At D = 64 a tile is half the bytes and twice as many tiles are kept in flight.
//     The per-thread cp.async gather this replaces spent ~45% of the kernel's issue slots on address arithmetic
//     (ncu: issue-active 43% at 12 warps/SM, 4.8 TB/s).
//   * decode: the G query heads of a KV head (1 <= G <= 16) ride in one m16n8k16 tensor-core tile so
//     K/V bytes are read once per group (fp32 softmax, warp-shuffle row reductions, P rounded to bf16
//     for P.V).  The CTA's 4 warps each own a 16-token strip of every tile and merge their
//     (max, sum, acc) through smem at the end.
//   * a decode work item may carry q_count consecutive query positions with G * q_count <= 16
//     (speculative decoding's verify step: the last token and its drafts).  Tile row r = G * j + h is
//     head kvh * G + h at position j; rows past G * q_count stay zero, and the K/V of the group is still
//     read once.  The decode kernel is compiled twice: for G = 4 (the row map folds to shifts and masks)
//     and for a group size read at run time.
// Rows of a page that lie beyond the sequence's last token are loaded as they are in HBM and masked; the pool is
// zero-initialised and only ever holds finite K/V values, so a masked probability of 0 never meets a NaN.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <functional>
#include <mutex>
#include <unordered_map>
#include <utility>

#include "gemm.h"
#include "kernels.h"
#include "launch.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kTile = 64;                       // tokens per smem tile (4 pages)
constexpr int kHalfBytes = kTile * 128;         // [64 tokens][64 dims] bf16, 128-byte rows, 128B swizzle
// head size D (64 or 128): a K (or V) tile is D / 64 halves, 16 KiB at D = 128 and 8 KiB at D = 64
template <int D>
__host__ __device__ constexpr int tile_bytes() { return (D / 64) * kHalfBytes; }
template <int D>
__host__ __device__ constexpr int stage_bytes() { return 2 * tile_bytes<D>(); }  // K + V

// Tiles in flight per CTA.  A 64-token tile is 32 KiB of K + V at D = 128 and 16 KiB at D = 64, so D = 64 keeps twice the
// tiles in flight: the bytes in flight per CTA are the same at both head sizes.
template <int D>
__host__ __device__ constexpr int stages() { return 2 * 128 / D; }
template <int D>
constexpr int attn_smem_bytes() {
  return stages<D>() * stage_bytes<D>() + 64 + 1024;  // stages + mbarriers + slack for the 1 KiB alignment the swizzle needs
}

// GC = the group size G when it is known at compile time (4), 0 = read G from group; D = head size (64 or 128)
template <int GC, int D>
__global__ void __launch_bounds__(128)
paged_attn_kernel(const __grid_constant__ CUtensorMap tm_kv, const __nv_bfloat16* __restrict__ q, int ldq,
                  __nv_bfloat16* __restrict__ out, int ldo, const int* __restrict__ block_tables, int max_blocks,
                  const AttnWork* __restrict__ work, int Hkv, int group, float scale_log2, float* __restrict__ split_ws) {
  static_assert(D == 64 || D == 128, "head size 64 or 128");
  constexpr int S = stages<D>();
  constexpr int kTileBytes = tile_bytes<D>(), kStageBytes = stage_bytes<D>();
  constexpr int KS = D / 16;  // k-steps of Q K^T, and n16 column pairs of P V
  constexpr int WT = 16;      // tokens of each tile handled by one warp
  constexpr int NT = WT / 8;
  const int G = GC ? GC : group;
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
  // split-KV (few sequences: gridDim.z parts per work item so that the context streams on all SMs): this CTA owns tiles
  // [t_begin, t_end) and leaves an unnormalised (max, sum, acc) per head for attn_merge_kernel
  const int parts = static_cast<int>(gridDim.z);
  const int part = static_cast<int>(blockIdx.z);
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
  auto issue_tile = [&](int tile, int stage) {
    const uint32_t dst = sbase + stage * kStageBytes;
    mbar_arrive_expect_tx(full_bar(stage), kStageBytes);
#pragma unroll
    for (int pg = 0; pg < 4; ++pg) {
      int page = tile * 4 + pg;
      page = page > last_page ? last_page : page;
      const int blk = __ldg(btab + page);
      const int row_k = ((blk * 2) * Hkv + kvh) * 16;  // row of the layer's [rows][D] view
      const int row_v = row_k + Hkv * 16;
#pragma unroll
      for (int half = 0; half < D / 64; ++half) {
        tma_load_2d(dst + half * kHalfBytes + pg * 2048, &tm_kv, full_bar(stage), half * 64, row_k, kEvictFirst);
        tma_load_2d(dst + kTileBytes + half * kHalfBytes + pg * 2048, &tm_kv, full_bar(stage), half * 64, row_v, kEvictFirst);
      }
    }
  };

  // All S stages are put in flight as early as the data allows.  Every cached token except the newest was written by an
  // earlier step, so tiles that end before the newest token are gathered BEFORE the dependency wait (ptx.cuh
  // griddep_enter) and overlap the RoPE/KV-write kernel upstream.
  const int safe_tiles = wk.q_pos0 / kTile;
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

  // ---- Q fragments (A operand, 16 rows x D dims as D / 16 k-steps)
  // fragment rows g and g + 8 are tile rows r = G * j + h, i.e. (j, h) = divmod(r, G)
  const int j0 = g / G, j1 = (g + 8) / G;
  uint32_t qf[KS][4];
  {
    const __nv_bfloat16* r0p = nullptr;
    const __nv_bfloat16* r1p = nullptr;
    // rows past the live ones (G * q_count) stay zero: they never touch the rows of the positions that exist
    const int nrows = G * wk.q_count;
    if (g < nrows) r0p = q + static_cast<size_t>(wk.q_tok0 + j0) * ldq + (kvh * G + g - j0 * G) * D;
    if (g + 8 < nrows) r1p = q + static_cast<size_t>(wk.q_tok0 + j1) * ldq + (kvh * G + g + 8 - j1 * G) * D;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      const int d = ks * 16 + tq * 2;
      qf[ks][0] = r0p ? *reinterpret_cast<const uint32_t*>(r0p + d) : 0u;
      qf[ks][1] = r1p ? *reinterpret_cast<const uint32_t*>(r1p + d) : 0u;
      qf[ks][2] = r0p ? *reinterpret_cast<const uint32_t*>(r0p + d + 8) : 0u;
      qf[ks][3] = r1p ? *reinterpret_cast<const uint32_t*>(r1p + d + 8) : 0u;
    }
  }

  float o[2 * KS][4];
#pragma unroll
  for (int i = 0; i < 2 * KS; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  const int wo = warp * 16;  // this warp's token offset inside a tile

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
      // smem address of 16-byte chunk `chunk` (0..D/8-1 over the D dims) of token row `tok` of a K or V tile
      auto chunk_addr = [&](uint32_t base, int tok, int chunk) {
        return base + (chunk >> 3) * kHalfBytes + tok * 128 + (((chunk & 7) ^ (tok & 7)) << 4);
      };
      // ---- S = Q K^T
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
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
      const int qp0 = wk.q_pos0 + j0;
      const int qp1 = wk.q_pos0 + j1;
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
      for (int i = 0; i < 2 * KS; ++i) {
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
        for (int dp = 0; dp < KS; ++dp) {
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

  // merge the 4 warps' partial softmax states: row r = G * j + h of each warp tile is head kvh * G + h at query position
  // j.  The stages are free here (the loop's last barrier followed the last tile, and no gather is in flight).
  float* so = reinterpret_cast<float*>(smem);            // [4 warps][16 rows][D]
  float* sm = so + 4 * 16 * D;                           // [4][16]
  float* sl = sm + 4 * 16;                               // [4][16]
  const int nrows = G * wk.q_count;
  if (g < nrows) {
#pragma unroll
    for (int dn = 0; dn < 2 * KS; ++dn) {
      float2 v = make_float2(o[dn][0], o[dn][1]);
      *reinterpret_cast<float2*>(so + (warp * 16 + g) * D + dn * 8 + tq * 2) = v;
    }
    if (tq == 0) {
      sm[warp * 16 + g] = m0;
      sl[warp * 16 + g] = l0;
    }
  }
  if (g + 8 < nrows) {
#pragma unroll
    for (int dn = 0; dn < 2 * KS; ++dn) {
      float2 v = make_float2(o[dn][2], o[dn][3]);
      *reinterpret_cast<float2*>(so + (warp * 16 + g + 8) * D + dn * 8 + tq * 2) = v;
    }
    if (tq == 0) {
      sm[warp * 16 + g + 8] = m1;
      sl[warp * 16 + g + 8] = l1;
    }
  }
  __syncthreads();
  // 128 / D rows at a time: thread tid owns dim tid % D of rows tid / D, tid / D + 128 / D, ... (at D = 128 the block's
  // 128 threads make tid / D zero; it is spelled out so that the D = 128 code is the single-row loop)
  const int d = D == 128 ? tid : tid % D;
  for (int r = D == 128 ? 0 : tid / D; r < nrows; r += 128 / D) {
    const int j = r / G, h = r - j * G;
    float mm = -INFINITY;
#pragma unroll
    for (int w = 0; w < 4; ++w) mm = fmaxf(mm, sm[w * 16 + r]);
    float num = 0.f, den = 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const float mw = sm[w * 16 + r];
      const float wgt = (mw == -INFINITY) ? 0.f : exp2f(mw - mm);
      num += so[(w * 16 + r) * D + d] * wgt;
      den += sl[w * 16 + r] * wgt;
    }
    if (parts == 1) {
      out[static_cast<size_t>(wk.q_tok0 + j) * ldo + (kvh * G + h) * D + d] = __float2bfloat16_rn(den > 0.f ? num / den : 0.f);
    } else {
      // position j's slab of [position][work][kv head][part][G heads][D acc | max | sum]: a launch whose items all
      // have q_count == 1 uses slab 0 only
      const size_t slab = static_cast<size_t>(gridDim.y) * Hkv * parts * (G * (D + 2));
      float* dst = split_ws + j * slab + ((static_cast<size_t>(blockIdx.y) * Hkv + kvh) * parts + part) * (G * (D + 2)) +
                   h * (D + 2);
      dst[d] = num;
      if (d == 0) {
        dst[D] = mm;
        dst[D + 1] = den;
      }
    }
  }
}

// out[token, head, :] = sum_p acc_p 2^(m_p - M) / sum_p l_p 2^(m_p - M) over the parts of a split decode work item
template <int D>
__global__ void __launch_bounds__(128)
attn_merge_kernel(const float* __restrict__ split_ws, __nv_bfloat16* __restrict__ out, int ldo, const AttnWork* __restrict__ work,
                  int Hkv, int G, int parts) {
  griddep_enter();
  const AttnWork wk = work[blockIdx.y];
  // 128 / D rows at a time, as in the decode kernel's epilogue
  const int kvh = blockIdx.x, d = D == 128 ? threadIdx.x : threadIdx.x % D;
  const size_t slab = static_cast<size_t>(gridDim.y) * Hkv * parts * (G * (D + 2));
  for (int r = D == 128 ? 0 : threadIdx.x / D; r < G * wk.q_count; r += 128 / D) {
    const int j = r / G, h = r - j * G;
    const float* base = split_ws + j * slab + (static_cast<size_t>(blockIdx.y) * Hkv + kvh) * parts * (G * (D + 2));
    float mm = -INFINITY;
    for (int p = 0; p < parts; ++p) mm = fmaxf(mm, base[(p * G + h) * (D + 2) + D]);
    float num = 0.f, den = 0.f;
    for (int p = 0; p < parts; ++p) {
      const float* s = base + (p * G + h) * (D + 2);
      const float wgt = (s[D] == -INFINITY) ? 0.f : exp2f(s[D] - mm);
      num += s[d] * wgt;
      den += s[D + 1] * wgt;
    }
    out[static_cast<size_t>(wk.q_tok0 + j) * ldo + (kvh * G + h) * D + d] = __float2bfloat16_rn(den > 0.f ? num / den : 0.f);
  }
}

// One tensor map per (KV-layer base pointer, head size D): the layer is viewed as [rows][D] bf16 with 2 * D-byte rows,
// gathered in boxes of 16 rows x 64 columns (one page-head half at D = 128, one page-head at D = 64).  The row count is an
// upper bound, not the allocation size: the kernel only ever addresses pages named by the block table.  The key holds D
// because the allocator may hand a freed layer's address to a pool of the other head size.
}  // namespace

int kv_map_for(const void* kv_layer, CUtensorMap* out, int head_dim) {
  struct KeyHash {
    size_t operator()(const std::pair<const void*, int>& k) const { return std::hash<const void*>()(k.first) ^ k.second; }
  };
  static std::unordered_map<std::pair<const void*, int>, CUtensorMap, KeyHash> cache;
  static std::mutex mu;
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find({kv_layer, head_dim});
  if (it == cache.end()) {
    CUtensorMap tm;
    if ((reinterpret_cast<uintptr_t>(kv_layer) & 255) != 0) return -5;
    if (int rc = tmap_encode_bf16_2d(&tm, kv_layer, 1ull << 30, head_dim, head_dim, 16, 64, 1)) return rc;
    if (cache.size() > 4096) cache.clear();
    it = cache.emplace(std::make_pair(kv_layer, head_dim), tm).first;
  }
  *out = it->second;
  return 0;
}

namespace {

template <int GC, int D>
int launch_decode(const CUtensorMap& tm, dim3 grid, cudaStream_t st, const __nv_bfloat16* q, int ldq, __nv_bfloat16* out,
                  int ldo, const int* block_tables, int max_blocks, const AttnWork* work, int Hkv, int G, float scale_log2,
                  float* split_ws) {
  static std::atomic<unsigned long long> attr_done{0};
  if (!ensure_dynamic_smem(paged_attn_kernel<GC, D>, attn_smem_bytes<D>(), &attr_done)) return -3;
  launch_pdl(paged_attn_kernel<GC, D>, grid, dim3(128), attn_smem_bytes<D>(), st, tm, q, ldq, out, ldo, block_tables,
             max_blocks, work, Hkv, G, scale_log2, split_ws);
  if (cudaGetLastError() != cudaSuccess) return -2;
  if (grid.z > 1) {
    launch_pdl(attn_merge_kernel<D>, dim3(grid.x, grid.y), dim3(128), 0, st, static_cast<const float*>(split_ws), out, ldo, work, Hkv,
               G, static_cast<int>(grid.z));
    if (cudaGetLastError() != cudaSuccess) return -2;
  }
  return 0;
}

}  // namespace

size_t attn_split_ws_bytes(int num_work, int Hq, int parts, int max_q, int head_dim) {
  return static_cast<size_t>(max_q) * num_work * Hq * parts * (head_dim + 2) * sizeof(float);
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
                    cudaStream_t st, float* split_ws, int split, int head_dim) {
  if (num_work <= 0) return 0;
  if (!attn_group_ok(Hq, Hkv) || !attn_head_dim_ok(head_dim)) return -1;
  if (split > 1 && !split_ws) return -1;
  const int G = Hq / Hkv;
  CUtensorMap tm;
  if (int rc = kv_map_for(kv_layer, &tm, head_dim)) return rc;
  const float scale_log2 = scale * 1.4426950408889634f;
  dim3 grid(Hkv, num_work, split > 1 ? split : 1);
  const __nv_bfloat16* qq = static_cast<const __nv_bfloat16*>(q);
  __nv_bfloat16* oo = static_cast<__nv_bfloat16*>(out);
  if (head_dim == 64) {
    if (G == 4) return launch_decode<4, 64>(tm, grid, st, qq, ldq, oo, ldo, block_tables, max_blocks, work, Hkv, G, scale_log2, split_ws);
    return launch_decode<0, 64>(tm, grid, st, qq, ldq, oo, ldo, block_tables, max_blocks, work, Hkv, G, scale_log2, split_ws);
  }
  if (G == 4) return launch_decode<4, 128>(tm, grid, st, qq, ldq, oo, ldo, block_tables, max_blocks, work, Hkv, G, scale_log2, split_ws);
  return launch_decode<0, 128>(tm, grid, st, qq, ldq, oo, ldo, block_tables, max_blocks, work, Hkv, G, scale_log2, split_ws);
}

}  // namespace b200
