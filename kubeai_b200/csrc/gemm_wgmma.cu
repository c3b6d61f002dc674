// Dense projection GEMM for the per-step hot path (SURVEY.md §8a K4/K8/K9/K10/K11):
//     out[t, n] = sum_k X[t, k] * W[n, k]        (bf16 x bf16 -> fp32 -> bf16)
// which is what the reference backend computes for qkv_proj / o_proj / gate_up_proj / down_proj / lm_head (vLLM
// model_executor/models/llama.py:81-121, :157-233; weights stored [N, K] K-major, outputs rounded to bf16 between ops).
//
// H100 (sm_90a) design:
//   * "swap-AB": the 128-row weight slab is the wgmma M operand (two consumer warpgroups of 64 rows each), the token tile
//     (64 / 128 / 256 tokens) is the N operand, so a decode step streams every weight byte once per token tile.
//   * one producer thread issues TMA loads (128B swizzle) of the weight slab and the token tile into a ring of shared
//     memory stages guarded by full / empty mbarriers; the consumers run wgmma.mma_async on the stages directly.  The
//     weight loads of the first ring fill go out before the PDL dependency wait (weights are static).
//   * split-K: with fewer tiles than SMs (o_proj / down_proj / qkv of a decode step) each tile's K range is cut into S
//     pieces on S CTAs, launched as thread-block clusters of c consecutive pieces: c = S when S-CTA clusters of the
//     whole grid are resident at once, else the largest divisor of S that is (1 at worst).  Each CTA of a cluster
//     finishes a 1/c share of the tile's tokens: it sums them over the S pieces in split order (a fixed order: the
//     result does not depend on timing) and runs the epilogue on them.  With c = S the pieces are read from the peers'
//     shared memory (DSMEM); with c < S every piece goes to an L2 workspace and, per share, the last cluster to arrive
//     sums it.  A thread loads up to 16 float4 of a piece before it adds any, so a decode-step share costs about S
//     round trips.
//   * epilogues: the fp32 tile is staged in shared memory (reusing the ring) and rounded to bf16 once, the rounding point
//     of a bf16 GEMM output; the elementwise op that follows a projection (residual add, SiLU * up, RoPE + paged KV write,
//     per-slab argmax) is applied to that rounded value with the same arithmetic as the standalone kernels (elementwise.cu).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <type_traits>

#include "gemm.h"
#include "gemm3.h"
#include "launch.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kSlab = 128;                     // weight rows per CTA
constexpr int kBlockK = 64;                    // bf16 per k-block == one 128-byte swizzle span
constexpr int kThreads = 384;                  // warpgroup 0: TMA producer; warpgroups 1-2: wgmma consumers + epilogue
constexpr int kConsumers = 256;
constexpr int kABytes = kSlab * kBlockK * 2;   // 16 KB
constexpr int kRingBytes = 192 * 1024;
constexpr int kPitch = kSlab + 4;              // fp32 staging row pitch (bank-conflict-free fragment stores)
constexpr int kMaxSplits = 16;

template <int BN>
struct Cfg {
  static constexpr int kBBytes = BN * kBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = kRingBytes / kStageBytes;   // 8, 6, 4
  static constexpr int kMisc = 2048;                          // mbarriers, per-token norm scales, flags
  static constexpr int kSmem = 1024 + kStages * kStageBytes + kMisc;
  static_assert(BN * kPitch * 4 <= kStages * kStageBytes, "staging tile must fit in the ring");
  static_assert(kSmem <= 232448, "227 KB per block on sm_90");
};

// the two consumer warpgroups only (the producer warpgroup has left the main loop)
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory"); }

__device__ __forceinline__ float bf16r(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
__device__ __forceinline__ float ldbf(const __nv_bfloat16* p) { return __bfloat162float(*p); }

// f(integral_constant<W>) with W the narrowest of 64, 128, .., BN that is >= nw (nw a multiple of 64, <= BN)
template <int BN, class F>
__device__ __forceinline__ void dispatch_width(int nw, F&& f) {
  if constexpr (BN > 64) {
    if (nw <= BN - 64) return dispatch_width<BN - 64>(nw, f);
  }
  f(std::integral_constant<int, BN>{});
}

// HD: the head size of the ROPE_KV epilogue (128, or 64 for the qkv projection of a 64-dimensional-head model)
template <int BN, int HD>
__global__ void __launch_bounds__(kThreads, 1) gemm_wgmma_kernel(const __grid_constant__ Gemm3Params P, int S) {
  using C = Cfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (sbase - smem_u32(smem_raw));
  const uint32_t bar_base = sbase + C::kStages * C::kStageBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (C::kStages + s); };
  float* inv_s = reinterpret_cast<float*>(smem + C::kStages * C::kStageBytes + 256);   // [BN] per-token norm scale
  int* flag_s = reinterpret_cast<int*>(smem + C::kStages * C::kStageBytes + 256 + 4 * 256);
  float* stg = reinterpret_cast<float*>(smem);                                         // [BN][kPitch] after the main loop

  const int tid = threadIdx.x;
  const int tiles_n = (P.N + kSlab - 1) / kSlab, ntt = (P.T + BN - 1) / BN;
  // several token tiles: the token tile is the fastest-varying CTA index (grid (ntt, slabs, S)), so the CTAs that share a
  // weight slab run together and read it from HBM once.  One token tile: grid (slabs, 1, S).
  const int slab = ntt > 1 ? blockIdx.y : blockIdx.x, tt = ntt > 1 ? blockIdx.x : 0;
  const int n0 = slab * kSlab, t0 = tt * BN, split = blockIdx.z;
  const int KB = (P.K + kBlockK - 1) / kBlockK;
  const int kb0 = static_cast<int>(static_cast<long long>(split) * KB / S);
  const int kb1 = static_cast<int>(static_cast<long long>(split + 1) * KB / S);

  if (tid == 0) {
    tma_prefetch_desc(&P.tm_w);
    tma_prefetch_desc(&P.tm_x);
    for (int s = 0; s < C::kStages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), kConsumers / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();
  griddep_launch();

  if (tid < 128) {
    // ---------------- producer
    if (tid == 0) {
      // a decode step reads each weight byte once; several token tiles read a slab once per tile, close together in time
      const uint64_t w_hint = ntt > 1 ? kEvictNormal : kEvictFirst;
      // the first ring fill: weights are static, so their loads go out before the dependency wait and stream while the
      // previous kernel finishes; the token tiles (activations written by the previous kernels) only after it.  Every
      // stage is armed for all its bytes (weight slab and token tile) when its weight load is issued.  The 256-token
      // instance (prefill steps, launches of hundreds of µs) loads in order after the wait: at its register cap the early
      // loads cost it a spill.
      const int pre = BN < 256 ? min(C::kStages, kb1 - kb0) : 0;
      for (int i = 0; i < pre; ++i) {
        mbar_arrive_expect_tx(full_bar(i), C::kStageBytes);
        tma_load_2d(sbase + i * C::kStageBytes, &P.tm_w, full_bar(i), (kb0 + i) * kBlockK, n0, w_hint);
      }
      griddep_wait();
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        const uint32_t a = sbase + stage * C::kStageBytes;
        if (kb - kb0 >= pre) {
          mbar_wait(empty_bar(stage), phase ^ 1);
          mbar_arrive_expect_tx(full_bar(stage), C::kStageBytes);
          tma_load_2d(a, &P.tm_w, full_bar(stage), kb * kBlockK, n0, w_hint);
        }
        tma_load_2d(a + kABytes, &P.tm_x, full_bar(stage), kb * kBlockK, t0, kEvictLast);
        if (++stage == C::kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    if (S > 1 && cluster_nctas() > 1) {   // the producer warpgroup takes part in the consumers' cluster barrier phases
      cluster_arrive();
      cluster_wait();
      if (cluster_nctas() == S) cluster_arrive();
    }
    return;
  }

  // ---------------- consumers
  griddep_wait();   // activations, residual and norm sums come from the previous kernels
  const int ctid = tid - 128, wg = ctid >> 7, wtid = ctid & 127, warp = ctid >> 5, lane = tid & 31;
  if (P.pro == GEMM3_PRO_NORM) {
    for (int t = ctid; t < BN; t += kConsumers) {
      float s = 0.f;
      if (t0 + t < P.T)
        for (int i = 0; i < P.ssq_slabs; ++i) s += P.ssq_in[static_cast<size_t>(t0 + t) * P.ssq_slabs + i];
      inv_s[t] = rsqrtf(s / static_cast<float>(P.K) + P.eps);
    }
    consumer_sync();
  }
  float acc[BN / 2];   // acc[j * 32 + ..]: the m64n64 fragment of tokens [64 j, 64 j + 64) (ptx.cuh wgmma_m64nk16)
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;

  // One wgmma per k16 step covers NW tokens: the whole tile, or for the ragged last token tile the narrowest width that
  // covers its tokens (the accumulators past NW keep their zeros).  Each output is the same fp32 chain whatever NW is.
  // k-block kb is issued before kb - 1 is waited for: one k-block in flight, then kb - 1's ring stage goes back.
  auto mainloop = [&](auto width) {
    constexpr int NW = decltype(width)::value;
    float(&d)[NW / 2] = *reinterpret_cast<float(*)[NW / 2]>(acc);
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(full_bar(stage), phase);
      const uint32_t a = sbase + stage * C::kStageBytes;
      if (P.pro == GEMM3_PRO_NORM) {
        // B tile := RMSNorm(residual) in place, rounded like rmsnorm_kernel: bf16(bf16(x * inv) * w)
        uint8_t* b = smem + stage * C::kStageBytes + kABytes;
        for (int c = ctid; c < BN * 8; c += kConsumers) {
          const int r = c >> 3, k = kb * kBlockK + (((c & 7) ^ (r & 7)) << 3);
          uint4* p = reinterpret_cast<uint4*>(b + r * 128 + (c & 7) * 16);
          uint4 u = *p;
          __nv_bfloat16* h = reinterpret_cast<__nv_bfloat16*>(&u);
          const float inv = inv_s[r];
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const float w = k + e < P.K ? ldbf(P.norm_w + k + e) : 0.f;
            h[e] = __float2bfloat16_rn(bf16r(__bfloat162float(h[e]) * inv) * w);
          }
          *p = u;
        }
        fence_proxy_async();
        consumer_sync();
      }
      wgmma_fence();
#pragma unroll
      for (int k16 = 0; k16 < kBlockK / 16; ++k16)
        wgmma_m64nk16<NW>(d, gmma_desc(a + wg * (64 * 128) + k16 * 32), gmma_desc(a + kABytes + k16 * 32));
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
      prev = stage;
      if (++stage == C::kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();   // the last stage is not handed back: the producer has no more loads
  };
  dispatch_width<BN>(min(BN, (P.T - t0 + 63) & ~63), mainloop);

  // ---------------- stage the fp32 tile: stg[token][row]
  consumer_sync();   // every wgmma of both warpgroups has read its stages: the ring is free
  {
    const int r0 = wg * 64 + (wtid >> 5) * 16 + (lane >> 2);
#pragma unroll
    for (int q = 0; q < BN / 8; ++q) {
      const int t = q * 8 + (lane & 3) * 2;
      stg[t * kPitch + r0] = acc[q * 4 + 0];
      stg[(t + 1) * kPitch + r0] = acc[q * 4 + 1];
      stg[t * kPitch + r0 + 8] = acc[q * 4 + 2];
      stg[(t + 1) * kPitch + r0 + 8] = acc[q * 4 + 3];
    }
  }
  consumer_sync();
  const int t_end = min(BN, P.T - t0);
  // With S > 1 the S pieces of a tile are S / c clusters of c (launch()): cluster rank == split % c.  Rank r finishes
  // the share [ta, tb) of the tile's tokens, cut like the K range; with no split one CTA finishes them all.
  const int csize = S > 1 ? cluster_nctas() : 1, rank = split % csize;
  const int ta = rank * t_end / csize, tb = (rank + 1) * t_end / csize;
  if (S > 1) {
    // c == S: the peers' staged tiles are read through distributed shared memory once every piece is staged.  c < S:
    // every piece goes to an L2 workspace; once a cluster's pieces are all out, its rank-r CTA counts one arrival for
    // share r, and the CTA that brings the count to S / c sums that share.  Either way the sum runs in split order
    // (p0 + p1 + ..), so the result does not depend on timing, and lands in the summing CTA's own staging tile.
    const int tile = tt * tiles_n + slab;
    const float* ws = P.ws + static_cast<size_t>(tile) * S * (BN * kSlab);
    const bool dsm = csize == S;
    if (!dsm) {
      float* my = P.ws + (static_cast<size_t>(tile) * S + split) * (BN * kSlab);
      for (int i = ctid; i < BN * kSlab / 4; i += kConsumers) {
        const int t = (i * 4) / kSlab, r = (i * 4) % kSlab;
        __stcg(reinterpret_cast<float4*>(my) + i, *reinterpret_cast<const float4*>(stg + t * kPitch + r));
      }
      __threadfence();
    }
    if (csize > 1) {
      cluster_arrive();
      cluster_wait();
    } else {
      consumer_sync();
    }
    if (!dsm) {
      if (ctid == 0) {
        int* cnt = P.counters + ntt + tile * csize + rank;   // after the per-token-tile counters of normed_out
        const int prev = atomicAdd(cnt, 1);
        const int last = prev == S / csize - 1;
        if (last) *cnt = 0;   // every cluster has arrived: reset for the next launch
        *flag_s = last;
      }
      consumer_sync();
      if (!*flag_s) return;
      __threadfence();
    }
    // U float4 of the share per thread at a time, all S pieces of them loaded one piece after the other: U loads in
    // flight per thread, so the sum costs S round trips per U float4.  U is the whole tile's float4 per thread in the 64-
    // and 128-token instances (8 / 16): a share is one batch, as the whole tile is when one CTA sums it.  The 256-token
    // instance (32 per thread) takes 8 at a time: at its 168-register cap 16 would spill.  Float4 c + 256 u of the share
    // is row 8 u below float4 c.
    constexpr int kRow4 = kSlab / 4, kPer = BN * kRow4 / kConsumers, U = kPer <= 16 ? kPer : 8;
    constexpr int kRowsPerPass = kConsumers / kRow4;
    const int n4 = (tb - ta) * kRow4;
    auto sum_share = [&](auto load) {   // load(c, u, s): float4 c + 256 u of the share in piece s
      for (int c = ctid; c < n4; c += U * kConsumers) {
        float4 v[U], w[U];
#pragma unroll
        for (int u = 0; u < U; ++u)
          if (c + u * kConsumers < n4) v[u] = load(c, u, 0);
        for (int s = 1; s < S; ++s) {   // split order: p0 + p1 + .., whichever piece finished last
#pragma unroll
          for (int u = 0; u < U; ++u)
            if (c + u * kConsumers < n4) w[u] = load(c, u, s);
#pragma unroll
          for (int u = 0; u < U; ++u) {
            v[u].x += w[u].x; v[u].y += w[u].y; v[u].z += w[u].z; v[u].w += w[u].w;
          }
        }
        float* dst = stg + (ta + c / kRow4) * kPitch + (c % kRow4) * 4;
#pragma unroll
        for (int u = 0; u < U; ++u)
          if (c + u * kConsumers < n4) *reinterpret_cast<float4*>(dst + u * kRowsPerPass * kPitch) = v[u];
      }
    };
    if (dsm) {
      sum_share([&](int c, int u, int s) {
        const uint32_t a = smem_u32(stg + (ta + c / kRow4) * kPitch + (c % kRow4) * 4);
        return dsmem_ld_f4(dsmem_map(a, s) + u * kRowsPerPass * kPitch * 4);   // a peer's shared memory is contiguous
      });
    } else {
      sum_share([&](int c, int u, int s) {
        const float* p = ws + static_cast<size_t>(s) * (BN * kSlab) + (ta + c / kRow4) * kSlab + (c % kRow4) * 4;
        return __ldcg(reinterpret_cast<const float4*>(p + u * kRowsPerPass * kSlab));
      });
    }
    if (dsm) cluster_arrive();   // done reading the peers' tiles; the matching wait comes before this CTA exits
    consumer_sync();
  }

  // ---------------- epilogue: one warp per token, each lane 4 consecutive rows of the slab
  constexpr int kWarps = kConsumers / 32;
  const int slabs = tiles_n;
  if (P.epi == GEMM3_EPI_RESADD) {
    // the residual of 4 of the warp's tokens is read before any of them is written back: 4 round trips in flight per
    // lane instead of one
    for (int tl0 = ta + warp; tl0 < tb; tl0 += 4 * kWarps) {
      float res[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int tl = tl0 + j * kWarps, r = lane * 4 + e;
          res[j][e] = tl < tb && n0 + r < P.N ? ldbf(P.out + static_cast<size_t>(t0 + tl) * P.ldo + n0 + r) : 0.f;
        }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int tl = tl0 + j * kWarps, t = t0 + tl;
        if (tl >= tb) break;
        const float* row = stg + tl * kPitch;
        float ss = 0.f;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int r = lane * 4 + e;
          if (n0 + r < P.N) {
            const __nv_bfloat16 z = __float2bfloat16_rn(bf16r(row[r]) + res[j][e]);
            P.out[static_cast<size_t>(t) * P.ldo + n0 + r] = z;
            const float zf = __bfloat162float(z);
            ss += zf * zf;
          }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
        if (lane == 0 && P.ssq_out) P.ssq_out[static_cast<size_t>(t) * slabs + slab] = ss;
      }
    }
  }
  for (int tl = ta + warp; tl < tb && P.epi != GEMM3_EPI_RESADD; tl += kWarps) {
    const int t = t0 + tl;
    const float* row = stg + tl * kPitch;
    if (P.epi == GEMM3_EPI_PLAIN) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int r = lane * 4 + e;
        if (n0 + r < P.N) P.out[static_cast<size_t>(t) * P.ldo + n0 + r] = __float2bfloat16_rn(row[r]);
      }
    } else if (P.epi == GEMM3_EPI_SILU) {
      // rows 0..63 of the slab are gate rows, 64..127 the matching up rows; act columns [slab*64, slab*64+64)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int r = lane * 2 + e;
        const __nv_bfloat16 s = silu_bf16(bf16r(row[r]));
        P.out[static_cast<size_t>(t) * P.ldo + slab * 64 + r] = __float2bfloat16_rn(__bfloat162float(s) * bf16r(row[r + 64]));
      }
    } else if (P.epi == GEMM3_EPI_ROPE_KV && HD == 128) {
      // one 128-row slab = one head of the fused qkv projection
      const int head = slab;
      const size_t page_stride = static_cast<size_t>(P.Hkv) * 16 * 128;
      const int slot = head >= P.Hq ? __ldg(P.slots + t) : 0;
      if (head < P.Hq + P.Hkv) {
        int pos = __ldg(P.positions + t);
        pos = pos < 0 ? 0 : (pos >= P.max_pos ? P.max_pos - 1 : pos);
        const __nv_bfloat16* cs = P.cos_sin + static_cast<size_t>(pos) * 128;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int r = lane * 2 + e;
          const float a = bf16r(row[r]), b = bf16r(row[r + 64]);
          const float cc = ldbf(cs + r), sn = ldbf(cs + 64 + r);
          // every bf16 op rounds, as in elementwise.cu rope_kv_kernel
          const float ac = bf16r(__fmul_rn(a, cc)), bs = bf16r(__fmul_rn(b, sn));
          const float bc = bf16r(__fmul_rn(b, cc)), as = bf16r(__fmul_rn(a, sn));
          const __nv_bfloat16 o1 = __float2bfloat16_rn(ac - bs), o2 = __float2bfloat16_rn(bc + as);
          __nv_bfloat16* dst = nullptr;
          if (head < P.Hq) dst = P.out + static_cast<size_t>(t) * P.ldo + head * 128;
          else if (slot >= 0)
            dst = P.kv_layer + static_cast<size_t>(slot >> 4) * 2 * page_stride + (static_cast<size_t>(head - P.Hq) * 16 + (slot & 15)) * 128;
          if (dst) {
            dst[r] = o1;
            dst[r + 64] = o2;
          }
        }
      } else if (slot >= 0) {
        const int vh = head - P.Hq - P.Hkv;
        __nv_bfloat16* dst = P.kv_layer + static_cast<size_t>(slot >> 4) * 2 * page_stride + page_stride +
                             (static_cast<size_t>(vh) * 16 + (slot & 15)) * 128;
#pragma unroll
        for (int e = 0; e < 4; ++e) dst[lane * 4 + e] = __float2bfloat16_rn(row[lane * 4 + e]);
      }
    } else if (HD == 64 && P.epi == GEMM3_EPI_ROPE_KV) {
      // D = 64: one 128-row slab = two heads of the fused qkv projection (q heads, then k, then v); the rotation pairs
      // rows (r, r + 32) of a head.  Heads are classified one by one, so a slab may hold the last k head and the first v
      // head (an odd kv_heads).
      constexpr int hd_log2 = 6, half_log2 = 5, D = 64, HALF = 32;
      const int head0 = slab << (7 - hd_log2);           // first head of the slab
      const size_t page_stride = static_cast<size_t>(P.Hkv) * 16 * D;
      const int slot = head0 + (128 >> hd_log2) > P.Hq ? __ldg(P.slots + t) : 0;
      __nv_bfloat16* kpage = P.kv_layer + static_cast<size_t>(slot >> 4) * 2 * page_stride;
      if (head0 < P.Hq + P.Hkv) {
        int pos = __ldg(P.positions + t);
        pos = pos < 0 ? 0 : (pos >= P.max_pos ? P.max_pos - 1 : pos);
        const __nv_bfloat16* cs = P.cos_sin + (static_cast<size_t>(pos) << hd_log2);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int p = lane * 2 + e;                     // pair p of the slab's 64
          const int head = head0 + (p >> half_log2), r = p & (HALF - 1);
          const int ra = ((p >> half_log2) << hd_log2) + r;  // slab row of the pair's first element
          const float a = bf16r(row[ra]), b = bf16r(row[ra + HALF]);
          __nv_bfloat16 o1, o2;
          if (head < P.Hq + P.Hkv) {
            const float cc = ldbf(cs + r), sn = ldbf(cs + HALF + r);
            // every bf16 op rounds, as in elementwise.cu rope_kv_kernel
            const float ac = bf16r(__fmul_rn(a, cc)), bs = bf16r(__fmul_rn(b, sn));
            const float bc = bf16r(__fmul_rn(b, cc)), as = bf16r(__fmul_rn(a, sn));
            o1 = __float2bfloat16_rn(ac - bs);
            o2 = __float2bfloat16_rn(bc + as);
          } else {                                        // a v head sharing the slab with the last k head
            o1 = __float2bfloat16_rn(a);
            o2 = __float2bfloat16_rn(b);
          }
          __nv_bfloat16* dst = nullptr;
          if (head < P.Hq) dst = P.out + static_cast<size_t>(t) * P.ldo + (head << hd_log2);
          else if (slot >= 0)
            dst = kpage + (head < P.Hq + P.Hkv ? 0 : page_stride) +
                  ((static_cast<size_t>(head < P.Hq + P.Hkv ? head - P.Hq : head - P.Hq - P.Hkv) * 16 + (slot & 15)) << hd_log2);
          if (dst) {
            dst[r] = o1;
            dst[r + HALF] = o2;
          }
        }
      } else if (slot >= 0) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int rr = lane * 4 + e;
          const int vh = head0 + (rr >> hd_log2) - P.Hq - P.Hkv;
          __nv_bfloat16* dst = kpage + page_stride + ((static_cast<size_t>(vh) * 16 + (slot & 15)) << hd_log2);
          dst[rr & (D - 1)] = __float2bfloat16_rn(row[rr]);
        }
      }
    } else {  // GEMM3_EPI_ARGMAX: best bf16 logit of this slab, lowest index on ties
      const int nv = min(P.N, P.n_valid);
      float best = -INFINITY;
      int bi = 0x7fffffff;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int n = n0 + lane * 4 + e;
        if (n < nv) {
          const float v = bf16r(row[lane * 4 + e]);
          if (v > best) { best = v; bi = n; }
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
      }
      if (lane == 0) P.cand[static_cast<size_t>(t) * slabs + slab] = make_float2(best, __int_as_float(bi));
    }
  }

  if (S > 1 && csize == S) cluster_wait();   // no peer still reads this CTA's staging tile

  if (P.epi == GEMM3_EPI_RESADD && P.normed_out) {
    // RMSNorm of the new residual for the next projection: needs the sums of every slab of these tokens, so the last of
    // the token tile's slabs x c CTAs to finish its share does it
    __threadfence();
    consumer_sync();
    if (ctid == 0) {
      int* c = P.counters + tt;
      const int prev = atomicAdd(c, 1);
      const int last = prev == tiles_n * csize - 1;
      if (last) *c = 0;
      *flag_s = last;
    }
    consumer_sync();
    if (!*flag_s) return;
    __threadfence();
    for (int tl = warp; tl < t_end; tl += kConsumers / 32) {
      const int t = t0 + tl;
      float s = 0.f;
      for (int i = 0; i < slabs; ++i) s += __ldcg(P.ssq_out + static_cast<size_t>(t) * slabs + i);
      const float inv = rsqrtf(s / static_cast<float>(P.N) + P.eps);
      for (int n = lane; n < P.N; n += 32) {
        const __nv_bfloat16 z = __ldcg(P.out + static_cast<size_t>(t) * P.ldo + n);
        const __nv_bfloat16 nb = __float2bfloat16_rn(__bfloat162float(z) * inv);
        P.normed_out[static_cast<size_t>(t) * P.ldo + n] = __float2bfloat16_rn(__bfloat162float(nb) * ldbf(P.norm_w_out + n));
      }
    }
  }
}

// out[s] = index of the best logit of row s over its per-slab candidates (lowest index wins ties, sampler.py:91)
__global__ void argmax_cand_kernel(const float2* __restrict__ cand, int* __restrict__ out, int slabs) {
  griddep_enter();
  const int s = blockIdx.x;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = threadIdx.x; i < slabs; i += blockDim.x) {
    const float2 c = __ldcg(cand + static_cast<size_t>(s) * slabs + i);
    const int idx = __float_as_int(c.y);
    if (c.x > best || (c.x == best && idx < bi)) {
      best = c.x;
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

// ---------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p) return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

template <int BN, int HD>
int launch(const Gemm3Params& p, const Gemm3Schedule& sch, cudaStream_t st) {
  using C = Cfg<BN>;
  static std::atomic<unsigned long long> attr_done{0}, cluster_done{0};
  if (!ensure_dynamic_smem(gemm_wgmma_kernel<BN, HD>, C::kSmem, &attr_done)) return -3;
  // clusters of up to kMaxSplits (16) CTAs: above 8 the cluster size is not portable
  if (!ensure_func_attribute(gemm_wgmma_kernel<BN, HD>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1, &cluster_done))
    return -3;
  const int slabs = (p.N + kSlab - 1) / kSlab, ntt = (p.T + BN - 1) / BN;
  const dim3 grid = ntt > 1 ? dim3(ntt, slabs, sch.S) : dim3(slabs, 1, sch.S);   // see the kernel's CTA order
  // Clusters of c consecutive pieces of a tile: the largest c dividing S whose clusters are all resident at once.  A GPC
  // holds a whole number of clusters, so on a 132-SM H100 only 30 clusters of 4 fit where 32 would be needed for
  // Llama-3-8B's o_proj and down_proj; those run as 64 pairs.  The count is queried once per device and cluster size; a
  // size the query refuses counts as not fitting, down to c = 1 (no cluster).
  static std::atomic<int> max_clusters[64][kMaxSplits + 1];   // [device][c]: 1 + resident clusters, 0 until queried
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -3;
  std::atomic<int>* fit = max_clusters[dev & 63];
  int c = sch.S;
  for (; c > 1; --c) {
    if (sch.S % c) continue;
    if (fit[c].load(std::memory_order_relaxed) == 0) {
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = grid;
      cfg.blockDim = dim3(kThreads);
      cfg.dynamicSmemBytes = C::kSmem;
      cudaLaunchAttribute a[1];
      a[0].id = cudaLaunchAttributeClusterDimension;
      a[0].val.clusterDim.x = 1;
      a[0].val.clusterDim.y = 1;
      a[0].val.clusterDim.z = c;
      cfg.attrs = a;
      cfg.numAttrs = 1;
      int n = 0;
      if (cudaOccupancyMaxActiveClusters(&n, gemm_wgmma_kernel<BN, HD>, &cfg) != cudaSuccess) {
        cudaGetLastError();   // not an error of the launch: this size just does not fit
        n = 0;
      }
      fit[c].store(n + 1, std::memory_order_relaxed);
    }
    if (static_cast<long long>(grid.x) * grid.y * (sch.S / c) <= fit[c].load(std::memory_order_relaxed) - 1) break;
  }
  cudaError_t e = launch_pdl_cluster(gemm_wgmma_kernel<BN, HD>, grid, dim3(1, 1, c), dim3(kThreads), C::kSmem, st, p, sch.S);
  return e == cudaSuccess ? 0 : -4;
}

int g_variant = 2;
int g_num_sms = 0;

// Split count that fills a device of `sms` SMs with tiles x S CTAs, each split at least 4 k-blocks deep.
int fill_splits(int tiles, int KB, int sms) {
  int s = sms / tiles;
  const int by_k = KB / 4 > 0 ? KB / 4 : 1;
  if (s > by_k) s = by_k;
  if (s > kMaxSplits) s = kMaxSplits;
  return s < 1 ? 1 : s;
}

}  // namespace

void gemm_set_variant(int v) { g_variant = (v == 1) ? 1 : 2; }
int gemm_variant() { return g_variant; }

int num_sms() {
  if (g_num_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || g_num_sms <= 0) g_num_sms = 132;
  }
  return g_num_sms;
}

int gemm_block_n_for(int T) { return T <= 64 ? 64 : T <= 128 ? 128 : 256; }
int gemm_block_n_index(int bn) { return bn == 64 ? 0 : bn == 128 ? 1 : 2; }

int gemm_plan_init(GemmPlan* p, const void* W, int N, int K, int ldw, float* ws, size_t ws_bytes, int* counters, int counters_cap) {
  memset(p, 0, sizeof(*p));
  p->N = N;
  p->K = K;
  p->w_ptr = W;
  p->ldw = ldw;
  p->ws = ws;
  p->ws_bytes = ws_bytes;
  p->counters = counters;
  p->counters_cap = counters_cap;
  if (K % 8 != 0 || ldw % 8 != 0) return -5;
  return tmap_encode_bf16_2d(&p->tm_w, W, N, K, ldw, kSlab, kBlockK, 1);
}

// Generic 2-D bf16 map: row-major [rows, cols] with leading dimension ld (elements), box = box_rows x box_cols,
// 128-byte swizzle when box_cols * 2 == 128 and swizzle128 != 0.  Out-of-range rows and columns read as zero.
int tmap_encode_bf16_2d(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, int box_rows,
                        int box_cols, int swizzle128) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return -1;
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -2;
}

int gemm_make_x_map(CUtensorMap* tm, const void* X, int rows, int K, int ldx, int block_n) {
  if (ldx % 8 != 0) return -5;
  return tmap_encode_bf16_2d(tm, X, rows, K, ldx, block_n, kBlockK, 1);
}

int gemm3_schedule(int N, int K, int T, int force, Gemm3Schedule* out) { return gemm3_schedule_for(N, K, T, force, num_sms(), out); }

int gemm3_schedule_for(int N, int K, int T, int force, int sms, Gemm3Schedule* out) {
  if (N < 1 || K < 8 || K % 8 || T < 1 || sms < 1) return -1;
  const int KB = (K + kBlockK - 1) / kBlockK, tiles_n = (N + kSlab - 1) / kSlab;
  int bn = gemm_block_n_for(T);
  if (T > 128 && force != 0) {   // the largest tile the kernel has that does not exceed the request
    if (force < 64) return -4;
    bn = force >= 256 ? 256 : force >= 128 ? 128 : 64;
    force = 0;
  }
  const int tiles = tiles_n * ((T + bn - 1) / bn);
  int S, rule;
  if (force >= 1 || force < -1) {   // the caller's split count
    const int n = force > 0 ? force : -force;
    if (n > kMaxSplits || n > KB) return -4;
    S = n;
    rule = 0;
  } else {
    S = fill_splits(tiles, KB, sms);
    rule = T > 128 ? 2 : 1;
  }
  out->block_n = bn;
  out->S = S;
  out->rule = rule;
  out->grid = tiles * S;
  return 0;
}

size_t gemm3_ws_bytes(int N, const Gemm3Schedule& sch, int T) {
  if (sch.S <= 1) return 0;
  const size_t tiles = static_cast<size_t>((N + kSlab - 1) / kSlab) * ((T + sch.block_n - 1) / sch.block_n);
  return tiles * sch.S * sch.block_n * kSlab * sizeof(float);
}

int gemm3_counters_needed(int N, const Gemm3Schedule& sch, int T) {
  const int ntt = (T + sch.block_n - 1) / sch.block_n;
  return ntt + ((N + kSlab - 1) / kSlab) * ntt * sch.S;
}

int gemm3_launch(const Gemm3Params& p, const Gemm3Schedule& sch, cudaStream_t st) {
  if (p.T <= 0) return 0;
  if (sch.S < 1 || sch.S > kMaxSplits || sch.S > (p.K + kBlockK - 1) / kBlockK) return -6;
  if (gemm3_ws_bytes(p.N, sch, p.T) > p.ws_bytes || gemm3_counters_needed(p.N, sch, p.T) > p.counters_cap) return -9;
  if ((p.epi == GEMM3_EPI_SILU || p.epi == GEMM3_EPI_ROPE_KV) && p.N % kSlab) return -5;   // whole heads / gate-up slab pairs
  if (p.epi == GEMM3_EPI_RESADD && p.normed_out && (!p.ssq_out || !p.norm_w_out)) return -5;
  if (p.pro == GEMM3_PRO_NORM && (!p.ssq_in || !p.norm_w)) return -5;
  if (p.epi == GEMM3_EPI_ROPE_KV && p.head_dim != 0 && p.head_dim != 64 && p.head_dim != 128) return -5;
  if (p.epi == GEMM3_EPI_ROPE_KV && p.head_dim == 64) {
    switch (sch.block_n) {
      case 64: return launch<64, 64>(p, sch, st);
      case 128: return launch<128, 64>(p, sch, st);
      case 256: return launch<256, 64>(p, sch, st);
      default: return -6;
    }
  }
  switch (sch.block_n) {
    case 64: return launch<64, 128>(p, sch, st);
    case 128: return launch<128, 128>(p, sch, st);
    case 256: return launch<256, 128>(p, sch, st);
    default: return -6;
  }
}

int gemm_run(const GemmPlan& p, const CUtensorMap& tm_x, int block_n, void* out, int ldo, int T, cudaStream_t st) {
  if (T <= 0) return 0;
  Gemm3Schedule sch;
  if (int rc = gemm3_schedule(p.N, p.K, T, 0, &sch)) return rc;
  if (sch.block_n != block_n) return -6;
  if (g_variant == 1) {
    sch.S = 1;
    sch.grid = ((p.N + kSlab - 1) / kSlab) * ((T + block_n - 1) / block_n);
  }
  Gemm3Params q;
  memset(&q, 0, sizeof(q));
  q.tm_w = p.tm_w;
  q.tm_x = tm_x;
  q.N = p.N; q.T = T; q.K = p.K;
  q.pro = GEMM3_PRO_NONE; q.epi = GEMM3_EPI_PLAIN;
  q.out = static_cast<__nv_bfloat16*>(out);
  q.ldo = ldo;
  q.n_valid = p.N;
  q.ws = p.ws; q.ws_bytes = p.ws_bytes;
  q.counters = p.counters; q.counters_cap = p.counters_cap;
  return gemm3_launch(q, sch, st);
}

int argmax_candidates(const void* cand, int* out, int S, int slabs, cudaStream_t st) {
  if (S <= 0) return 0;
  launch_pdl(argmax_cand_kernel, dim3(S), dim3(256), 0, st, static_cast<const float2*>(cand), out, slabs);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

}  // namespace b200
