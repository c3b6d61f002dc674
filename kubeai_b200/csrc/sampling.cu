// Token selection for sampled rows (SURVEY.md §8a K11): temperature, top-k, top-p and a seeded exponential race over
// bf16 logits.  Semantics are vLLM V1's (vllm/v1/sample/sampler.py:223-297, ops/topk_topp_sampler.py:328-416), made
// deterministic:
//   - temperature < 1e-5: argmax, lowest index on ties (the same token as argmax_kernel in elementwise.cu);
//   - z_v = float(l_v) / temperature (fp32);
//   - min_p keeps every token with fp32 (z_v - z_max) >= log(min_p) (compared in double): vLLM's p_v >= min_p * p_max as a
//     fixed predicate, monotone in z, so it is one more key threshold;
//   - top-k keeps every token whose z is >= the k-th largest z (ties at the k-th value are kept);
//   - top-p keeps token v iff the softmax mass of the min_p- and top-k-kept tokens with z strictly greater than z_v is < p,
//     so tie groups are kept or dropped whole;
//   - the token is the argmax over the kept tokens of z_v - log(E_v), E_v = -log(u_v) ~ Exp(1) (the probs / q race of
//     vLLM's random_sample), lowest index on ties.  u_v = ((x >> 9) + 0.5) * 2^-23 is exact in fp32 and strictly inside
//     (0, 1); x is word v & 3 of Philox4x32-10 with counter (v >> 2, n, 0, 0) and key (seed_lo, seed_hi).
// The result is a pure function of (logits row, parameters, seed, n): it does not depend on the batch, the row's place in
// it, or the order in which threads run.
//
// One CTA per row, no sort.  bf16 logits have at most 65536 distinct values, each with an order-preserving 16-bit key, and
// temperature is monotonic, so both thresholds are keys.  They are found with a 256-bin histogram over the high byte of the
// key, then one over the low byte inside the bin that holds the threshold.  Each bin holds a count and a fixed-point mass
// floor(exp(z_v - z_max) * 2^40); both are summed with integer shared-memory atomics, whose result does not depend on
// arrival order (2^40 * 2^17 tokens fits in 64 bits).  The passes re-read the row (250 KB at Llama-3's vocabulary), which
// is still in L2 right after the lm_head:
//   1 row max (top-p, min_p)   2 high-byte histogram   3 low-byte histogram of the top-k bin   3b the same for the min_p
//   bin, when min_p cuts deeper than top-k under top-p   4 the same for the top-p bin (skipped when pass 3 / 3b holds it)
//   5 the race over the tokens at or above the threshold.  min_p's key is found by a binary search over the 65536 keys.
// Rows with temperature only run pass 5 alone.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "kernels.h"
#include "launch.h"
#include "ptx.cuh"

namespace b200 {

namespace {

constexpr int kThreads = 1024;
constexpr float kSamplingEps = 1e-5f;            // vllm/v1/sample/sampler.py _SAMPLING_EPS
constexpr float kMassScale = 1099511627776.0f;   // 2^40
constexpr int kPrivSmem = 256 * 32 * (8 + 4);     // 32 copies of a 256-bin (mass, count) histogram: 96 KiB

__device__ __forceinline__ void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint32_t lo0 = 0xD2511F53u * c[0], hi0 = __umulhi(0xD2511F53u, c[0]);
    const uint32_t lo1 = 0xCD9E8D57u * c[2], hi1 = __umulhi(0xCD9E8D57u, c[2]);
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
    c[0] = n0;
    c[1] = lo1;
    c[2] = n2;
    c[3] = lo0;
  }
}

// order-preserving key of a bf16 bit pattern (-0 and +0 share one key: they are the same logit)
__device__ __forceinline__ uint32_t key_of(uint32_t b) {
  if (b == 0x8000u) b = 0;
  return (b & 0x8000u) ? (~b & 0xFFFFu) : (b | 0x8000u);
}
__device__ __forceinline__ uint32_t bits_of_key(uint32_t k) { return (k & 0x8000u) ? (k & 0x7FFFu) : (~k & 0xFFFFu); }
__device__ __forceinline__ float bf16_bits_to_f32(uint32_t b) { return __uint_as_float(b << 16); }

// Visit every token of the row, 8 at a time from 16-byte loads (two loads in flight per thread), then the scalar tail.
template <class F>
__device__ __forceinline__ void visit_row(const uint16_t* __restrict__ row, int V, F&& f) {
  const int nvec = V >> 3;
  const uint4* r4 = reinterpret_cast<const uint4*>(row);
  for (int i = threadIdx.x; i < nvec; i += 2 * kThreads) {
    const int i2 = i + kThreads;
    const uint4 a = r4[i];
    const uint4 c = i2 < nvec ? r4[i2] : make_uint4(0, 0, 0, 0);
    const uint32_t wa[4] = {a.x, a.y, a.z, a.w}, wc[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) f(i * 8 + j, (wa[j >> 1] >> ((j & 1) * 16)) & 0xFFFFu);
    if (i2 < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) f(i2 * 8 + j, (wc[j >> 1] >> ((j & 1) * 16)) & 0xFFFFu);
    }
  }
  for (int v = nvec * 8 + threadIdx.x; v < V; v += kThreads) f(v, static_cast<uint32_t>(row[v]));
}

// (score, index) argmax over the CTA, lowest index on ties (argmax_kernel's reduction)
__device__ __forceinline__ int block_argmax(float best, int bi, float* sb, int* si) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) {
      best = ob;
      bi = oi;
    }
  }
  if ((threadIdx.x & 31) == 0) {
    sb[threadIdx.x >> 5] = best;
    si[threadIdx.x >> 5] = bi;
  }
  __syncthreads();
  best = sb[threadIdx.x & 31];
  bi = si[threadIdx.x & 31];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) {
      best = ob;
      bi = oi;
    }
  }
  return bi;
}

// One warp: the largest bin b with pred(above + sum(h[b..255])), or -1.  The suffix sum does not increase with b and pred
// is true for large sums, so the answer is the top of the run of bins where it holds.  *above_b gets sum(h[b+1..255]).
template <class T, class Pred>
__device__ __forceinline__ int warp_last_bin(const T* h, unsigned long long above, Pred pred, unsigned long long* above_b) {
  const int lane = threadIdx.x & 31;
  unsigned long long loc[8], chunk = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    loc[j] = static_cast<unsigned long long>(h[lane * 8 + j]);
    chunk += loc[j];
  }
  unsigned long long incl = chunk;   // sum over lanes >= this lane
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long v = __shfl_down_sync(0xffffffffu, incl, o);
    if (lane + o < 32) incl += v;
  }
  unsigned long long run = incl - chunk, before = 0;
  int best = -1;
#pragma unroll
  for (int j = 7; j >= 0; --j) {
    const unsigned long long prev = run;
    run += loc[j];
    if (best < 0 && pred(above + run)) {
      best = lane * 8 + j;
      before = prev;
    }
  }
  const unsigned bal = __ballot_sync(0xffffffffu, best >= 0);
  if (!bal) return -1;
  const int src = 31 - __clz(bal);
  *above_b = __shfl_sync(0xffffffffu, before, src);
  return __shfl_sync(0xffffffffu, best, src);
}

__global__ void __launch_bounds__(kThreads) sample_kernel(const uint16_t* __restrict__ logits, int ld,
                                                          const int32_t* __restrict__ rows, int row_words, int V,
                                                          int* __restrict__ out) {
  __shared__ uint32_t cnt_hi[256], cnt_lo[256];
  __shared__ unsigned long long mass_hi[256], mass_lo[256];
  __shared__ float sb[32];
  __shared__ int si[32];
  __shared__ uint32_t s_kmax, s_thr, s_tm;
  extern __shared__ __align__(16) unsigned char dyn_smem[];   // kPrivSmem: per-lane histogram copies
  unsigned long long* priv_mass = reinterpret_cast<unsigned long long*>(dyn_smem);
  uint32_t* priv_cnt = reinterpret_cast<uint32_t*>(dyn_smem + 256 * 32 * sizeof(unsigned long long));
  griddep_enter();
  const int s = blockIdx.x;
  const uint16_t* row = logits + static_cast<size_t>(s) * ld;
  // rows of 6 words carry no min_p (steps without a min_p row keep their size)
  SampleRow P;
  memcpy(&P, rows + static_cast<size_t>(s) * row_words, 6 * sizeof(int32_t));
  P.min_p = row_words > 6 ? __int_as_float(rows[static_cast<size_t>(s) * row_words + 6]) : 0.f;

  if (!(P.temperature >= kSamplingEps)) {
    // greedy: argmax_kernel's comparisons, so the same token
    float best = -INFINITY;
    int bi = 0x7fffffff;
    visit_row(row, V, [&](int v, uint32_t b) {
      const float f = bf16_bits_to_f32(b);
      if (f > best || (f == best && v < bi)) {
        best = f;
        bi = v;
      }
    });
    bi = block_argmax(best, bi, sb, si);
    if (threadIdx.x == 0) out[s] = bi == 0x7fffffff ? 0 : bi;
    return;
  }

  const float T = P.temperature;
  const bool topk_on = P.top_k > 0 && P.top_k < V;
  const bool topp_on = P.top_p > 0.f && P.top_p < 1.f;
  const bool minp_on = P.min_p > 0.f;
  uint32_t thr = 0;   // the race runs over the tokens with key >= thr
  float zmax = 0.f;
  uint32_t tm = 0;    // min_p: the smallest kept key
  if (topp_on || minp_on) {
    // pass 1: row max, as a key (an integer max does not depend on order)
    uint32_t km = 0;
    visit_row(row, V, [&](int, uint32_t b) { km = max(km, key_of(b)); });
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) km = max(km, __shfl_xor_sync(0xffffffffu, km, o));
    if (threadIdx.x == 0) s_kmax = 0;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) atomicMax(&s_kmax, km);
    __syncthreads();
    zmax = __fdiv_rn(bf16_bits_to_f32(bits_of_key(s_kmax)), T);
    if (minp_on) {
      // the smallest key t with (z(t) - z_max) >= log(min_p): the row max satisfies it (min_p <= 1), and -NaN keys sit
      // below -inf and fail it, so the predicate is false then true along the keys.  A +NaN key sits above +inf: a row
      // holding +NaN has a NaN z_max, no key passes, tm is the NaN key and the race (NaN scores never win) returns token 0
      // (so does top-p there: every mass is 0, so tp is 0xFFFF).  Greedy, temperature-only and top-k rows skip the NaN.
      if (threadIdx.x == 0) {
        const double lm = log(static_cast<double>(P.min_p));
        uint32_t lo = 0, hi = s_kmax;
        while (lo < hi) {
          const uint32_t mid = (lo + hi) >> 1;
          const float d = __fsub_rn(__fdiv_rn(bf16_bits_to_f32(bits_of_key(mid)), T), zmax);
          if (static_cast<double>(d) >= lm) hi = mid;
          else lo = mid + 1;
        }
        s_tm = lo;
      }
      __syncthreads();
      tm = s_tm;
    }
  }
  if (topk_on || topp_on) {
    auto fixed_mass = [&](uint32_t b) {
      const float m = expf(__fsub_rn(__fdiv_rn(bf16_bits_to_f32(b), T), zmax));   // in [0, 1]
      return __float2ull_rz(__fmul_rn(m, kMassScale));
    };
    // bin < 0: histogram of the high byte of every key; else of the low byte of the keys whose high byte is `bin`.
    // Logits fall into a dozen high-byte bins (sign and exponent), so every lane adds into its own copy of the
    // histogram (copy = lane, bank = lane: no two lanes of an atomic instruction collide); the copies are then summed.
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    auto histogram = [&](int bin, uint32_t* c, unsigned long long* m) {
      for (int i = threadIdx.x; i < 256 * 32; i += kThreads) {
        priv_cnt[i] = 0;
        priv_mass[i] = 0;
      }
      __syncthreads();
      visit_row(row, V, [&](int, uint32_t b) {
        const uint32_t k = key_of(b);
        if (bin >= 0 && static_cast<int>(k >> 8) != bin) return;
        const uint32_t slot = (bin >= 0 ? (k & 0xFFu) : (k >> 8)) * 32 + lane;
        if (topk_on) atomicAdd(&priv_cnt[slot], 1u);          // counts serve top-k, masses top-p
        if (topp_on) atomicAdd(&priv_mass[slot], fixed_mass(b));
      });
      __syncthreads();
      for (int j = warp; j < 256; j += kThreads / 32) {
        uint32_t cs = priv_cnt[j * 32 + lane];
        unsigned long long ms = priv_mass[j * 32 + lane];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          cs += __shfl_xor_sync(0xffffffffu, cs, o);
          ms += __shfl_xor_sync(0xffffffffu, ms, o);
        }
        if (lane == 0) {
          c[j] = cs;
          m[j] = ms;
        }
      }
      __syncthreads();
    };
    const bool lead = threadIdx.x < 32;
    histogram(-1, cnt_hi, mass_hi);   // pass 2
    // top-k: the k-th largest key = the largest key t with count(key >= t) >= k
    int bk = -1;
    uint32_t tk = 0;
    unsigned long long z = 0;   // fixed-point mass of the top-k-kept tokens
    if (topk_on) {
      const unsigned long long k = static_cast<unsigned long long>(P.top_k);
      auto reach = [&](unsigned long long c) { return c >= k; };
      unsigned long long cab = 0, unused = 0;
      if (lead) bk = warp_last_bin(cnt_hi, 0ull, reach, &cab);   // k <= V - 1: always found
      if (threadIdx.x == 0) s_thr = static_cast<uint32_t>(bk);
      __syncthreads();
      bk = static_cast<int>(s_thr);
      histogram(bk, cnt_lo, mass_lo);   // pass 3
      if (lead) {
        const int lo = warp_last_bin(cnt_lo, cab, reach, &unused);
        tk = (static_cast<uint32_t>(bk) << 8) | static_cast<uint32_t>(lo);
        if (topp_on) {
          // mass of the kept tokens: the bins above bk and the keys >= tk inside it
          unsigned long long m = 0;
          for (int i = threadIdx.x; i < 256; i += 32) m += (i > bk ? mass_hi[i] : 0ull) + (i >= lo ? mass_lo[i] : 0ull);
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) m += __shfl_xor_sync(0xffffffffu, m, o);
          z = m;
        }
      }
    } else if (topp_on && lead) {
      unsigned long long m = 0;
      for (int i = threadIdx.x; i < 256; i += 32) m += mass_hi[i];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m += __shfl_xor_sync(0xffffffffu, m, o);
      z = m;
    }
    int lo_bin = topk_on ? bk : -1;   // the high-byte bin whose low-byte histograms cnt_lo / mass_lo hold
    if (topp_on && minp_on) {
      // top-p runs over the mass of the tokens at or above max(tk, tm): when min_p cuts deeper, that is the bins above
      // tm's and the keys >= tm inside it
      const int bm = static_cast<int>(tm >> 8);
      if (bm != lo_bin) histogram(bm, cnt_lo, mass_lo);   // pass 3b
      lo_bin = bm;
      if (lead && tm > tk) {
        unsigned long long m = 0;
        for (int i = threadIdx.x; i < 256; i += 32)
          m += (i > bm ? mass_hi[i] : 0ull) + (i >= static_cast<int>(tm & 0xFFu) ? mass_lo[i] : 0ull);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m += __shfl_xor_sync(0xffffffffu, m, o);
        z = m;
      }
    }
    uint32_t tp = 0;
    if (topp_on) {
      // top-p: keep v iff mass(kept, key > key_v) < p * z, i.e. key_v >= the largest key t with mass(kept, key >= t) >=
      // p * z.  Every high-byte bin at or below bk holds at least z >= p * z of kept mass, so the search over the whole-row
      // histogram lands at or above bk, and above bk every token is kept.
      const double X = static_cast<double>(P.top_p) * static_cast<double>(z);
      auto reach = [&](unsigned long long m) { return static_cast<double>(m) >= X; };
      unsigned long long mab = 0, unused = 0;
      int bp = 0;
      if (lead) bp = warp_last_bin(mass_hi, 0ull, reach, &mab);
      if (threadIdx.x == 0) s_thr = static_cast<uint32_t>(bp);
      __syncthreads();
      bp = static_cast<int>(s_thr);
      if (bp != lo_bin) histogram(bp, cnt_lo, mass_lo);   // pass 4 (pass 3 / 3b already holds bin lo_bin)
      if (lead) {
        const int lo = warp_last_bin(mass_lo, mab, reach, &unused);
        tp = (static_cast<uint32_t>(bp) << 8) | static_cast<uint32_t>(lo);
      }
    }
    __syncthreads();   // every reader of s_thr is past it
    if (threadIdx.x == 0) s_thr = max(max(tk, tp), tm);
    __syncthreads();
    thr = s_thr;
  } else {
    thr = tm;
  }

  // pass 5: the exponential race over the tokens with key >= thr
  const uint32_t seed_lo = P.seed_lo, seed_hi = P.seed_hi, n = static_cast<uint32_t>(P.n);
  float best = -INFINITY;
  int bi = 0x7fffffff;
  int group = -1;
  uint32_t w[4] = {0, 0, 0, 0};
  visit_row(row, V, [&](int v, uint32_t b) {
    if (key_of(b) < thr) return;
    if ((v >> 2) != group) {
      group = v >> 2;
      w[0] = static_cast<uint32_t>(group); w[1] = n; w[2] = 0; w[3] = 0;
      philox4x32_10(w, seed_lo, seed_hi);
    }
    const uint32_t x = w[v & 3];
    const float u = __fmul_rn(__fadd_rn(static_cast<float>(x >> 9), 0.5f), 1.0f / 8388608.0f);   // exact, in (0, 1)
    const float e = -logf(u);
    const float score = __fsub_rn(__fdiv_rn(bf16_bits_to_f32(b), T), logf(e));
    if (score > best || (score == best && v < bi)) {
      best = score;
      bi = v;
    }
  });
  bi = block_argmax(best, bi, sb, si);
  if (threadIdx.x == 0) out[s] = bi == 0x7fffffff ? 0 : bi;
}

// Log-probabilities of one row per CTA, vLLM V1's raw_logprobs (vllm/v1/sample/sampler.py compute_logprobs /
// gather_logprobs) made deterministic: lp_v = (l_v - m) - log(sum_u exp(l_u - m)) in fp32, m = the row max.  Each thread
// sums its tokens in visit order, then a fixed shuffle tree adds the 1024 partials, so the sum (and every lp) is a pure
// function of the row.  The top N are chosen by 16-bit key (exact bf16 order; -0 and +0 are one key), lowest id on ties:
//   1 row max   2 sum of exp + high-byte count histogram   3 low-byte count histogram of the bin of the N-th key
//   4 collect the keys above the N-th key and the ties at it, then rank the <= 20 + kTieCap entries.
// When more than kTieCap tokens tie at the N-th key they are taken in id order by a chunked ballot scan instead (slow, rare
// on real logits).  Rows with N = 0 stop after pass 2 and the sampled token's gather.
// kRank adds the token's rank, vLLM's batched_count_greater_than: the number of tokens whose key is >= the token's key
// (so equal logits share a rank, and -0 / +0 are one key).  It is counted exactly in pass 2, with integer adds whose sum
// does not depend on order, so no extra pass reads the row; N = 0 rows get it too.  Without kRank the kernel is the same
// code as before ranks existed.
constexpr int kTieCap = 64;
constexpr int kCntSmem = 256 * 32 * 4;   // 32 per-lane copies of a 256-bin count histogram: 32 KiB

template <bool kRank>
__global__ void __launch_bounds__(kThreads) logprobs_kernel(const uint16_t* __restrict__ logits, int ld, int V,
                                                            const int* __restrict__ rows, const int* __restrict__ top_n,
                                                            const int* __restrict__ tokens, float* __restrict__ out_lp,
                                                            int lp_ld, float* __restrict__ out_top_lp, int top_lp_ld,
                                                            int* __restrict__ out_top_ids, int* __restrict__ out_rank) {
  __shared__ uint32_t cnt_hi[256], cnt_lo[256];
  __shared__ float sred[32];
  __shared__ int swc[32];
  __shared__ uint32_t s_kmax, s_thr, s_count, s_above, s_need, s_ties, s_rank;
  __shared__ float s_logz;
  __shared__ uint32_t ent_key[kMaxLogprobs + kTieCap];
  __shared__ int ent_id[kMaxLogprobs + kTieCap];
  extern __shared__ __align__(16) uint32_t priv_cnt[];   // kCntSmem
  griddep_enter();
  const int i = blockIdx.x;
  const int r = rows ? rows[i] : i;
  const uint16_t* row = logits + static_cast<size_t>(r) * ld;
  const int N = min(max(top_n[i], 0), min(V, kMaxLogprobs));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t kt = 0;   // kRank: the token's key (above every key when the id is out of range: rank 0)
  if (kRank) {
    const int t = tokens[r];
    kt = (t >= 0 && t < V) ? key_of(row[t]) : 0x10000u;
  }

  // pass 1: row max, as a key
  uint32_t km = 0;
  visit_row(row, V, [&](int, uint32_t b) { km = max(km, key_of(b)); });
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) km = max(km, __shfl_xor_sync(0xffffffffu, km, o));
  if (threadIdx.x == 0) s_kmax = 0;
  if (kRank && threadIdx.x == 0) s_rank = 0;
  if (N > 0)
    for (int j = threadIdx.x; j < 256 * 32; j += kThreads) priv_cnt[j] = 0;
  __syncthreads();
  if (lane == 0) atomicMax(&s_kmax, km);
  __syncthreads();
  const float m = bf16_bits_to_f32(bits_of_key(s_kmax));

  // pass 2: sum of exp (fixed order) and the high-byte histogram (per-lane copies: no bank collisions within a warp)
  float acc = 0.f;
  uint32_t ge = 0;   // kRank: tokens with key >= kt
  visit_row(row, V, [&](int, uint32_t b) {
    acc = __fadd_rn(acc, expf(__fsub_rn(bf16_bits_to_f32(b), m)));
    if (N > 0) atomicAdd(&priv_cnt[(key_of(b) >> 8) * 32 + lane], 1u);
    if (kRank) ge += key_of(b) >= kt ? 1u : 0u;
  });
  if (kRank) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ge += __shfl_xor_sync(0xffffffffu, ge, o);
    if (lane == 0) atomicAdd(&s_rank, ge);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc = __fadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, o));
  if (lane == 0) sred[warp] = acc;
  __syncthreads();
  if (warp == 0) {
    float t = sred[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t = __fadd_rn(t, __shfl_xor_sync(0xffffffffu, t, o));
    if (lane == 0) s_logz = logf(t);
  }
  __syncthreads();
  const float logz = s_logz;
  // the same arithmetic for every token of one key, so equal logits (and -0 / +0) get the same bits
  auto lp_of_key = [&](uint32_t k) { return __fsub_rn(__fsub_rn(bf16_bits_to_f32(bits_of_key(k)), m), logz); };
  if (threadIdx.x == 0) {
    const int t = tokens[r];
    out_lp[static_cast<size_t>(i) * lp_ld] = (t >= 0 && t < V) ? lp_of_key(key_of(row[t])) : __int_as_float(0x7fc00000);
    if (kRank) out_rank[i] = static_cast<int>(s_rank);
  }
  if (N == 0) return;

  auto reduce_hist = [&](uint32_t* c) {
    __syncthreads();
    for (int j = warp; j < 256; j += kThreads / 32) {
      uint32_t cs = priv_cnt[j * 32 + lane];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) cs += __shfl_xor_sync(0xffffffffu, cs, o);
      if (lane == 0) c[j] = cs;
    }
    __syncthreads();
  };
  const unsigned long long need_n = static_cast<unsigned long long>(N);
  auto reach = [&](unsigned long long c) { return c >= need_n; };
  reduce_hist(cnt_hi);
  int bk = 0;
  unsigned long long cab = 0;
  if (warp == 0) bk = warp_last_bin(cnt_hi, 0ull, reach, &cab);   // N <= V: always found
  if (threadIdx.x == 0) {
    s_thr = static_cast<uint32_t>(bk);
    s_above = static_cast<uint32_t>(cab);
  }
  for (int j = threadIdx.x; j < 256 * 32; j += kThreads) priv_cnt[j] = 0;
  __syncthreads();
  bk = static_cast<int>(s_thr);

  // pass 3: low-byte histogram inside the bin of the N-th key
  visit_row(row, V, [&](int, uint32_t b) {
    const uint32_t k = key_of(b);
    if (static_cast<int>(k >> 8) == bk) atomicAdd(&priv_cnt[(k & 0xFFu) * 32 + lane], 1u);
  });
  reduce_hist(cnt_lo);
  if (warp == 0) {
    unsigned long long above_lo = 0;
    const int lo = warp_last_bin(cnt_lo, static_cast<unsigned long long>(s_above), reach, &above_lo);
    if (lane == 0) {
      s_thr = (static_cast<uint32_t>(bk) << 8) | static_cast<uint32_t>(lo);
      s_above += static_cast<uint32_t>(above_lo);   // tokens with a key above the N-th key: < N
      s_need = static_cast<uint32_t>(N) - s_above;   // ties at it to keep, >= 1
      s_ties = cnt_lo[lo];
      s_count = 0;
    }
  }
  __syncthreads();
  const uint32_t thr = s_thr;
  const bool few_ties = s_ties <= static_cast<uint32_t>(kTieCap);

  // pass 4: every key above the threshold (< 20 of them) and, when they are few, every tie at it
  visit_row(row, V, [&](int v, uint32_t b) {
    const uint32_t k = key_of(b);
    if (k > thr || (few_ties && k == thr)) {
      const uint32_t slot = atomicAdd(&s_count, 1u);
      ent_key[slot] = k;
      ent_id[slot] = v;
    }
  });
  __syncthreads();
  int count = static_cast<int>(s_count);
  if (!few_ties) {
    // the lowest-id ties, 1024 ids at a time in id order (CTA-uniform loop)
    int slot = count, need = static_cast<int>(s_need);
    for (int c = 0; c < V && need > 0; c += kThreads) {
      const int v = c + static_cast<int>(threadIdx.x);
      const bool tie = v < V && key_of(row[v]) == thr;
      const unsigned bal = __ballot_sync(0xffffffffu, tie);
      if (lane == 0) swc[warp] = __popc(bal);
      __syncthreads();
      int before = 0, total = 0;
      for (int w = 0; w < kThreads / 32; ++w) {
        before += w < warp ? swc[w] : 0;
        total += swc[w];
      }
      const int pos = before + __popc(bal & ((1u << lane) - 1u));
      if (tie && pos < need) {
        ent_key[slot + pos] = thr;
        ent_id[slot + pos] = v;
      }
      const int take = min(total, need);
      slot += take;
      need -= take;
      __syncthreads();
    }
    count = slot;
  }
  // rank = entries before this one (higher key, or the same key and a lower id); the first N go out in rank order
  if (static_cast<int>(threadIdx.x) < count) {
    const uint32_t k = ent_key[threadIdx.x];
    const int v = ent_id[threadIdx.x];
    int rank = 0;
    for (int q = 0; q < count; ++q) rank += (ent_key[q] > k || (ent_key[q] == k && ent_id[q] < v)) ? 1 : 0;
    if (rank < N) {
      out_top_ids[static_cast<size_t>(i) * kMaxLogprobs + rank] = v;
      out_top_lp[static_cast<size_t>(i) * top_lp_ld + rank] = lp_of_key(k);
    }
  }
}

}  // namespace

int logprobs_rows(const void* logits, int ld, int V, const int* rows, const int* top_n, int n, const int* tokens, float* lp,
                  int lp_ld, float* top_lp, int top_lp_ld, int* top_ids, cudaStream_t st, int* rank) {
  if (n <= 0) return 0;
  if (V < 1 || ld < V || ld % 8 || (reinterpret_cast<uintptr_t>(logits) & 15)) return -1;
  if (rank)
    launch_pdl(logprobs_kernel<true>, dim3(n), dim3(kThreads), kCntSmem, st, static_cast<const uint16_t*>(logits), ld, V, rows,
               top_n, tokens, lp, lp_ld, top_lp, top_lp_ld, top_ids, rank);
  else
    launch_pdl(logprobs_kernel<false>, dim3(n), dim3(kThreads), kCntSmem, st, static_cast<const uint16_t*>(logits), ld, V, rows,
               top_n, tokens, lp, lp_ld, top_lp, top_lp_ld, top_ids, rank);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

int sample_rows(const void* logits, int ld, const void* rows, int row_words, int S, int V, int* out, cudaStream_t st) {
  if (S <= 0) return 0;
  if (V < 1 || ld < V || ld % 8 || (reinterpret_cast<uintptr_t>(logits) & 15) || (row_words != 6 && row_words != 7)) return -1;
  static std::atomic<unsigned long long> smem_set{0};
  if (!ensure_dynamic_smem(sample_kernel, kPrivSmem, &smem_set)) return -2;
  launch_pdl(sample_kernel, dim3(S), dim3(kThreads), kPrivSmem, st, static_cast<const uint16_t*>(logits), ld,
             static_cast<const int32_t*>(rows), row_words, V, out);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

}  // namespace b200
