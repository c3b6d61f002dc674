// Host launchers for the non-GEMM kernels (elementwise.cu, attention.cu).  All pointers are device
// pointers, all tensors bf16 unless stated; return 0 on success, negative on bad shape / launch error.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "partials.cuh"

namespace b200 {

// ssq (optional): [T, ssq_slabs] fp32, the row's sum of squares in slab 0 and zeros elsewhere (RMSNorm prologue of the fused GEMM)
int embed_gather(const void* table, const int* ids, void* out, int T, int H, int vocab, cudaStream_t st, float* ssq = nullptr,
                 int ssq_slabs = 0);
// out[s] = rmsnorm(x[r] (+ residual[r])) * w,  r = row_index ? row_index[s] : s.
// residual (optional) is updated in place with bf16(x + residual) unless row_index is given.
// Every consumer of a GEMM output takes an optional PartialView: when pv.ws != nullptr the input is the fp32
// stream-K partials of the preceding deferred GEMM (summed + rounded to bf16 on load) instead of the bf16 tensor.
int rmsnorm(const void* x, void* residual, const void* w, void* out, const int* row_index, int rows, int H,
            float eps, cudaStream_t st, PartialView pv = no_partials());
int rope_kv_write(void* qkv, const int* positions, const int* slots, const void* cos_sin, void* kv_layer,
                  int T, int Hq, int Hkv, int max_pos, cudaStream_t st, PartialView pv = no_partials());
// interleaved: gate/up columns alternate in 64-column blocks (engine layout) instead of [gate | up]
int silu_mul(const void* gate_up, void* out, int T, int I, cudaStream_t st, PartialView pv = no_partials(), int interleaved = 0);
// gate_up weight rows: logical [gate | up] <-> physical (64 gate rows, their 64 up rows, ...); dst != src
int permute_gate_up(void* dst, const void* src, int I, int H, int to_physical, cudaStream_t st);
int argmax_rows(const void* logits, int* out, int S, int V, int ld, cudaStream_t st, PartialView pv = no_partials());
int init_uniform(void* p, size_t n, uint32_t seed, float scale, float offset, cudaStream_t st);

// One unit of attention work: q_count query tokens of one sequence starting at row q_tok0 of the
// step's token batch; the first of them sits at absolute position q_pos0 in the sequence.
struct AttnWork {
  int q_tok0;
  int q_count;  // 1 for decode, <= 16 for a prefill tile
  int q_pos0;
  int seq;      // row of block_tables
};

// Paged causal attention, head_dim 128, GQA group 4 (Hq = 4 * Hkv), page = 16 tokens.
//   q: rows of the fused qkv buffer (leading dim ldq), out: [T, Hq*128] (leading dim ldo)
//   kv_layer: [block][2][Hkv][16][128];  block_tables: [num_seqs, max_blocks] int32
//   decode != 0: every work item has q_count == 1 and the CTA's 4 warps split the KV range.
int paged_attention(const void* q, int ldq, void* out, int ldo, const void* kv_layer, const int* block_tables,
                    int max_blocks, const AttnWork* work, int num_work, int Hq, int Hkv, float scale,
                    int decode, cudaStream_t st, float* split_ws = nullptr, int split = 1);
// split-KV decode (few sequences): `split` CTAs per (work item, KV head) each stream a slice of the context and leave an
// unnormalised partial in split_ws (attn_split_ws_bytes), merged by a second tiny kernel.  attn_decode_split picks `split`.
size_t attn_split_ws_bytes(int num_work, int Hkv, int parts);
int attn_decode_split(int num_work, int Hkv, int max_ctx, int sms);

// Chunked-prefill attention on wgmma (attention_wgmma.cu): work items of up to kPrefillQueryBlock query tokens, one CTA per
// (work item, query head); q rows are read from the fused qkv buffer [qkv_rows, ldq].
constexpr int kPrefillQueryBlock = 64;
int paged_attention_prefill_tc(const void* qkv, int qkv_rows, int ldq, void* out, int ldo, const void* kv_layer, const int* block_tables,
                               int max_blocks, const AttnWork* work, int num_work, int Hq, int Hkv, float scale, cudaStream_t st);

}  // namespace b200
