// Host launchers for the non-GEMM kernels (elementwise.cu, attention.cu).  All pointers are device
// pointers, all tensors bf16 unless stated; return 0 on success, negative on bad shape / launch error.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <vector>

namespace b200 {

int embed_gather(const void* table, const int* ids, void* out, int T, int H, int vocab, cudaStream_t st);
// out[s] = rmsnorm(x[r] (+ residual[r])) * w,  r = row_index ? row_index[s] : s.
// residual (optional) is updated in place with bf16(x + residual) unless row_index is given.
int rmsnorm(const void* x, void* residual, const void* w, void* out, const int* row_index, int rows, int H,
            float eps, cudaStream_t st);
// Last-token pooling (pooling.cu): out[s] (fp32 [rows, H]) = the final RMSNorm of row row_index[s] of x (+ residual, as
// rmsnorm with a row_index), bit-identical in bf16 to rmsnorm over the same rows, then L2-normalised in fp32 when
// flags[s] != 0.  H % 256 == 0 and H <= 8192; row_index and flags are device int arrays [rows].
int pool_rows(const void* x, const void* residual, const void* w, const int* row_index, const int* flags, int rows, int H,
              float eps, float* out, cudaStream_t st);
// A score head's tail (pooling.cu): out[s, 0..L) (fp32 [rows, L]) = the logits sw [L, H] . y of the same normed row y
// as pool_rows, in fp32 in a fixed order, then, when flags[s] != 0, the activation act (kScore*: sigmoid, softmax over
// the L logits, or none).  1 <= L <= kMaxScoreLabels: one warp applies the activation, lane l holding logit l.
constexpr int kMaxScoreLabels = 32;
enum { kScoreSigmoid = 1, kScoreSoftmax = 2, kScoreNone = 3 };
int score_rows(const void* x, const void* residual, const void* w, const void* sw, const int* row_index, const int* flags,
               int rows, int H, int L, int act, float eps, float* out, cudaStream_t st);
// head_dim D = 64 or 128: qkv rows [(Hq + 2 Hkv) * D], cos_sin rows [D], kv_layer [block][2][Hkv][16][D]
int rope_kv_write(void* qkv, const int* positions, const int* slots, const void* cos_sin, void* kv_layer,
                  int T, int Hq, int Hkv, int max_pos, cudaStream_t st, int head_dim = 128);
// interleaved: gate/up columns alternate in 64-column blocks (engine layout) instead of [gate | up]
int silu_mul(const void* gate_up, void* out, int T, int I, cudaStream_t st, int interleaved = 0);
// gate_up weight rows: logical [gate | up] <-> physical (64 gate rows, their 64 up rows, ...); dst != src
int permute_gate_up(void* dst, const void* src, int I, int H, int to_physical, cudaStream_t st);
int argmax_rows(const void* logits, int* out, int S, int V, int ld, cudaStream_t st);
int init_uniform(void* p, size_t n, uint32_t seed, float scale, float offset, cudaStream_t st);
// Parallel sampling's fork (kv_fork.cu): for every pair i and every layer l, copy the block_bytes of page src[i] to page
// dst[i] at kv + l * layer_stride_bytes (src / dst device int arrays; sizes and kv 16-byte aligned).  Bit-exact; nothing
// outside the dst pages is written.
int kv_copy_blocks(void* kv, int num_layers, int64_t layer_stride_bytes, int64_t block_bytes, const int* src, const int* dst,
                   int n_pairs, cudaStream_t st);

// Per-row sampling parameters (sampling.cu; b200_sample_row at the ABI): temperature < 1e-5 is greedy, top_k <= 0 or >= V,
// top_p <= 0 or >= 1 and min_p <= 0 are off; the noise of the row is Philox4x32-10 keyed by the seed and counted by n, the
// index of the token being generated.
struct SampleRow {
  float temperature;
  int top_k;
  float top_p;
  uint32_t seed_lo, seed_hi;
  int n;
  float min_p;
};
// out[s] = the token sampled from bf16 logits row s ([S, ld], ld % 8 == 0) under row s of `rows` (device memory): rows of
// row_words = 7 words (a SampleRow) or 6 (the same without min_p, which is then off)
int sample_rows(const void* logits, int ld, const void* rows, int row_words, int S, int V, int* out, cudaStream_t st);

// Sparse logits edits (penalties.cu): logit_bias, min_tokens and the repetition / frequency / presence penalties of vLLM V1,
// applied in fp32 to the entries a request's record list names and written back rounded to bf16.  A list holds one record
// per distinct token id, sorted by id: its count in the output, whether it is in the prompt, whether it is a stop id (EOS
// included unless ignore_eos) banned until min_tokens tokens exist, and its bias.
enum { kPenPrompt = 1, kPenStop = 2, kPenBias = 4 };
struct PenaltyRec {
  int id;
  int count;       // occurrences in the generated tokens
  float bias;      // with kPenBias
  uint32_t flags;  // kPen*
};
// One edited row of a step: logits row `row`, record list `slot`; repetition 1 = off.  history: the list counts the
// generated tokens (some penalty is on), so penalize_update adds each sampled token to it.
struct PenaltyRow {
  int row, slot;
  float presence, frequency, repetition;
  int n_generated, min_tokens, history;
};
// Record list of one request from host token lists (the prompt and output only when `history`; stops only when they apply)
void penalty_records(const int32_t* prompt, int n_prompt, const int32_t* output, int n_output, bool history,
                     const int32_t* bias_ids, const float* bias_values, int n_bias, const int32_t* stops, int n_stops,
                     std::vector<PenaltyRec>* out);
// Record lists live in recs[slot * cap ...], their lengths in lens[slot].  penalize_rows edits the n rows in place and
// saves the raw bf16 entries it overwrites in save [n][cap]; penalize_restore writes them back; penalize_update adds
// sampled[row] of every history row to its list (count + 1, or a new record in id order).  Device pointers throughout.
int penalize_rows(void* logits, int ld, const PenaltyRow* rows, int n, const PenaltyRec* recs, const int* lens, int cap,
                  uint16_t* save, cudaStream_t st);
int penalize_restore(void* logits, int ld, const PenaltyRow* rows, int n, const PenaltyRec* recs, const int* lens, int cap,
                     const uint16_t* save, cudaStream_t st);
int penalize_update(const PenaltyRow* rows, int n, const int* sampled, PenaltyRec* recs, int* lens, int cap, cudaStream_t st);

// Log-probabilities (sampling.cu; vLLM's raw_logprobs) of n rows of bf16 logits ([., ld], ld % 8 == 0): row i is
// r = rows ? rows[i] : i, its N = clamp(top_n[i], 0, min(V, kMaxLogprobs)).  lp[i * lp_ld] gets the log-probability of
// tokens[r]; top_lp[i * top_lp_ld + j] and top_ids[i * kMaxLogprobs + j], j < N, the N most likely tokens (by logit,
// lowest id on ties).  Entries past N are not written.  rank (optional): rank[i] = the number of tokens whose logit is >=
// that of tokens[r] (vLLM's prompt-logprob rank).  Every pointer is device memory.
constexpr int kMaxLogprobs = 20;
int logprobs_rows(const void* logits, int ld, int V, const int* rows, const int* top_n, int n, const int* tokens, float* lp,
                  int lp_ld, float* top_lp, int top_lp_ld, int* top_ids, cudaStream_t st, int* rank = nullptr);

// One unit of attention work: q_count query tokens of one sequence starting at row q_tok0 of the
// step's token batch; the first of them sits at absolute position q_pos0 in the sequence.
struct AttnWork {
  int q_tok0;
  int q_count;  // decode: 1, or up to kDecodeRows / G consecutive positions (a speculative verify); prefill: <= kPrefillQueryBlock
  int q_pos0;
  int seq;      // row of block_tables
};

// rows of decode attention's mma tile: a work item's G query heads times its q_count positions (the last token and its
// speculative drafts) must fit in it
constexpr int kDecodeRows = 16;

// the group sizes G = Hq / Hkv the attention kernels serve: Hkv divides Hq and 1 <= G <= 16
inline bool attn_group_ok(int Hq, int Hkv) { return Hkv >= 1 && Hq % Hkv == 0 && Hq / Hkv >= 1 && Hq / Hkv <= kDecodeRows; }

// the head sizes D the attention kernels, the qkv epilogue and the KV pool serve
inline bool attn_head_dim_ok(int D) { return D == 64 || D == 128; }

// Paged causal attention, head_dim D (attn_head_dim_ok), G = Hq / Hkv query heads per KV head (attn_group_ok), page = 16 tokens.
//   q: rows of the fused qkv buffer (leading dim ldq), out: [T, Hq*D] (leading dim ldo)
//   kv_layer: [block][2][Hkv][16][D];  block_tables: [num_seqs, max_blocks] int32
//   every work item has 1 <= q_count and G * q_count <= kDecodeRows (position j causally masked at q_pos0 + j); the CTA's
//   4 warps split the KV range.  Chunked prefill is paged_attention_prefill_tc.
int paged_attention(const void* q, int ldq, void* out, int ldo, const void* kv_layer, const int* block_tables,
                    int max_blocks, const AttnWork* work, int num_work, int Hq, int Hkv, float scale,
                    cudaStream_t st, float* split_ws = nullptr, int split = 1, int head_dim = 128);
// split-KV decode (few sequences): `split` CTAs per (work item, KV head) each stream a slice of the context and leave an
// unnormalised partial per query head in split_ws (attn_split_ws_bytes, max_q = the largest q_count of the launch), merged
// by a second tiny kernel.  attn_decode_split picks `split`.
size_t attn_split_ws_bytes(int num_work, int Hq, int parts, int max_q = 1, int head_dim = 128);
int attn_decode_split(int num_work, int Hkv, int max_ctx, int sms);

// Chunked-prefill attention on wgmma (attention_wgmma.cu): work items of up to kPrefillQueryBlock query tokens, one CTA per
// (work item, query head); q rows are read from the fused qkv buffer [qkv_rows, ldq].
constexpr int kPrefillQueryBlock = 64;
int paged_attention_prefill_tc(const void* qkv, int qkv_rows, int ldq, void* out, int ldo, const void* kv_layer, const int* block_tables,
                               int max_blocks, const AttnWork* work, int num_work, int Hq, int Hkv, float scale, cudaStream_t st,
                               int head_dim = 128);

}  // namespace b200
