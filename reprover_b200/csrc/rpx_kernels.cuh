// rpx_kernels.cuh — launchers of the encoder's non-GEMM kernels (defined in rpx_attention.cu and
// rpx_elementwise.cu).  The top-k launchers are declared in rpx_topk_common.cuh.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace rpx {

// ---- rpx_attention.cu
// qkv [T, 3*heads*d_kv] bf16 packed tokens; out [T, heads*d_kv] bf16;
// bias_lut [heads][2*max_distance+1] fp32, entry (delta + max_distance), delta = key - query clamped.
int launch_t5_attention(const __nv_bfloat16* qkv, __nv_bfloat16* out, const int32_t* cu_seqlens,
                        const float* bias_lut, int n_tokens, int n_seqs, int max_len, int n_heads, int d_kv,
                        int max_distance, cudaStream_t stream);

// The kernel's three modes (rpx_attention.cu): the encoder's, decoder causal self-attention, cross-attention.
enum class AttnMode : int { kBidirectional = 0, kCausal = 1, kCross = 2 };
// One attention launch in any mode.  q: [q_rows, q_ld] bf16, head h's queries in columns [q_col + 64 h, +64);
// kv: [kv_rows, kv_ld] bf16, keys / values of head h at k_col + 64 h / v_col + 64 h; out [*, ld_out] bf16, head h in
// columns [64 h, 64 h + 64).  cu_q: the queries' sequences; cu_kv: the keys' (kCross only; the self modes use
// cu_q).  bias_lut: [heads][2 max_distance + 1] (unused in kCross).  max_len: longest query sequence.
struct AttnArgs {
  const __nv_bfloat16* q;
  int q_rows, q_ld, q_col;
  const __nv_bfloat16* kv;
  int kv_rows, kv_ld, k_col, v_col;
  __nv_bfloat16* out;
  int ld_out;
  const int32_t* cu_q;
  const int32_t* cu_kv;
  const float* bias_lut;
  int n_seqs, max_len, n_heads, d_kv, max_distance;
};
int launch_t5_attention_mode(AttnMode mode, const AttnArgs& args, cudaStream_t stream);

// ---- rpx_generate.cu
// Decode self-attention: query (row r, head h) of step t against keys p = 0..t of its hypothesis.  cache: one layer,
// [max_length][rows][ld = 3 inner] bf16 (q | k | v, head h at 64 h of each); cache row p * rows + lin[r][p] holds
// position p of row r's hypothesis (lin [rows][max_length] int32; null: the row's own slot r at every position).
// Score q.k (unscaled) + lut[h][max(p - t, -max_distance) + max_distance]; out [rows, inner] bf16.
// Rows of a state with state_done[4 (r / beams)] != 0 are not written (state_done: BeamStepArgs::state, or null).
struct DecodeAttnArgs {
  const __nv_bfloat16* cache;
  const int32_t* lin;
  const float* lut;
  __nv_bfloat16* out;
  const int32_t* state_done;  // [states][4], word 0 = done (BeamStepArgs::state), or null
  int t, rows, ld, inner, n_heads, max_length, max_distance, beams;
};
int launch_decode_attention(const DecodeAttnArgs& a, cudaStream_t stream);

// One search step over fp32 logits [rows, vocab], rows = states * beams (rpx_generate.cu documents the rules).
// tokens [max_length][rows]: the input token of every row at every step (step t + 1's are written here).
// state [states][4]: done, early-stop heuristic unsatisfied, finished-buffer parity, unused.
// Finished hypotheses (beams > 1): [2][rows] scores / lengths / flags, [2][rows][max_length] generated tokens.
// Greedy (beams == 1) keeps each row's generated length in fin_len[r].  trace_*: this step's log-probs (greedy:
// logits) [rows, vocab], parents (global row) and tokens [rows] of the next step's running rows, or null.
struct BeamStepArgs {
  const float* logits;
  int32_t* tokens;
  int32_t* lin;  // [2][rows][max_length], parity t & 1 is step t's
  float* run_score;
  float* fin_score;
  int32_t* fin_len;
  int32_t* fin_flag;
  int32_t* fin_seq;
  int32_t* state;
  int32_t* done_count;
  int32_t* last_step;  // max over states of (step at which the state's search ended) + 1: the steps HF runs
  float* trace_scores;
  int32_t* trace_parents;
  int32_t* trace_tokens;
  float penalty;  // (float)((t + 1) ** length_penalty), computed in double as Python does
  int t, rows, beams, vocab, max_length, eos;
};
// Dynamic shared memory of one beam step CTA (the beams * vocab candidate keys).
size_t beam_step_smem_bytes(int beams, int vocab);
// Allows the beam step kernel up to max_smem bytes of dynamic shared memory on the current device (once per decoder).
int configure_search_step(size_t max_smem);
int launch_search_step(const BeamStepArgs& a, int states, cudaStream_t stream);

struct GenerateInitArgs {
  int32_t* tokens;
  int32_t* lin;  // null for greedy
  float* run_score;
  float* fin_score;
  int32_t* fin_len;
  int32_t* fin_flag;
  int32_t* state;
  int32_t* done_count;
  int32_t* out_len;
  int32_t* last_step;
  int rows, states, beams, max_length, start_id;
};
int launch_generate_init(const GenerateInitArgs& a, cudaStream_t stream);

// sequences [states * n_ret, max_length] int64: start id, the generated tokens, fill_id after them; scores
// [states * n_ret] (beams > 1); out_len = 1 + the longest returned hypothesis.
struct GenerateFinishArgs {
  const int32_t* tokens;
  const float* fin_score;
  const int32_t* fin_len;
  const int32_t* fin_seq;
  const int32_t* state;
  int64_t* sequences;
  float* scores;
  int32_t* out_len;
  int rows, beams, n_ret, max_length, start_id, fill_id;
};
int launch_generate_finish(const GenerateFinishArgs& a, int states, cudaStream_t stream);

// ---- rpx_elementwise.cu
// ByT5 tokenisation of packed byte strings into packed token ids (byte + 3, EOS = 1 last,
// truncated to max_seq_len including EOS).  cu_bytes / cu_tokens are [n_seqs + 1] device arrays.
int launch_tokenize_bytes(const uint8_t* bytes, const int64_t* cu_bytes, const int32_t* cu_tokens,
                          int32_t* ids, int n_seqs, int n_tokens, cudaStream_t stream);
// Padded [B, L] int64 ids -> packed ids using cu_tokens (first len_b ids of each row).
int launch_pack_ids(const int64_t* ids, const int32_t* cu_tokens, int32_t* packed, int batch, int seq_len,
                    int n_tokens, int vocab, int32_t* bad_flag, cudaStream_t stream);
// lens[b] = sum(mask[b, :]); flag |= 1 if the mask is not a prefix of ones or a row is empty.
int launch_mask_lengths(const int64_t* mask, int32_t* lens, int32_t* bad_flag, int batch, int seq_len,
                        cudaStream_t stream);
// h32[t] = table[ids[t]] (fp32), h16 = bf16(h32), ss[0][t] = sum h32^2, ss[1..n_parts)[t] = 0.
int launch_embed(const int32_t* ids, const float* table, float* h32, __nv_bfloat16* h16, float* ss,
                 int ss_stride, int n_parts, int n_tokens, int d_model, cudaStream_t stream);
// Final RMSNorm + masked mean-pool + L2 normalise (retrieval/model.py:108-114):
//   out[s] = normalize( (1/len_s) * sum_t  w .* h32[t] * rs[t] )
int launch_pool_normalize(const float* h32, const float* ss, int ss_stride, int n_parts, const float* ln_w,
                          const int32_t* cu_tokens, void* out, int out_dtype, int n_seqs, int d_model,
                          float eps, cudaStream_t stream, float* group_scratch = nullptr, int max_len = 0);
// Final RMSNorm of every token (the encoder's `last_hidden_state`) into a padded [batch, seq_len, d_model] output:
//   out[b, p] = w .* h32[cu[b] + p] * rs[cu[b] + p]  for p < len_b,  0  for p >= len_b.
// `lane_ss`: sum the ss parts in pool_partial_kernel's order (latency path) instead of pool_normalize_kernel's.
// `out` must be 16-byte aligned.
int launch_hidden_store(const float* h32, const float* ss, int ss_stride, int n_parts, bool lane_ss, const float* ln_w,
                        const int32_t* cu_tokens, void* out, int out_dtype, int batch, int seq_len, int d_model,
                        float eps, cudaStream_t stream);

// Weight packing (rpx_encoder_create): dst[n, k] = bf16(src[n, k] * scale[k]) (scale may be null),
// rows written at dst_row0 + (n / blk) * blk_stride + (n % blk)  (FFN interleave when blk_stride != blk).
int launch_pack_weight(const float* src, const float* scale, __nv_bfloat16* dst, int n_rows, int n_cols,
                       int dst_row0, int blk, int blk_stride, cudaStream_t stream);

}  // namespace rpx
