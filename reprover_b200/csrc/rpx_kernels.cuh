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
