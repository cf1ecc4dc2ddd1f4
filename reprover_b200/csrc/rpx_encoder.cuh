// rpx_encoder.cuh — the encoder's handle and the parts of its forward pass (rpx_encoder.cu) that the generator's
// decoder (rpx_decoder.cu) runs as well: the workspace, the GEMM launchers, the bias table, forward().
#pragma once
#include <vector>

#include "rpx.h"
#include "rpx_common.cuh"
#include "rpx_gemm.cuh"

namespace rpx {

struct LayerW {
  const __nv_bfloat16* qkv;  // [3*inner, D]   (ln0 folded)
  const __nv_bfloat16* o;    // [D, inner]
  const __nv_bfloat16* wi;   // [2*d_ff, D]    (ln1 folded; wi_0 / wi_1 interleaved in 128-row blocks)
  const __nv_bfloat16* wo;   // [D, d_ff]
};

struct ProfRec {
  int cls;
  cudaEvent_t a, b;
};

}  // namespace rpx

struct rpx_encoder {
  rpx_t5_config cfg;
  int inner = 0;
  int n_parts = 0;      // RMSNorm partial sums per row on the throughput path: one per 128-wide n-tile
  int n_parts_lat = 0;  // ... on the latency path: one per 32-column chunk
  int latency_tokens = 0;  // calls with at most this many packed tokens take the latency path (0: never)
  size_t layer_bytes = 0;  // packed weights of one layer (qkv | o | wi | wo, contiguous from LayerW::qkv)
  const float* emb = nullptr;
  const float* final_ln = nullptr;
  const float* bias_lut = nullptr;
  std::vector<rpx::LayerW> layers;
  float* debug_hidden = nullptr;
  bool profiling = false;
  std::vector<rpx::ProfRec> prof_pending;
  std::vector<cudaEvent_t> event_pool;
  float prof_ms[RPX_N_KERNEL_CLASSES] = {0};
  int64_t prof_launches[RPX_N_KERNEL_CLASSES] = {0};
  std::vector<int32_t> h_cu_tokens;
  std::vector<int32_t> h_lens;
};

namespace rpx {

// Relative-attention configs the bucket function and the attention kernel's shared bias table support.
int check_rel_attention(int rel_buckets, int rel_max_distance, bool bidirectional);
int validate_cfg(const rpx_t5_config* c);

// Relative-position bias LUT: lut[h][delta + R] = rel_bias[bucket(delta)][h] for delta = key - query in [-R, R],
// with HF's bidirectional (encoder) or unidirectional (decoder) buckets.  The bucket table is computed on the host
// and staged through `d_buckets` (2R + 1 int32).  Synchronises `st`: the host table is pageable and dies on return.
// The caller has checked the config (check_rel_attention).
int build_bias_lut(const float* d_rel_bias, int n_heads, int rel_buckets, int R, bool bidirectional, int32_t* d_buckets,
                   float* d_lut, cudaStream_t st);

// Device buffers of one forward pass over T packed tokens in S sequences.
struct Workspace {
  int32_t* cu_tokens;
  int64_t* cu_bytes;
  int32_t* ids;
  int32_t* lens;
  int32_t* flag;
  float* h32;
  __nv_bfloat16* h16;
  __nv_bfloat16* qkv;
  __nv_bfloat16* attn;
  __nv_bfloat16* ffn;
  float* ssA;
  float* ssB;
  size_t total;
};
// The S-sized members come first, at offsets that depend on S alone; base == nullptr only sizes.
Workspace carve(const rpx_encoder* e, uint8_t* base, int64_t T, int64_t S);

// Calls of at most this many tokens run their kernel chain under programmatic dependent launch: it hides
// the prologue of each kernel behind the tail of its predecessor, which matters while the tails are a
// noticeable share of a kernel's time.
constexpr int kPdlMaxTokens = 16384;

struct PdlScope {
  explicit PdlScope(bool on) { set_pdl_scope(on); }
  ~PdlScope() { set_pdl_scope(false); }
};

// RMSNorm partial sums per row: one per 128 columns on the throughput path (EpiWsResidual: two per 256-wide
// tile), one per 32-column chunk on the latency path.
int ss_parts(int d_model, bool latency);

// The encoder's four GEMMs, each on the tiles the forward pass uses for T tokens on the throughput or the
// latency path (rpx_encoder.cu documents each).  A is [T, K], B is [N, K] (packed weights).
int qkv_gemm(bool latency, int T, const void* A, const void* B, int N, int K, const RowScale& rs, __nv_bfloat16* out,
             const void* prefetch, size_t prefetch_bytes, cudaStream_t st);
int oproj_gemm(bool latency, int T, const void* A, const void* B, int N, int K, float* h32, __nv_bfloat16* h16,
               float* ss_out, cudaStream_t st);
int ffn_down_gemm(bool latency, int T, const void* A, const void* B, int N, int K, float* h32, __nv_bfloat16* h16,
                  float* ss_out, cudaStream_t st);
int ffn_up_gemm(bool latency, int T, const void* A, const void* B, int N, int K, const RowScale& rs,
                __nv_bfloat16* out, cudaStream_t st);
// The generator's output head: out [T, N] fp32 = A B^T * rs[m], always on the throughput core.
int head_gemm(int T, const void* A, const void* B, int N, int K, const RowScale& rs, float* out, cudaStream_t st);

// What forward() writes after the last block.
//   kPooled    final RMSNorm + masked mean + L2 normalise: [S, D]
//   kHidden    final RMSNorm of every token (`last_hidden_state`): [S, seq_len, D], rows past a sequence's length zeroed
//   kResidual  nothing: the last block's residual stream stays in ws.h32 / ws.h16 and its RMSNorm partial sums
//              ([n_parts][T]) in ws.ssA, for a caller that folds the final RMSNorm into its own GEMM.  Always
//              on the throughput tiles.
enum class OutKind { kPooled, kHidden, kResidual };

// The forward pass proper.  ws.ids / ws.cu_tokens are already populated on `st`.  `seq_len` is the padded row
// length of a kHidden output (unused otherwise).
int forward(rpx_encoder* e, const Workspace& ws, int T, int S, int max_len, OutKind kind, int seq_len, void* d_out,
            int out_dtype, cudaStream_t st);

}  // namespace rpx
