// rpx_encoder.cu — the ByT5 / T5 encoder forward (+ pool + normalise) on packed tokens.
//
// Replaces `PremiseRetriever._encode` (reference retrieval/model.py:92-114) and the HF
// `T5Stack` it calls (modeling_t5.py:637-792): per layer
//     h += O( attn( RMSNorm(h) ) )                      modeling_t5.py:366-375
//     h += wo( gelu_new(wi_0 n) * (wi_1 n) ), n = RMSNorm(h)   :146-150, :115-131
// then final RMSNorm, masked mean over tokens, L2 normalise.
//
// Data layout in HBM (T = packed tokens of the call, D = d_model):
//     h32  [T, D] fp32   residual stream (master copy)
//     h16  [T, D] bf16   same values, GEMM A operand
//     qkv  [T, 3*H*64] bf16,  attn [T, H*64] bf16,  ffn [T, d_ff] bf16
//     ssA / ssB [n_parts][T] fp32  per-row partial sums of h32^2, one per n-tile of the GEMM that
//                             produced h32 (12 for d_model = 1472) -> RMSNorm row scale
// RMSNorm never runs as its own kernel: its weight vector is folded into the next
// GEMM's B operand when the weights are packed, and the row scale rsqrt(mean(h^2)+eps)
// is applied to the fp32 accumulator in that GEMM's epilogue (rpx_gemm.cuh RowScale).
#include <math.h>

#include <new>
#include <vector>

#include "rpx_gemm_launch.cuh"
#include "rpx_kernels.cuh"

namespace rpx {

namespace {

// Throughput-path tiles of QKV: 128 x 128.  The accumulator tile (64 KB) and a 4-deep operand ring fit the 227 KB
// of shared memory an H100 block may use.  The gated FFN up-projection, O-proj and FFN-down run on
// gemm_ws_kernel's 128 x 256 tiles instead (rpx_gemm_ws.cuh); QKV measured 6 % slower there, its epilogue no
// longer overlapping the next tile's MMAs.
constexpr int kBlockN = 128;

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

}  // namespace

}  // namespace rpx

// T5 relative-position bucket, bidirectional (HF modeling_t5.py:189-234), float32 math
// like the reference implementation.  Host function, exported for the CPU parity test.
// Precondition (check_rel_attention): max_distance > num_buckets / 4, else the log-spaced branch divides by 0.
extern "C" int32_t rpx_t5_relative_bucket(int32_t relative_position, int32_t num_buckets, int32_t max_distance) {
  int nb = num_buckets / 2;
  int ret = relative_position > 0 ? nb : 0;
  int n = relative_position < 0 ? -relative_position : relative_position;
  const int max_exact = nb / 2;
  if (n < max_exact) return ret + n;
  float v = logf((float)n / (float)max_exact) / (float)log((double)max_distance / (double)max_exact) *
            (float)(nb - max_exact);
  int large = max_exact + (int)v;
  if (large > nb - 1) large = nb - 1;
  return ret + large;
}

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

namespace {

struct PackedLayout {
  size_t emb, final_ln, bias_lut, bucket_tmp, layer0, layer_stride, qkv, o, wi, wo, total;
};

PackedLayout packed_layout(const rpx_t5_config& c) {
  PackedLayout L{};
  const size_t D = c.d_model, inner = (size_t)c.num_heads * c.d_kv, F = c.d_ff;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off = align_up(off + bytes, 256);
    return o;
  };
  L.emb = take((size_t)c.vocab_size * D * 4);
  L.final_ln = take(D * 4);
  L.bias_lut = take((size_t)c.num_heads * (2 * c.rel_max_distance + 1) * 4);
  L.bucket_tmp = take((size_t)(2 * c.rel_max_distance + 1) * 4);
  L.layer0 = off;
  L.qkv = 0;
  size_t lo = 0;
  auto ltake = [&](size_t bytes) {
    size_t o = lo;
    lo = align_up(lo + bytes, 256);
    return o;
  };
  L.qkv = ltake(3 * inner * D * 2);
  L.o = ltake(D * inner * 2);
  L.wi = ltake(2 * F * D * 2);
  L.wo = ltake(D * F * 2);
  L.layer_stride = lo;
  L.total = L.layer0 + lo * (size_t)c.num_layers;
  return L;
}

// The bucket formula takes log(max_distance / max_exact) with max_exact = buckets / 4, so max_distance must
// exceed it; 2048 bounds the bias table the attention kernel keeps in shared memory.
int check_rel_attention(int rel_buckets, int rel_max_distance) {
  RPX_REQUIRE(rel_buckets >= 4 && rel_buckets % 4 == 0 && rel_max_distance > rel_buckets / 4 && rel_max_distance <= 2048,
              RPX_ERR_UNSUPPORTED, "unsupported relative attention config (%d buckets, max distance %d)", rel_buckets,
              rel_max_distance);
  return RPX_OK;
}

int validate_cfg(const rpx_t5_config* c) {
  RPX_REQUIRE(c != nullptr, RPX_ERR_INVALID, "config is null");
  RPX_REQUIRE(c->d_kv == 64, RPX_ERR_UNSUPPORTED, "d_kv=%d: only 64 is implemented", c->d_kv);
  RPX_REQUIRE(c->d_model % 64 == 0 && c->d_model > 0, RPX_ERR_UNSUPPORTED, "d_model=%d must be a multiple of 64", c->d_model);
  RPX_REQUIRE(c->d_ff % 128 == 0 && c->d_ff > 0, RPX_ERR_UNSUPPORTED, "d_ff=%d must be a multiple of 128", c->d_ff);
  RPX_REQUIRE(c->num_heads > 0 && c->num_layers > 0 && c->vocab_size > 0, RPX_ERR_INVALID, "bad config");
  return check_rel_attention(c->rel_buckets, c->rel_max_distance);
}

__global__ void bias_lut_kernel(const float* __restrict__ rel_bias, const int32_t* __restrict__ buckets,
                                float* __restrict__ lut, int n_heads, int width) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_heads * width) return;
  const int h = i / width, j = i % width;
  lut[i] = rel_bias[buckets[j] * n_heads + h];
}

// Relative-position bias LUT: lut[h][delta + R] = rel_bias[bucket(delta)][h] for delta = key - query in [-R, R].
// The bucket table is computed on the host and staged through `d_buckets` (2R + 1 int32).  Synchronises `st`:
// the host table is pageable and dies on return.  The caller has checked the config (check_rel_attention).
int build_bias_lut(const float* d_rel_bias, int n_heads, int rel_buckets, int R, int32_t* d_buckets, float* d_lut,
                   cudaStream_t st) {
  const int width = 2 * R + 1;
  std::vector<int32_t> buckets(width);
  for (int j = 0; j < width; ++j) buckets[j] = rpx_t5_relative_bucket(j - R, rel_buckets, R);
  RPX_CUDA_OK(cudaMemcpyAsync(d_buckets, buckets.data(), (size_t)width * 4, cudaMemcpyHostToDevice, st));
  bias_lut_kernel<<<ceil_div(n_heads * width, 256), 256, 0, st>>>(d_rel_bias, d_buckets, d_lut, n_heads, width);
  RPX_CUDA_OK(cudaGetLastError());
  RPX_CUDA_OK(cudaStreamSynchronize(st));
  return RPX_OK;
}

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

Workspace carve(const rpx_encoder* e, uint8_t* base, int64_t T, int64_t S) {
  Workspace w{};
  const size_t D = e->cfg.d_model, inner = e->inner, F = e->cfg.d_ff;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    uint8_t* p = base ? base + off : nullptr;
    off = align_up(off + bytes, 256);
    return p;
  };
  w.cu_tokens = (int32_t*)take((S + 1) * 4);
  w.cu_bytes = (int64_t*)take((S + 1) * 8);
  w.lens = (int32_t*)take((S + 1) * 4);
  w.flag = (int32_t*)take(256);
  w.ids = (int32_t*)take(T * 4);
  w.h32 = (float*)take(T * D * 4);
  w.h16 = (__nv_bfloat16*)take(T * D * 2);
  w.qkv = (__nv_bfloat16*)take(T * 3 * inner * 2);
  w.attn = (__nv_bfloat16*)take(T * inner * 2);
  w.ffn = (__nv_bfloat16*)take(T * F * 2);
  const size_t parts = e->n_parts > e->n_parts_lat ? e->n_parts : e->n_parts_lat;
  w.ssA = (float*)take(parts * T * 4);
  w.ssB = (float*)take(parts * T * 4);
  w.total = off;
  return w;
}

struct Prof {
  rpx_encoder* e;
  cudaStream_t st;
  int cls;
  cudaEvent_t a = nullptr, b = nullptr;
  Prof(rpx_encoder* e_, cudaStream_t st_, int cls_) : e(e_), st(st_), cls(cls_) {
    if (!e->profiling) return;
    a = get();
    b = get();
    cudaEventRecord(a, st);
  }
  ~Prof() {
    if (!e->profiling) return;
    cudaEventRecord(b, st);
    e->prof_pending.push_back({cls, a, b});
  }
  cudaEvent_t get() {
    if (!e->event_pool.empty()) {
      cudaEvent_t ev = e->event_pool.back();
      e->event_pool.pop_back();
      return ev;
    }
    cudaEvent_t ev;
    cudaEventCreate(&ev);
    return ev;
  }
};

// ---------------------------------------------------------------------------------------------
// Latency path: one proof state per call (`retrieve`, retrieval/model.py:348-357, encodes ONE context).
// With T of a few hundred tokens the 128-row tiles of the throughput path leave most of the GPU idle
// (QKV: 9 tiles, O / FFN-down: 12 tiles for a 128-token state) and every GEMM is bound by the latency of
// streaming its operands through a handful of SMs.  Here the same contraction core runs narrow tiles:
//   up to 384 tokens   QKV, O-proj, FFN-down on 64-ROW tiles (one wgmma row block) x 64 columns with a 12-deep
//                      ring of 16 KB stages: 6 row tiles x 23 column tiles = 138 CTAs at 384 tokens for
//                      d_model = 1472; a narrow GEMM's time is its k-blocks times the round trip of the operand
//                      ring divided by the ring depth, and half-empty 128-row tiles would cost their full intake
//   beyond             128 x 64 tiles, 6-deep ring (what fits beside the 34 KB accumulator tile)
//   FFN-up             128 x 128 tiles = 64 gated hidden units (128 x 64 = 32 units up to 128 tokens), B tile in
//                      two boxes (gate rows, linear rows)
// K is never split, so every output element is accumulated over k in the same order whatever the tile, and
// the residual epilogues write their RMSNorm partial sums per 32-column chunk (n_parts_lat of them) whatever
// the tile: a state's embedding does not depend on what it was batched with.
constexpr int kLatBlockN = 64;
constexpr int kLatStages = 6;
constexpr int kLatSmallM = 64;
constexpr int kLatSmallStages = 12;
constexpr int kLatSmallMMaxTokens = 384;
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
int ss_parts(int d_model, bool latency) { return ceil_div(d_model, latency ? 32 : 128); }

// The encoder's four GEMMs, each on the tiles the forward pass uses for T tokens on the throughput or the
// latency path.  forward(), forward_latency_layer() and rpx_debug_encoder_gemm all launch through these, so the
// epilogue tests run exactly the launches an encode call runs.  A is [T, K], B is [N, K] (packed weights).

// out [T, N] = bf16(A B^T * rs[m]).  On the latency path the CTAs the GEMM leaves idle fetch `prefetch` into L2.
int qkv_gemm(bool latency, int T, const void* A, const void* B, int N, int K, const RowScale& rs, __nv_bfloat16* out,
             const void* prefetch, size_t prefetch_bytes, cudaStream_t st) {
  EpiStoreBF16::Params ep{out, N, rs};
  if (!latency) return launch_gemm<kBlockN, EpiStoreBF16>(A, K, B, K, T, N, K, ep, st);
  if (T <= kLatSmallMMaxTokens)
    return launch_gemm<kLatBlockN, EpiStoreBF16, false, kLatSmallStages, false, kLatSmallM>(A, K, B, K, T, N, K, ep, st, 0,
                                                                                             prefetch, prefetch_bytes);
  return launch_gemm<kLatBlockN, EpiStoreBF16, false, kLatStages>(A, K, B, K, T, N, K, ep, st, 0, prefetch, prefetch_bytes);
}

// h32 [T, N] += A B^T, h16 = bf16(h32), ss_out = partial sums of h32^2 ([ss_parts(N)][T]).
// The throughput path runs gemm_ws_kernel with the residual block streamed into shared memory.  How its 227 KB
// are split is chosen per site (RES_BUFS chunk buffers of 8 KB per consumer, STAGES operand stages of 48 KB), as
// measured fastest at 2^18 tokens on an H100 80GB HBM3 at a 700 W power limit (tools/encoder_gemm_bench.py):
//   O-proj   (K = 384, 6 k-blocks): 4 stages and 2 chunk buffers.  It is memory-bound, and its A operand is a
//            third of its HBM reads: the deep ring loads 4 of the next tile's 6 k-blocks while the epilogue
//            runs.  3 stages and 5 buffers took 3 % longer, 2 stages and 7 buffers 4 %.
//   FFN-down (K = 3584, 56 k-blocks): 3 stages and 5 chunk buffers.  With 2 buffers per consumer the epilogue
//            waited on 3 residual round trips per tile and took 5 % longer.
// CLUSTER is chosen the same way, on an H100 80GB HBM3 at a 400 W power limit (alternated runs of both forms):
//   O-proj   unclustered: 1.81-1.92 ms against 1.90-1.96 ms as pairs.  Being HBM-bound, it gains nothing from the
//            lower L2 traffic and pays for the coupling of the pair.  Its split as pairs (3 stages, 5 buffers)
//            took 1.85-1.96 ms.
//   FFN-down pairs: 6.31-6.44 ms against 6.38-6.59 ms unclustered.  As pairs, 4 stages and 2 buffers took
//            6.50-6.58 ms, so the split stays.
template <int RES_BUFS, int STAGES, int CLUSTER>
int residual_gemm(bool latency, int T, const void* A, const void* B, int N, int K, float* h32, __nv_bfloat16* h16,
                  float* ss_out, cudaStream_t st) {
  EpiResidualParams ep{h32, h16, N, ss_out, T};
  if (!latency) return launch_gemm_ws<EpiWsResidual<RES_BUFS>, STAGES, CLUSTER>(A, K, B, K, T, N, K, ep, st);
  if (T <= kLatSmallMMaxTokens)
    return launch_gemm<kLatBlockN, EpiResidualChunkSS, false, kLatSmallStages, false, kLatSmallM>(A, K, B, K, T, N, K, ep, st);
  return launch_gemm<kLatBlockN, EpiResidualChunkSS, false, kLatStages>(A, K, B, K, T, N, K, ep, st);
}
int oproj_gemm(bool latency, int T, const void* A, const void* B, int N, int K, float* h32, __nv_bfloat16* h16,
               float* ss_out, cudaStream_t st) {
  return residual_gemm<2, 4, 1>(latency, T, A, B, N, K, h32, h16, ss_out, st);
}
int ffn_down_gemm(bool latency, int T, const void* A, const void* B, int N, int K, float* h32, __nv_bfloat16* h16,
                  float* ss_out, cudaStream_t st) {
  return residual_gemm<5, 3, 2>(latency, T, A, B, N, K, h32, h16, ss_out, st);
}

// out [T, N/2] = bf16(gelu_new(A B^T_gate * rs[m]) * (A B^T_linear * rs[m])).  B interleaves the gate and linear
// rows in 128-row blocks (rpx_encoder_create), and every tile pairs gate column j with linear column j + 128 of
// its 256-row block, so N must be a whole number of such blocks.
// The throughput path runs the core as pairs (kFfnUpCluster): at 2^18 tokens on an H100 80GB HBM3 at a 400 W power
// limit they took 11.60-11.87 ms against 12.61-12.70 ms unclustered (cuBLAS: 10.4-10.7 ms, tools/gemm_bench.py).
int ffn_up_gemm(bool latency, int T, const void* A, const void* B, int N, int K, const RowScale& rs,
                __nv_bfloat16* out, cudaStream_t st) {
  RPX_REQUIRE(N % 256 == 0, RPX_ERR_UNSUPPORTED, "ffn-up gemm: N=%d must be a multiple of 256 (2 x d_ff, d_ff %% 128 == 0)", N);
  const int F = N / 2;
  if (!latency) {
    EpiWsGeGLU::Params ep{out, F, rs};
    return launch_gemm_ws<EpiWsGeGLU, kFfnUpStages, kFfnUpCluster>(A, K, B, K, T, N, K, ep, st);
  }
  // hidden units per tile: 32 (64-column tiles, T <= 128: 112 CTAs) or 64 (128-column tiles: 56 x ceil(T/128))
  if (T <= kBlockM) {
    EpiGeGLUT<32>::Params ep{out, F, rs};
    return launch_gemm<64, EpiGeGLUT<32>, false, kLatStages, true>(A, K, B, K, T, N, K, ep, st);
  }
  EpiGeGLUT<64>::Params ep{out, F, rs};
  return launch_gemm<128, EpiGeGLUT<64>, false, kGemmStages, true>(A, K, B, K, T, N, K, ep, st);
}

int forward_latency_layer(rpx_encoder* e, const Workspace& ws, const LayerW& w, const void* next_weights,
                          size_t next_bytes, int T, int S, int max_len, cudaStream_t st) {
  const rpx_t5_config& c = e->cfg;
  const int D = c.d_model, inner = e->inner, F = c.d_ff, P = e->n_parts_lat;
  const float inv_d = 1.0f / (float)D;
  {
    Prof p(e, st, 1);
    // the QKV projection occupies 18 x ceil(T/64) (or 18 x ceil(T/128)) SMs for 6 heads: the rest of the GPU
    // fetches the next layer's weights into L2
    RPX_TRY(qkv_gemm(true, T, ws.h16, w.qkv, 3 * inner, D, RowScale{ws.ssA, P, T, inv_d, c.ln_eps}, ws.qkv, next_weights,
                     next_bytes, st));
  }
  {
    Prof p(e, st, 2);
    RPX_TRY(launch_t5_attention(ws.qkv, ws.attn, ws.cu_tokens, e->bias_lut, T, S, max_len, c.num_heads, c.d_kv,
                                c.rel_max_distance, st));
  }
  {
    Prof p(e, st, 3);
    RPX_TRY(oproj_gemm(true, T, ws.attn, w.o, D, inner, ws.h32, ws.h16, ws.ssB, st));
  }
  {
    Prof p(e, st, 4);
    RPX_TRY(ffn_up_gemm(true, T, ws.h16, w.wi, 2 * F, D, RowScale{ws.ssB, P, T, inv_d, c.ln_eps}, ws.ffn, st));
  }
  {
    Prof p(e, st, 5);
    RPX_TRY(ffn_down_gemm(true, T, ws.ffn, w.wo, D, F, ws.h32, ws.h16, ws.ssA, st));
  }
  return RPX_OK;
}

// What forward() writes after the last block.
//   kPooled  final RMSNorm + masked mean + L2 normalise: [S, D]
//   kHidden  final RMSNorm of every token (`last_hidden_state`): [S, seq_len, D], rows past a sequence's length zeroed
enum class OutKind { kPooled, kHidden };

// The forward pass proper.  ws.ids / ws.cu_tokens are already populated on `st`.  `seq_len` is the padded row
// length of a kHidden output (unused for kPooled).
int forward(rpx_encoder* e, const Workspace& ws, int T, int S, int max_len, OutKind kind, int seq_len, void* d_out,
            int out_dtype, cudaStream_t st) {
  const rpx_t5_config& c = e->cfg;
  const int D = c.d_model, inner = e->inner, F = c.d_ff;
  // the latency path needs d_ff in 128-unit blocks for its split-B tiles (validate_cfg) and narrow-tile n
  const bool latency = T <= e->latency_tokens && D % 32 == 0 && (3 * inner) % 32 == 0;
  const int P = latency ? e->n_parts_lat : e->n_parts;
  const float inv_d = 1.0f / (float)D;
  PdlScope pdl_scope(latency || T <= kPdlMaxTokens);
  {
    Prof p(e, st, 0);
    RPX_TRY(launch_embed(ws.ids, e->emb, ws.h32, ws.h16, ws.ssA, T, P, T, D, st));
  }
  auto dump = [&](int slab) -> int {
    if (e->debug_hidden)
      RPX_CUDA_OK(cudaMemcpyAsync(e->debug_hidden + (size_t)slab * T * D, ws.h32, (size_t)T * D * 4,
                                  cudaMemcpyDeviceToDevice, st));
    return RPX_OK;
  };
  RPX_TRY(dump(0));
  for (int l = 0; l < c.num_layers; ++l) {
    const LayerW& w = e->layers[l];
    if (latency) {
      const bool has_next = l + 1 < c.num_layers;
      RPX_TRY(forward_latency_layer(e, ws, w, has_next ? e->layers[l + 1].qkv : nullptr, has_next ? e->layer_bytes : 0, T, S,
                                    max_len, st));
      RPX_TRY(dump(l + 1));
      continue;
    }
    {
      Prof p(e, st, 1);
      RPX_TRY(qkv_gemm(false, T, ws.h16, w.qkv, 3 * inner, D, RowScale{ws.ssA, P, T, inv_d, c.ln_eps}, ws.qkv, nullptr, 0,
                       st));
    }
    {
      Prof p(e, st, 2);
      RPX_TRY(launch_t5_attention(ws.qkv, ws.attn, ws.cu_tokens, e->bias_lut, T, S, max_len, c.num_heads, c.d_kv,
                                  c.rel_max_distance, st));
    }
    {
      Prof p(e, st, 3);
      RPX_TRY(oproj_gemm(false, T, ws.attn, w.o, D, inner, ws.h32, ws.h16, ws.ssB, st));
    }
    {
      Prof p(e, st, 4);
      RPX_TRY(ffn_up_gemm(false, T, ws.h16, w.wi, 2 * F, D, RowScale{ws.ssB, P, T, inv_d, c.ln_eps}, ws.ffn, st));
    }
    {
      Prof p(e, st, 5);
      RPX_TRY(ffn_down_gemm(false, T, ws.ffn, w.wo, D, F, ws.h32, ws.h16, ws.ssA, st));
    }
    RPX_TRY(dump(l + 1));
  }
  if (kind == OutKind::kHidden) {
    Prof p(e, st, 6);
    // the latency path pools with pool_partial_kernel: its order of the ss parts keeps the rows consistent with it
    RPX_TRY(launch_hidden_store(ws.h32, ws.ssA, T, P, latency, e->final_ln, ws.cu_tokens, d_out, out_dtype, S, seq_len, D,
                                c.ln_eps, st));
  } else {
    Prof p(e, st, 6);
    // latency path: per-group partial rows go where the (now dead) FFN activations were — T rows of d_ff
    // bf16 hold T rows of d_model fp32 when d_ff >= 2 d_model (else the single-kernel pool runs)
    float* scratch = latency && (size_t)F * 2 >= (size_t)D * 4 ? reinterpret_cast<float*>(ws.ffn) : nullptr;
    RPX_TRY(launch_pool_normalize(ws.h32, ws.ssA, T, P, e->final_ln, ws.cu_tokens, d_out, out_dtype, S, D,
                                  c.ln_eps, st, scratch, max_len));
  }
  return RPX_OK;
}

}  // namespace
}  // namespace rpx

using namespace rpx;

extern "C" {

size_t rpx_encoder_packed_bytes(const rpx_t5_config* cfg) {
  if (validate_cfg(cfg) != RPX_OK) return 0;
  return packed_layout(*cfg).total;
}

int rpx_encoder_create(const rpx_t5_config* cfg, const rpx_t5_weights* w, void* d_packed, size_t packed_bytes,
                       void* stream, rpx_encoder** out) {
  RPX_TRY(validate_cfg(cfg));
  RPX_REQUIRE(w && d_packed && out, RPX_ERR_INVALID, "rpx_encoder_create: null argument");
  DeviceInfo dev;
  RPX_TRY(get_device_info(&dev));
  const PackedLayout L = packed_layout(*cfg);
  RPX_REQUIRE(packed_bytes >= L.total, RPX_ERR_WORKSPACE, "packed buffer too small: %zu < %zu", packed_bytes, L.total);
  RPX_REQUIRE((reinterpret_cast<uintptr_t>(d_packed) & 255) == 0, RPX_ERR_INVALID, "packed buffer must be 256-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* base = static_cast<uint8_t*>(d_packed);
  const int D = cfg->d_model, inner = cfg->num_heads * cfg->d_kv, F = cfg->d_ff;

  rpx_encoder* e = new (std::nothrow) rpx_encoder();
  RPX_REQUIRE(e != nullptr, RPX_ERR_INVALID, "out of host memory");
  e->cfg = *cfg;
  e->inner = inner;
  e->n_parts = ss_parts(D, false);
  e->n_parts_lat = ss_parts(D, true);
  auto fail = [&](int code) {
    delete e;
    return code;
  };
#define TRY_E(expr)                        \
  do {                                     \
    int _s = (expr);                       \
    if (_s != RPX_OK) return fail(_s);     \
  } while (0)
#define CUDA_E(expr)                                                                                   \
  do {                                                                                                 \
    cudaError_t _c = (expr);                                                                           \
    if (_c != cudaSuccess) {                                                                           \
      set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_c));           \
      return fail(RPX_ERR_CUDA);                                                                       \
    }                                                                                                  \
  } while (0)

  CUDA_E(cudaMemcpyAsync(base + L.emb, w->d_shared, (size_t)cfg->vocab_size * D * 4, cudaMemcpyDeviceToDevice, st));
  CUDA_E(cudaMemcpyAsync(base + L.final_ln, w->d_final_ln, (size_t)D * 4, cudaMemcpyDeviceToDevice, st));
  e->emb = reinterpret_cast<const float*>(base + L.emb);
  e->final_ln = reinterpret_cast<const float*>(base + L.final_ln);

  TRY_E(build_bias_lut(w->d_rel_bias, cfg->num_heads, cfg->rel_buckets, cfg->rel_max_distance,
                       reinterpret_cast<int32_t*>(base + L.bucket_tmp), reinterpret_cast<float*>(base + L.bias_lut), st));
  e->bias_lut = reinterpret_cast<const float*>(base + L.bias_lut);

  e->layers.resize(cfg->num_layers);
  for (int l = 0; l < cfg->num_layers; ++l) {
    uint8_t* lb = base + L.layer0 + L.layer_stride * l;
    __nv_bfloat16* qkv = reinterpret_cast<__nv_bfloat16*>(lb + L.qkv);
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(lb + L.o);
    __nv_bfloat16* wi = reinterpret_cast<__nv_bfloat16*>(lb + L.wi);
    __nv_bfloat16* wo = reinterpret_cast<__nv_bfloat16*>(lb + L.wo);
    // q | k | v stacked, RMSNorm(ln0) weight folded along K
    TRY_E(launch_pack_weight(w->h_q[l], w->h_ln0[l], qkv, inner, D, 0, inner, inner, st));
    TRY_E(launch_pack_weight(w->h_k[l], w->h_ln0[l], qkv, inner, D, inner, inner, inner, st));
    TRY_E(launch_pack_weight(w->h_v[l], w->h_ln0[l], qkv, inner, D, 2 * inner, inner, inner, st));
    TRY_E(launch_pack_weight(w->h_o[l], nullptr, o, D, inner, 0, D, D, st));
    // wi_0 rows -> [j*256, j*256+128), wi_1 rows -> [j*256+128, j*256+256); ln1 folded
    TRY_E(launch_pack_weight(w->h_wi0[l], w->h_ln1[l], wi, F, D, 0, 128, 256, st));
    TRY_E(launch_pack_weight(w->h_wi1[l], w->h_ln1[l], wi, F, D, 128, 128, 256, st));
    TRY_E(launch_pack_weight(w->h_wo[l], nullptr, wo, D, F, 0, D, D, st));
    e->layers[l] = LayerW{qkv, o, wi, wo};
    e->layer_bytes = L.layer_stride;
  }
  // the packed image is complete on return, so the caller may release the fp32 weights at once
  CUDA_E(cudaStreamSynchronize(st));
#undef TRY_E
#undef CUDA_E
  *out = e;
  return RPX_OK;
}

int rpx_encoder_destroy(rpx_encoder* enc) {
  if (!enc) return RPX_OK;
  for (auto& r : enc->prof_pending) {
    cudaEventDestroy(r.a);
    cudaEventDestroy(r.b);
  }
  for (auto ev : enc->event_pool) cudaEventDestroy(ev);
  delete enc;
  return RPX_OK;
}

size_t rpx_encoder_workspace_bytes(const rpx_encoder* enc, int64_t max_tokens, int64_t max_seqs) {
  if (!enc || max_tokens <= 0 || max_seqs <= 0) return 0;
  return carve(enc, nullptr, max_tokens, max_seqs).total;
}

int rpx_encode_bytes(rpx_encoder* enc, const uint8_t* d_bytes, const int64_t* h_offsets, int32_t n_seqs,
                     int32_t max_seq_len, void* d_out, int32_t out_dtype, void* d_workspace,
                     size_t workspace_bytes, void* stream) {
  RPX_REQUIRE(enc && h_offsets && d_out && d_workspace, RPX_ERR_INVALID, "rpx_encode_bytes: null argument");
  RPX_REQUIRE(n_seqs > 0, RPX_ERR_INVALID, "rpx_encode_bytes: n_seqs=%d", n_seqs);
  RPX_REQUIRE(max_seq_len >= 1, RPX_ERR_INVALID, "rpx_encode_bytes: max_seq_len=%d", max_seq_len);
  RPX_REQUIRE(h_offsets[0] >= 0, RPX_ERR_INVALID, "rpx_encode_bytes: negative offset");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  auto& cu = enc->h_cu_tokens;
  cu.resize((size_t)n_seqs + 1);
  cu[0] = 0;
  int max_len = 0;
  int64_t total = 0;
  for (int s = 0; s < n_seqs; ++s) {
    const int64_t nb = h_offsets[s + 1] - h_offsets[s];
    RPX_REQUIRE(nb >= 0, RPX_ERR_INVALID, "rpx_encode_bytes: offsets not monotone at %d", s);
    const int64_t nt = nb + 1 < (int64_t)max_seq_len ? nb + 1 : (int64_t)max_seq_len;
    total += nt;
    RPX_REQUIRE(total < (int64_t)INT32_MAX, RPX_ERR_UNSUPPORTED, "rpx_encode_bytes: more than 2^31 tokens in one call");
    cu[s + 1] = (int32_t)total;
    if ((int)nt > max_len) max_len = (int)nt;
  }
  RPX_REQUIRE(d_bytes != nullptr || h_offsets[n_seqs] == h_offsets[0], RPX_ERR_INVALID, "rpx_encode_bytes: d_bytes is null");
  const int T = (int)total;
  const Workspace ws = carve(enc, static_cast<uint8_t*>(d_workspace), T, n_seqs);
  RPX_REQUIRE(ws.total <= workspace_bytes, RPX_ERR_WORKSPACE, "workspace too small: need %zu, have %zu (tokens=%d seqs=%d)",
              ws.total, workspace_bytes, T, n_seqs);
  RPX_REQUIRE((reinterpret_cast<uintptr_t>(d_workspace) & 255) == 0, RPX_ERR_INVALID, "workspace must be 256-byte aligned");
  RPX_CUDA_OK(cudaMemcpyAsync(ws.cu_tokens, cu.data(), ((size_t)n_seqs + 1) * 4, cudaMemcpyHostToDevice, st));
  RPX_CUDA_OK(cudaMemcpyAsync(ws.cu_bytes, h_offsets, ((size_t)n_seqs + 1) * 8, cudaMemcpyHostToDevice, st));
  RPX_TRY(launch_tokenize_bytes(d_bytes, ws.cu_bytes, ws.cu_tokens, ws.ids, n_seqs, T, st));
  return forward(enc, ws, T, n_seqs, max_len, OutKind::kPooled, 0, d_out, out_dtype, st);
}

}  // extern "C"

namespace {

// rpx_encode_ids and rpx_encode_ids_hidden on padded int64 [batch, seq_len] ids: validate, take the row lengths
// from the mask (seq_len for every row without one), pack the ids, run the forward pass, report ids outside the
// vocabulary.  `fn` names the entry point in error messages.
int encode_padded_ids(const char* fn, rpx_encoder* enc, const int64_t* d_input_ids, const int64_t* d_attention_mask,
                      int32_t batch, int32_t seq_len, OutKind kind, void* d_out, int32_t out_dtype, void* d_workspace,
                      size_t workspace_bytes, void* stream) {
  RPX_REQUIRE(enc && d_input_ids && d_out && d_workspace, RPX_ERR_INVALID, "%s: null argument", fn);
  RPX_REQUIRE(batch > 0 && seq_len > 0, RPX_ERR_INVALID, "%s: batch=%d seq_len=%d", fn, batch, seq_len);
  RPX_REQUIRE((int64_t)batch * seq_len < (int64_t)INT32_MAX, RPX_ERR_UNSUPPORTED, "%s: batch too large", fn);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // Worst case all tokens valid: the workspace must fit that (callers size it with batch*seq_len).
  const Workspace ws_max = carve(enc, static_cast<uint8_t*>(d_workspace), (int64_t)batch * seq_len, batch);
  RPX_REQUIRE(ws_max.total <= workspace_bytes, RPX_ERR_WORKSPACE, "workspace too small: need %zu, have %zu", ws_max.total,
              workspace_bytes);
  RPX_REQUIRE((reinterpret_cast<uintptr_t>(d_workspace) & 255) == 0, RPX_ERR_INVALID, "workspace must be 256-byte aligned");
  RPX_CUDA_OK(cudaMemsetAsync(ws_max.flag, 0, 4, st));
  auto& lens = enc->h_lens;
  lens.assign((size_t)batch + 1, seq_len);
  if (d_attention_mask) {
    RPX_TRY(launch_mask_lengths(d_attention_mask, ws_max.lens, ws_max.flag, batch, seq_len, st));
    RPX_CUDA_OK(cudaMemcpyAsync(lens.data(), ws_max.lens, (size_t)batch * 4, cudaMemcpyDeviceToHost, st));
    RPX_CUDA_OK(cudaMemcpyAsync(&lens[batch], ws_max.flag, 4, cudaMemcpyDeviceToHost, st));
    RPX_CUDA_OK(cudaStreamSynchronize(st));
    RPX_REQUIRE(lens[batch] == 0, RPX_ERR_MASK,
                "attention_mask must be a right-padded prefix of ones with at least one token per row");
  }
  auto& cu = enc->h_cu_tokens;
  cu.resize((size_t)batch + 1);
  cu[0] = 0;
  int max_len = 0;
  for (int b = 0; b < batch; ++b) {
    cu[b + 1] = cu[b] + lens[b];
    if (lens[b] > max_len) max_len = lens[b];
  }
  const int T = cu[batch];
  // Same carve order/sizes as ws_max for the leading (S-sized) members, so cu_tokens/flag do not move;
  // the T-sized members are re-carved for the actual token count.
  const Workspace ws = carve(enc, static_cast<uint8_t*>(d_workspace), T, batch);
  RPX_CUDA_OK(cudaMemcpyAsync(ws.cu_tokens, cu.data(), ((size_t)batch + 1) * 4, cudaMemcpyHostToDevice, st));
  RPX_TRY(launch_pack_ids(d_input_ids, ws.cu_tokens, ws.ids, batch, seq_len, T, enc->cfg.vocab_size, ws.flag, st));
  RPX_TRY(forward(enc, ws, T, batch, max_len, kind, seq_len, d_out, out_dtype, st));
  // ids outside [0, vocab) are reported after the fact (the forward ran with id 0 in their place).
  int32_t flag = 0;
  RPX_CUDA_OK(cudaMemcpyAsync(&flag, ws.flag, 4, cudaMemcpyDeviceToHost, st));
  RPX_CUDA_OK(cudaStreamSynchronize(st));
  RPX_REQUIRE((flag & 2) == 0, RPX_ERR_INVALID, "input_ids contains ids outside [0, %d)", enc->cfg.vocab_size);
  return RPX_OK;
}

}  // namespace

extern "C" {

int rpx_encode_ids(rpx_encoder* enc, const int64_t* d_input_ids, const int64_t* d_attention_mask, int32_t batch,
                   int32_t seq_len, void* d_out, int32_t out_dtype, void* d_workspace, size_t workspace_bytes,
                   void* stream) {
  RPX_REQUIRE(d_attention_mask, RPX_ERR_INVALID, "rpx_encode_ids: null argument");
  return encode_padded_ids("rpx_encode_ids", enc, d_input_ids, d_attention_mask, batch, seq_len, OutKind::kPooled, d_out,
                           out_dtype, d_workspace, workspace_bytes, stream);
}

int rpx_encode_ids_hidden(rpx_encoder* enc, const int64_t* d_input_ids, const int64_t* d_attention_mask, int32_t batch,
                          int32_t seq_len, void* d_out, int32_t out_dtype, void* d_workspace, size_t workspace_bytes,
                          void* stream) {
  RPX_REQUIRE(out_dtype == RPX_DTYPE_BF16 || out_dtype == RPX_DTYPE_F32, RPX_ERR_INVALID,
              "rpx_encode_ids_hidden: out_dtype=%d", out_dtype);
  RPX_REQUIRE((reinterpret_cast<uintptr_t>(d_out) & 15) == 0, RPX_ERR_INVALID,
              "rpx_encode_ids_hidden: d_out must be 16-byte aligned");
  return encode_padded_ids("rpx_encode_ids_hidden", enc, d_input_ids, d_attention_mask, batch, seq_len, OutKind::kHidden,
                           d_out, out_dtype, d_workspace, workspace_bytes, stream);
}

int rpx_encoder_set_latency_tokens(rpx_encoder* enc, int32_t max_tokens) {
  RPX_REQUIRE(enc, RPX_ERR_INVALID, "null encoder");
  RPX_REQUIRE(max_tokens >= 0, RPX_ERR_INVALID, "rpx_encoder_set_latency_tokens: %d", max_tokens);
  enc->latency_tokens = max_tokens;
  return RPX_OK;
}

int rpx_encoder_set_debug_hidden(rpx_encoder* enc, float* d_hidden) {
  RPX_REQUIRE(enc, RPX_ERR_INVALID, "null encoder");
  enc->debug_hidden = d_hidden;
  return RPX_OK;
}

int rpx_encoder_set_profiling(rpx_encoder* enc, int32_t enable) {
  RPX_REQUIRE(enc, RPX_ERR_INVALID, "null encoder");
  enc->profiling = enable != 0;
  return RPX_OK;
}

int rpx_debug_encoder_gemm(int32_t site, int32_t latency, const void* d_A, const void* d_B, int32_t T, int32_t N,
                           int32_t K, float ln_eps, const float* d_ss_in, void* d_out, float* d_h32, void* d_h16,
                           float* d_ss_out, const void* d_prefetch, size_t prefetch_bytes, void* stream) {
  RPX_REQUIRE(site >= RPX_EGEMM_QKV && site <= RPX_EGEMM_FFN_DOWN, RPX_ERR_INVALID, "rpx_debug_encoder_gemm: site=%d", site);
  RPX_REQUIRE(d_A && d_B, RPX_ERR_INVALID, "rpx_debug_encoder_gemm: null operand");
  RPX_REQUIRE(T > 0 && N > 0 && K > 0, RPX_ERR_INVALID, "rpx_debug_encoder_gemm: T=%d N=%d K=%d", T, N, K);
  const bool lat = latency != 0;
  const bool residual = site == RPX_EGEMM_OPROJ || site == RPX_EGEMM_FFN_DOWN;
  const int D = residual ? N : K;
  RPX_REQUIRE(D % 64 == 0, RPX_ERR_UNSUPPORTED, "rpx_debug_encoder_gemm: d_model=%d must be a multiple of 64", D);
  if (residual)
    RPX_REQUIRE(d_h32 && d_h16 && d_ss_out, RPX_ERR_INVALID, "rpx_debug_encoder_gemm: residual site needs h32, h16, ss_out");
  else
    RPX_REQUIRE(d_ss_in && d_out, RPX_ERR_INVALID, "rpx_debug_encoder_gemm: site %d needs ss_in and out", site);
  RPX_REQUIRE(d_prefetch == nullptr || (lat && site == RPX_EGEMM_QKV), RPX_ERR_INVALID,
              "rpx_debug_encoder_gemm: only the latency QKV projection prefetches");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PdlScope pdl_scope(lat || T <= kPdlMaxTokens);
  const RowScale rs{d_ss_in, ss_parts(D, lat), T, 1.0f / (float)D, ln_eps};
  auto* out = static_cast<__nv_bfloat16*>(d_out);
  auto* h16 = static_cast<__nv_bfloat16*>(d_h16);
  switch (site) {
    case RPX_EGEMM_QKV: return qkv_gemm(lat, T, d_A, d_B, N, K, rs, out, d_prefetch, prefetch_bytes, st);
    case RPX_EGEMM_OPROJ: return oproj_gemm(lat, T, d_A, d_B, N, K, d_h32, h16, d_ss_out, st);
    case RPX_EGEMM_FFN_UP: return ffn_up_gemm(lat, T, d_A, d_B, N, K, rs, out, st);
    default: return ffn_down_gemm(lat, T, d_A, d_B, N, K, d_h32, h16, d_ss_out, st);
  }
}

int rpx_debug_attention_lut(const float* d_rel_bias, int32_t n_heads, int32_t rel_buckets, int32_t rel_max_distance,
                            float* d_lut, void* stream) {
  RPX_REQUIRE(d_rel_bias && d_lut, RPX_ERR_INVALID, "rpx_debug_attention_lut: null argument");
  RPX_REQUIRE(n_heads > 0, RPX_ERR_INVALID, "rpx_debug_attention_lut: n_heads=%d", n_heads);
  RPX_TRY(check_rel_attention(rel_buckets, rel_max_distance));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int32_t* d_buckets = nullptr;
  RPX_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&d_buckets), (size_t)(2 * rel_max_distance + 1) * 4, st));
  const int rc = build_bias_lut(d_rel_bias, n_heads, rel_buckets, rel_max_distance, d_buckets, d_lut, st);
  RPX_CUDA_OK(cudaFreeAsync(d_buckets, st));
  return rc;
}

int rpx_debug_attention(int32_t latency, const void* d_qkv, void* d_out, const int32_t* d_cu_seqlens,
                        const float* d_lut, int32_t n_tokens, int32_t n_seqs, int32_t max_len, int32_t n_heads,
                        int32_t rel_max_distance, void* stream) {
  RPX_REQUIRE(d_qkv && d_out && d_cu_seqlens && d_lut, RPX_ERR_INVALID, "rpx_debug_attention: null argument");
  RPX_REQUIRE(n_tokens > 0 && max_len > 0 && n_heads > 0, RPX_ERR_INVALID,
              "rpx_debug_attention: n_tokens=%d max_len=%d n_heads=%d", n_tokens, max_len, n_heads);
  RPX_REQUIRE(n_seqs > 0, RPX_ERR_INVALID, "rpx_debug_attention: n_seqs=%d", n_seqs);
  RPX_REQUIRE(n_seqs <= 65535, RPX_ERR_UNSUPPORTED, "rpx_debug_attention: n_seqs=%d exceeds the 65535 grid limit", n_seqs);
  RPX_REQUIRE(rel_max_distance > 0 && rel_max_distance <= 2048, RPX_ERR_INVALID,
              "rpx_debug_attention: rel_max_distance=%d", rel_max_distance);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  PdlScope pdl_scope(latency != 0 || n_tokens <= kPdlMaxTokens);
  return launch_t5_attention(static_cast<const __nv_bfloat16*>(d_qkv), static_cast<__nv_bfloat16*>(d_out), d_cu_seqlens,
                             d_lut, n_tokens, n_seqs, max_len, n_heads, 64, rel_max_distance, st);
}

int rpx_encoder_read_profile(rpx_encoder* enc, float* h_ms, int64_t* h_launches) {
  RPX_REQUIRE(enc && h_ms && h_launches, RPX_ERR_INVALID, "null argument");
  for (auto& r : enc->prof_pending) {
    RPX_CUDA_OK(cudaEventSynchronize(r.b));
    float ms = 0.f;
    RPX_CUDA_OK(cudaEventElapsedTime(&ms, r.a, r.b));
    enc->prof_ms[r.cls] += ms;
    enc->prof_launches[r.cls] += 1;
    enc->event_pool.push_back(r.a);
    enc->event_pool.push_back(r.b);
  }
  enc->prof_pending.clear();
  for (int i = 0; i < RPX_N_KERNEL_CLASSES; ++i) {
    h_ms[i] = enc->prof_ms[i];
    h_launches[i] = enc->prof_launches[i];
    enc->prof_ms[i] = 0.f;
    enc->prof_launches[i] = 0;
  }
  return RPX_OK;
}

}  // extern "C"
