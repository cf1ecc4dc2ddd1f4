// rpx_decoder.cu — the tactic generator's teacher-forced forward: HF T5ForConditionalGeneration(input_ids,
// attention_mask, labels) (modeling_t5.py, T5ForConditionalGeneration.forward; the reference calls it at
// generation/model.py:101-111) on packed tokens.
//
//   encoder    forward() of rpx_encoder.cu over the states, stopped before the final RMSNorm (OutKind::kResidual)
//   cross K/V  one GEMM for every decoder layer: [T_enc, D] x [n_dec_layers * 2 * inner, D]^T with
//              encoder.final_layer_norm folded into B and the row scale of the encoder's last partial sums in the
//              epilogue (the QKV launcher), so the encoder's final hidden state is never materialised
//   decoder    embed(_shift_right(labels)), then per layer, each GEMM through the encoder's launchers:
//                h += O(causal_attn(RMSNorm(h)))             self-attention, unidirectional bias
//                h += O_c(cross_attn(Q_c RMSNorm(h), K/V))   no bias; keys = the row's encoder tokens
//                h += wo(gelu_new(wi_0 n) * (wi_1 n))        n = RMSNorm(h)
//   head       logits = RMSNorm(h) W_head^T (decoder.final_layer_norm and the optional d_model ** -0.5 folded
//              into W_head), fp32; then per decoder token log_softmax and the label's log-probability, per row
//              their sum in token order.
// Row b's decoder tokens are positions [0, len_b) with len_b = 1 + the last position whose label is not -100; the
// positions past it are never computed.
//
// The encoder and the cross K / V are the prefill that rpx_seq2seq_forward, rpx_seq2seq_generate and
// rpx_seq2seq_evaluate share (`prefill` below); evaluate runs it once and hands it to both the teacher-forced half and
// the search, as the reference's `validation_step` needs both on one batch.
#include <math.h>

#include <new>
#include <vector>

#include "rpx_encoder.cuh"
#include "rpx_gemm_launch.cuh"
#include "rpx_kernels.cuh"

namespace rpx {
namespace {

struct DecLayerW {
  const __nv_bfloat16* qkv;  // [3*inner, D]  (ln0 folded)
  const __nv_bfloat16* o;    // [D, inner]
  const __nv_bfloat16* cq;   // [inner, D]    (ln1 folded)
  const __nv_bfloat16* co;   // [D, inner]
  const __nv_bfloat16* wi;   // [2*d_ff, D]   (ln2 folded; wi_0 / wi_1 interleaved in 128-row blocks)
  const __nv_bfloat16* wo;   // [D, d_ff]
};

}  // namespace
}  // namespace rpx

struct rpx_t5_decoder {
  rpx_t5_config cfg;
  int inner = 0;
  int n_parts = 0;  // RMSNorm partial sums per row (throughput path)
  int n_kv = 0;     // columns of the cross K / V matrix: num_layers * 2 * inner
  int start_id = 0;
  const float* emb = nullptr;
  const float* bias_lut = nullptr;
  const __nv_bfloat16* head = nullptr;     // [vocab, D]
  const __nv_bfloat16* cross_kv = nullptr;  // [n_kv, D]: layer l's K rows at 2 l inner, V rows at (2 l + 1) inner
  std::vector<rpx::DecLayerW> layers;
  std::vector<int32_t> h_lens;  // enc lens [B], enc flag, dec lens [B], dec flag
  std::vector<int32_t> h_cu;
  // generate: pinned words the host polls (done-state counts of two step blocks, out_len, ids flag) and the events
  // that mark them written
  int32_t* h_poll = nullptr;
  cudaEvent_t poll_ev[2] = {nullptr, nullptr};
};

namespace rpx {
namespace {

constexpr int kIgnore = -100;  // HF CrossEntropyLoss ignore_index, and what `_shift_right` replaces by the pad id

struct DecPackedLayout {
  size_t emb, bias_lut, bucket_tmp, head_scale, head, cross_kv, layer0, layer_stride, qkv, o, cq, co, wi, wo, total;
};

DecPackedLayout dec_packed_layout(const rpx_t5_config& c) {
  DecPackedLayout L{};
  const size_t D = c.d_model, inner = (size_t)c.num_heads * c.d_kv, F = c.d_ff, V = c.vocab_size;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off = align_up(off + bytes, 256);
    return o;
  };
  L.emb = take(V * D * 4);
  L.bias_lut = take((size_t)c.num_heads * (2 * c.rel_max_distance + 1) * 4);
  L.bucket_tmp = take((size_t)(2 * c.rel_max_distance + 1) * 4);
  L.head_scale = take(D * 4);
  L.head = take(V * D * 2);
  L.cross_kv = take((size_t)c.num_layers * 2 * inner * D * 2);
  L.layer0 = off;
  size_t lo = 0;
  auto ltake = [&](size_t bytes) {
    size_t o = lo;
    lo = align_up(lo + bytes, 256);
    return o;
  };
  L.qkv = ltake(3 * inner * D * 2);
  L.o = ltake(D * inner * 2);
  L.cq = ltake(inner * D * 2);
  L.co = ltake(D * inner * 2);
  L.wi = ltake(2 * F * D * 2);
  L.wo = ltake(D * F * 2);
  L.layer_stride = lo;
  L.total = L.layer0 + lo * (size_t)c.num_layers;
  return L;
}

int validate_dec_cfg(const rpx_t5_config* c) {
  RPX_TRY(validate_cfg(c));
  RPX_TRY(check_rel_attention(c->rel_buckets, c->rel_max_distance, false));
  // the head GEMM's n-tiles: N % 32 == 0
  RPX_REQUIRE(c->vocab_size % 32 == 0, RPX_ERR_UNSUPPORTED, "decoder: vocab_size=%d must be a multiple of 32",
              c->vocab_size);
  return RPX_OK;
}

__global__ void scale_vec_kernel(const float* __restrict__ src, float s, float* __restrict__ dst, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[i] * s;
}

// One warp per row of labels [batch, out_len]: lens[b] = 1 + the last position whose label is not -100 (0 if none);
// flag |= 2 when a label is neither -100 nor in [0, vocab).
__global__ void label_lengths_kernel(const int64_t* __restrict__ labels, int32_t* __restrict__ lens,
                                     int32_t* __restrict__ bad_flag, int batch, int out_len, int vocab) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= batch) return;
  int last = -1, bad = 0;
  for (int j = lane; j < out_len; j += 32) {
    const int64_t y = labels[(int64_t)row * out_len + j];
    if (y != kIgnore) {
      last = j;
      if (y < 0 || y >= vocab) bad = 1;
    }
  }
  for (int off = 16; off; off >>= 1) {
    last = max(last, __shfl_xor_sync(0xffffffffu, last, off));
    bad |= __shfl_xor_sync(0xffffffffu, bad, off);
  }
  if (lane == 0) {
    lens[row] = last + 1;
    if (bad) atomicOr(bad_flag, 2);
  }
}

// Largest s with cu[s] <= t  (cu is non-decreasing, cu[0] = 0, cu[n] > t).
__device__ __forceinline__ int find_row(const int32_t* __restrict__ cu, int n, int t) {
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (cu[mid] <= t) lo = mid; else hi = mid;
  }
  return lo;
}

// HF `_shift_right` on packed decoder tokens: token p of row b is fed start (p = 0) or labels[b, p - 1], -100 fed as
// the pad id (= start, checked by the caller); its target is labels[b, p].
__global__ void pack_decoder_kernel(const int64_t* __restrict__ labels, const int32_t* __restrict__ cu,
                                    int32_t* __restrict__ in_ids, int32_t* __restrict__ targets, int batch,
                                    int out_len, int n_tokens, int start_id) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_tokens) return;
  const int b = find_row(cu, batch, t);
  const int p = t - cu[b];
  const int64_t* row = labels + (int64_t)b * out_len;
  const int64_t prev = p == 0 ? (int64_t)start_id : row[p - 1];
  in_ids[t] = prev == kIgnore ? start_id : (int32_t)prev;
  targets[t] = (int32_t)row[p];
}

// One warp per decoder token: log_softmax over the vocab of its fp32 logits row, lp[t] = that of its target (0 for
// an ignored target).  The maximum in fp32, the sum of exp(x - max) in fp64 (lane-strided, then a fixed xor tree).
__global__ void token_logprob_kernel(const float* __restrict__ logits, const int32_t* __restrict__ targets,
                                     double* __restrict__ lp, int n_tokens, int vocab) {
  const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= n_tokens) return;
  const float* x = logits + (int64_t)t * vocab;
  float mx = -INFINITY;
  for (int j = lane; j < vocab; j += 32) mx = fmaxf(mx, x[j]);
  for (int off = 16; off; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
  double s = 0.0;
  for (int j = lane; j < vocab; j += 32) s += exp((double)x[j] - (double)mx);
  for (int off = 16; off; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if (lane == 0) {
    const int y = targets[t];
    lp[t] = y == kIgnore ? 0.0 : ((double)x[y] - (double)mx) - log(s);
  }
}

// One thread per row: the sum of its counted tokens' log-probabilities in token order, and their count.
__global__ void seq_logprob_kernel(const double* __restrict__ lp, const int32_t* __restrict__ targets,
                                   const int32_t* __restrict__ cu, double* __restrict__ seq_lp,
                                   int32_t* __restrict__ seq_count, int batch) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  double s = 0.0;
  int n = 0;
  for (int t = cu[b]; t < cu[b + 1]; ++t) {
    if (targets[t] != kIgnore) {
      s += lp[t];
      ++n;
    }
  }
  seq_lp[b] = s;
  seq_count[b] = n;
}

// One warp per output row (b, p) of logits [batch, out_len, vocab]: decoder token cu[b] + p while p < len_b, zeros
// past it.  vocab % 4 == 0.
__global__ void scatter_logits_kernel(const float* __restrict__ packed, const int32_t* __restrict__ cu,
                                      float* __restrict__ out, int64_t n_rows, int out_len, int vocab) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= n_rows) return;
  const int b = (int)(row / out_len), p = (int)(row % out_len);
  const int t0 = cu[b], len = cu[b + 1] - t0;
  float4* dst = reinterpret_cast<float4*>(out + row * vocab);
  const int n4 = vocab >> 2;
  if (p >= len) {
    for (int c = lane; c < n4; c += 32) dst[c] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  const float4* src = reinterpret_cast<const float4*>(packed + (int64_t)(t0 + p) * vocab);
  for (int c = lane; c < n4; c += 32) dst[c] = src[c];
}

// Device buffers of one call.  Every region is sized for the worst case (all positions tokens), so none moves with
// the actual token counts; within the forward workspaces, carve() keeps the S-sized members in place.  The prefill's
// regions (the encoder's workspace and the cross K / V) come first; each half carves its own regions after them, from
// `base` on.  Each carve_* sizes only when `base` is null.
struct PrefillWs {
  size_t enc_off;
  __nv_bfloat16* cross_kv;  // [B * in_len, n_kv]
  size_t total;
};

// The teacher-forced half: the decoder's workspace (the encoder's members, for the decoder tokens) and its own.
struct SeqWs {
  size_t dec_off;
  float* logits;            // [B * out_len, vocab]
  double* tok_lp;           // [B * out_len]
  int32_t* targets;         // [B * out_len]
  size_t total;
};

struct Carver {
  uint8_t* base;
  size_t off = 0;
  uint8_t* take(size_t bytes) {
    uint8_t* p = base ? base + off : nullptr;
    off = align_up(off + bytes, 256);
    return p;
  }
};

PrefillWs carve_prefill(const rpx_t5_decoder* d, const rpx_encoder* e, uint8_t* base, int64_t B, int64_t in_len) {
  PrefillWs w{};
  const int64_t Te = B * in_len;
  Carver c{base};
  w.enc_off = c.off;
  c.take(carve(e, nullptr, Te, B).total);
  w.cross_kv = (__nv_bfloat16*)c.take((size_t)Te * d->n_kv * 2);
  w.total = c.off;
  return w;
}

SeqWs carve_seq(const rpx_t5_decoder* d, const rpx_encoder* e, uint8_t* base, int64_t B, int64_t out_len) {
  SeqWs w{};
  const int64_t Td = B * out_len;
  Carver c{base};
  w.dec_off = c.off;
  c.take(carve(e, nullptr, Td, B).total);
  w.logits = (float*)c.take((size_t)Td * d->cfg.vocab_size * 4);
  w.tok_lp = (double*)c.take((size_t)Td * 8);
  w.targets = (int32_t*)c.take((size_t)Td * 4);
  w.total = c.off;
  return w;
}

int check_pair(const rpx_t5_decoder* d, const rpx_encoder* e) {
  const rpx_t5_config &a = d->cfg, &b = e->cfg;
  RPX_REQUIRE(a.vocab_size == b.vocab_size && a.d_model == b.d_model && a.d_kv == b.d_kv && a.d_ff == b.d_ff &&
                  a.num_heads == b.num_heads && a.ln_eps == b.ln_eps,
              RPX_ERR_INVALID, "decoder and encoder configs differ (vocab, d_model, d_kv, d_ff, heads or eps)");
  return RPX_OK;
}

// One decoder block: self-attention, cross-attention, FFN.  The RMSNorm partial sums enter in *ss_in and leave in
// *ss_in as well (the two buffers alternate three times).
int decoder_layer(const rpx_t5_decoder* d, const DecLayerW& w, int layer, const Workspace& ws, int T, int B,
                  int max_len, const __nv_bfloat16* cross_kv, int T_enc, const int32_t* cu_enc, float** ss_in,
                  float** ss_other, cudaStream_t st) {
  const rpx_t5_config& c = d->cfg;
  const int D = c.d_model, inner = d->inner, F = c.d_ff, P = d->n_parts;
  const float inv_d = 1.0f / (float)D;
  float* sa = *ss_in;
  float* sb = *ss_other;
  RPX_TRY(qkv_gemm(false, T, ws.h16, w.qkv, 3 * inner, D, RowScale{sa, P, T, inv_d, c.ln_eps}, ws.qkv, nullptr, 0, st));
  AttnArgs self{ws.qkv, T, 3 * inner, 0, ws.qkv, T, 3 * inner, inner, 2 * inner, ws.attn, inner, ws.cu_tokens,
                ws.cu_tokens, d->bias_lut, B, max_len, c.num_heads, c.d_kv, c.rel_max_distance};
  RPX_TRY(launch_t5_attention_mode(AttnMode::kCausal, self, st));
  RPX_TRY(oproj_gemm(false, T, ws.attn, w.o, D, inner, ws.h32, ws.h16, sb, st));
  // cross-attention queries go where the (consumed) self-attention q | k | v were
  RPX_TRY(qkv_gemm(false, T, ws.h16, w.cq, inner, D, RowScale{sb, P, T, inv_d, c.ln_eps}, ws.qkv, nullptr, 0, st));
  AttnArgs cross{ws.qkv, T, inner, 0, cross_kv, T_enc, d->n_kv, 2 * layer * inner, (2 * layer + 1) * inner, ws.attn,
                 inner, ws.cu_tokens, cu_enc, nullptr, B, max_len, c.num_heads, c.d_kv, 0};
  RPX_TRY(launch_t5_attention_mode(AttnMode::kCross, cross, st));
  RPX_TRY(oproj_gemm(false, T, ws.attn, w.co, D, inner, ws.h32, ws.h16, sa, st));
  RPX_TRY(ffn_up_gemm(false, T, ws.h16, w.wi, 2 * F, D, RowScale{sa, P, T, inv_d, c.ln_eps}, ws.ffn, st));
  RPX_TRY(ffn_down_gemm(false, T, ws.ffn, w.wo, D, F, ws.h32, ws.h16, sb, st));
  *ss_in = sb;
  *ss_other = sa;
  return RPX_OK;
}

// ---------------------------------------------------------------------------------------------- generate
// The search half over B states, nb beams, R = B nb rows.  Nothing here grows with the step: the KV cache holds
// every step's q | k | v rows in place, [num_layers][max_length][R][3 inner] bf16.

// The search's own state: what the init, step and finish kernels read and write besides the logits.
struct SearchBufs {
  int32_t* tokens;          // [max_length][R]
  int32_t* lin;             // [2][R][max_length]
  float* run_score;         // [R]
  float* fin_score;         // [2][R]
  int32_t* fin_len;         // [2][R]
  int32_t* fin_flag;        // [2][R]
  int32_t* fin_seq;         // [2][R][max_length]
  int32_t* state;           // [B][4]
  int32_t* counters;        // done count, out_len, last step
};

SearchBufs carve_search(Carver& c, int64_t B, int64_t R, int64_t ML) {
  SearchBufs s{};
  s.tokens = (int32_t*)c.take((size_t)ML * R * 4);
  s.lin = (int32_t*)c.take(2 * (size_t)R * ML * 4);
  s.run_score = (float*)c.take((size_t)R * 4);
  s.fin_score = (float*)c.take(2 * (size_t)R * 4);
  s.fin_len = (int32_t*)c.take(2 * (size_t)R * 4);
  s.fin_flag = (int32_t*)c.take(2 * (size_t)R * 4);
  s.fin_seq = (int32_t*)c.take(2 * (size_t)R * ML * 4);
  s.state = (int32_t*)c.take((size_t)B * 16);
  s.counters = (int32_t*)c.take(16);
  return s;
}

struct GenWs {
  size_t dec_off;
  __nv_bfloat16* cross_kv;  // the prefill's
  __nv_bfloat16* cache;
  float* logits;            // [R, vocab]
  SearchBufs s;
  size_t cache_layer;       // elements of one layer's cache
  size_t total;
};

GenWs carve_gen(const rpx_t5_decoder* d, const rpx_encoder* e, uint8_t* base, __nv_bfloat16* cross_kv, int64_t B,
                int64_t nb, int64_t ML) {
  GenWs w{};
  const int64_t R = B * nb;
  Carver c{base};
  w.dec_off = c.off;
  c.take(carve(e, nullptr, R, B).total);
  w.cross_kv = cross_kv;
  w.cache_layer = (size_t)ML * R * 3 * d->inner;
  w.cache = (__nv_bfloat16*)c.take(w.cache_layer * d->cfg.num_layers * 2);
  w.logits = (float*)c.take((size_t)R * d->cfg.vocab_size * 4);
  w.s = carve_search(c, B, R, ML);
  w.total = c.off;
  return w;
}

// The search's three launches, shared by search() and rpx_debug_search so that both run the same kernels with the
// same arguments.  A search over B states of nb beams (R = B nb rows; greedy: nb = 1, one state per row).
struct SearchShape {
  int B, nb, V, ML;
  int rows() const { return B * nb; }
  int states() const { return nb > 1 ? B : rows(); }  // greedy: one state per row
};

int search_init(const SearchBufs& s, const SearchShape& sh, int start_id, cudaStream_t st) {
  const int R = sh.rows(), nb = sh.nb;
  GenerateInitArgs ia{s.tokens, nb > 1 ? s.lin : nullptr, s.run_score, s.fin_score, s.fin_len, s.fin_flag, s.state,
                      s.counters, s.counters + 1, s.counters + 2, R, sh.states(), nb, sh.ML, start_id};
  return launch_generate_init(ia, st);
}

// Step t on logits [R, V]; the trace, if any, records it while t < trace->max_steps.
int search_step(const SearchBufs& s, const SearchShape& sh, const float* logits, double length_penalty, int eos_id,
                const rpx_generate_trace* trace, int t, cudaStream_t st) {
  const int R = sh.rows(), V = sh.V;
  const bool tr = trace && t < trace->max_steps;
  BeamStepArgs sa{logits, s.tokens, s.lin, s.run_score, s.fin_score, s.fin_len, s.fin_flag, s.fin_seq, s.state,
                  s.counters, s.counters + 2, tr ? trace->d_scores + (size_t)t * R * V : nullptr,
                  tr ? trace->d_parents + (size_t)t * R : nullptr, tr ? trace->d_tokens + (size_t)t * R : nullptr,
                  (float)pow((double)(t + 1), length_penalty), t, R, sh.nb, V, sh.ML, eos_id};
  return launch_search_step(sa, sh.states(), st);
}

int search_finish(const SearchBufs& s, const SearchShape& sh, int num_return, int start_id, int eos_id,
                  int64_t* d_sequences, float* d_scores, cudaStream_t st) {
  const int nb = sh.nb;
  GenerateFinishArgs fa{s.tokens, s.fin_score, s.fin_len, s.fin_seq, s.state, d_sequences, d_scores, s.counters + 1,
                        sh.rows(), nb, num_return, sh.ML, start_id, nb > 1 && start_id == 0 ? eos_id : start_id};
  return launch_generate_finish(fa, sh.states(), st);
}

// One decoder step for all R rows at position t: embed the rows' current tokens, every layer on the latency-path
// launchers (self-attention over the cache, cross-attention over the state's encoder tokens), then the head into
// fp32 logits [R, vocab].
int decode_step(const rpx_t5_decoder* d, const rpx_encoder* e, const GenWs& g, const Workspace& dw, const int32_t* cu_enc,
                int T_enc, int B, int nb, int ML, int t, cudaStream_t st) {
  const rpx_t5_config& c = d->cfg;
  const int R = B * nb, D = c.d_model, inner = d->inner, F = c.d_ff, P = e->n_parts_lat;
  const float inv_d = 1.0f / (float)D;
  RPX_TRY(launch_embed(g.s.tokens + (size_t)t * R, d->emb, dw.h32, dw.h16, dw.ssA, R, P, R, D, st));
  float* sa = dw.ssA;
  float* sb = dw.ssB;
  for (int l = 0; l < c.num_layers; ++l) {
    const DecLayerW& w = d->layers[l];
    __nv_bfloat16* cache = g.cache + g.cache_layer * l;
    RPX_TRY(qkv_gemm(true, R, dw.h16, w.qkv, 3 * inner, D, RowScale{sa, P, R, inv_d, c.ln_eps},
                     cache + (size_t)t * R * 3 * inner, nullptr, 0, st));
    DecodeAttnArgs da{cache, nb > 1 ? g.s.lin + (size_t)(t & 1) * R * ML : nullptr, d->bias_lut, dw.attn, g.s.state,
                      t, R, 3 * inner, inner, c.num_heads, ML, c.rel_max_distance, nb};
    RPX_TRY(launch_decode_attention(da, st));
    RPX_TRY(oproj_gemm(true, R, dw.attn, w.o, D, inner, dw.h32, dw.h16, sb, st));
    RPX_TRY(qkv_gemm(true, R, dw.h16, w.cq, inner, D, RowScale{sb, P, R, inv_d, c.ln_eps}, dw.qkv, nullptr, 0, st));
    AttnArgs cross{dw.qkv, R, inner, 0, g.cross_kv, T_enc, d->n_kv, 2 * l * inner, (2 * l + 1) * inner, dw.attn, inner,
                   dw.cu_tokens, cu_enc, nullptr, B, nb, c.num_heads, c.d_kv, 0};
    RPX_TRY(launch_t5_attention_mode(AttnMode::kCross, cross, st));
    RPX_TRY(oproj_gemm(true, R, dw.attn, w.co, D, inner, dw.h32, dw.h16, sa, st));
    RPX_TRY(ffn_up_gemm(true, R, dw.h16, w.wi, 2 * F, D, RowScale{sa, P, R, inv_d, c.ln_eps}, dw.ffn, st));
    RPX_TRY(ffn_down_gemm(true, R, dw.ffn, w.wo, D, F, dw.h32, dw.h16, sb, st));
    float* tmp = sa;
    sa = sb;
    sb = tmp;
  }
  return head_gemm(R, dw.h16, d->head, c.vocab_size, D, RowScale{sa, P, R, inv_d, c.ln_eps}, g.logits, st);
}

// Steps enqueued between two reads of the done-state count.
constexpr int kPollSteps = 8;
constexpr int kMaxBeams = 128;
constexpr size_t kMaxStepSmem = 227 * 1024 - 16 * 1024;  // the beam step's candidate keys, beside its static arrays

// ---------------------------------------------------------------------------------------------- the three stages
// rpx_seq2seq_forward, _generate and _evaluate are each a sequence of these: prefill, then the teacher-forced half, the
// search half, or both on the one prefill.

// What the prefill leaves for the halves.
struct Prefill {
  Workspace ew;  // the encoder's workspace for T_enc tokens: cu_tokens = the states' offsets, flag = the id-range flag
  int T_enc, max_enc;
  int T_dec, max_dec;  // with labels: the decoder tokens and the longest row; dec->h_cu[B + 1, 2B + 1] their offsets
};

// Argument checks of the teacher-forced half.
int check_seq_args(const char* fn, int batch, int in_len, int out_len, const float* d_logits) {
  RPX_REQUIRE(batch > 0 && in_len > 0 && out_len > 0, RPX_ERR_INVALID, "%s: batch=%d in_len=%d out_len=%d", fn, batch,
              in_len, out_len);
  RPX_REQUIRE(batch <= 65535, RPX_ERR_UNSUPPORTED, "%s: batch=%d exceeds the 65535 grid limit", fn, batch);
  RPX_REQUIRE((int64_t)batch * in_len < (int64_t)INT32_MAX && (int64_t)batch * out_len < (int64_t)INT32_MAX,
              RPX_ERR_UNSUPPORTED, "%s: batch too large", fn);
  RPX_REQUIRE(d_logits == nullptr || (reinterpret_cast<uintptr_t>(d_logits) & 15) == 0, RPX_ERR_INVALID,
              "%s: d_logits must be 16-byte aligned", fn);
  return RPX_OK;
}

// Argument checks of the search half.
int check_gen_args(const char* fn, int batch, int in_len, int num_beams, int num_return, int max_length, int eos_id,
                   const float* d_scores, int V) {
  RPX_REQUIRE(batch > 0 && in_len > 0, RPX_ERR_INVALID, "%s: batch=%d in_len=%d", fn, batch, in_len);
  RPX_REQUIRE(num_beams >= 1 && num_beams <= kMaxBeams, RPX_ERR_INVALID, "%s: num_beams=%d outside [1, %d]", fn,
              num_beams, kMaxBeams);
  RPX_REQUIRE(num_return >= 1 && num_return <= num_beams, RPX_ERR_INVALID,
              "%s: num_return=%d outside [1, num_beams=%d]", fn, num_return, num_beams);
  RPX_REQUIRE(num_beams == 1 || 2 * num_beams <= V, RPX_ERR_INVALID, "%s: 2 * num_beams=%d exceeds vocab_size=%d", fn,
              2 * num_beams, V);
  RPX_REQUIRE(num_beams == 1 || d_scores, RPX_ERR_INVALID, "%s: beam search needs d_scores", fn);
  RPX_REQUIRE(max_length >= 2, RPX_ERR_INVALID, "%s: max_length=%d must be at least 2", fn, max_length);
  RPX_REQUIRE(eos_id >= 0 && eos_id < V, RPX_ERR_INVALID, "%s: eos_id=%d outside [0, %d)", fn, eos_id, V);
  RPX_REQUIRE(num_beams == 1 || beam_step_smem_bytes(num_beams, V) <= kMaxStepSmem, RPX_ERR_UNSUPPORTED,
              "%s: num_beams * vocab_size=%d candidates exceed one CTA's shared memory", fn, num_beams * V);
  RPX_REQUIRE(batch <= 65535 && (int64_t)batch * in_len < (int64_t)INT32_MAX &&
                  (int64_t)batch * num_beams * max_length < (int64_t)INT32_MAX,
              RPX_ERR_UNSUPPORTED, "%s: batch too large", fn);
  return RPX_OK;
}

// The search step's shared-memory opt-in and the pinned words the search polls, once per decoder handle.
int init_search(rpx_t5_decoder* dec) {
  if (dec->h_poll) return RPX_OK;
  RPX_TRY(configure_search_step(kMaxStepSmem));
  RPX_CUDA_OK(cudaHostAlloc(reinterpret_cast<void**>(&dec->h_poll), 32, cudaHostAllocDefault));
  for (cudaEvent_t& ev : dec->poll_ev) RPX_CUDA_OK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  return RPX_OK;
}

// Stage 1, the prefill.  The states' mask lengths and, with labels, the labels' lengths (into lab_lens / lab_flag)
// are read back in one synchronisation, none without mask and labels.  Then the host offsets, the packed ids, the
// encoder stopped before its final RMSNorm, and the cross K / V of every decoder layer into pw.cross_kv, which is
// skipped only when there is no search and no decoder token.  Host offsets in dec->h_cu: [0, B] the states',
// [B + 1, 2B + 1] the decoder tokens' (with labels), [2B + 2, 3B + 2] left to the search.
int prefill(rpx_t5_decoder* dec, rpx_encoder* enc, const int64_t* d_input_ids, const int64_t* d_attention_mask, int B,
            int in_len, const int64_t* d_labels, int out_len, int32_t* lab_lens, int32_t* lab_flag, uint8_t* base,
            const PrefillWs& pw, bool search, Prefill* p, cudaStream_t st) {
  const rpx_t5_config& c = dec->cfg;
  const int D = c.d_model, V = c.vocab_size;
  const Workspace e_max = carve(enc, base + pw.enc_off, (int64_t)B * in_len, B);

  // ---- lengths: the state mask's and the labels', read back together
  RPX_CUDA_OK(cudaMemsetAsync(e_max.flag, 0, 4, st));
  auto& h = dec->h_lens;  // enc lens [B], enc flag, dec lens [B], dec flag
  h.assign(2 * (size_t)B + 2, in_len);
  h[B] = 0;
  h[2 * B + 1] = 0;
  if (d_attention_mask) {
    RPX_TRY(launch_mask_lengths(d_attention_mask, e_max.lens, e_max.flag, B, in_len, st));
    RPX_CUDA_OK(cudaMemcpyAsync(h.data(), e_max.lens, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
    RPX_CUDA_OK(cudaMemcpyAsync(&h[B], e_max.flag, 4, cudaMemcpyDeviceToHost, st));
  }
  if (d_labels) {
    RPX_CUDA_OK(cudaMemsetAsync(lab_flag, 0, 4, st));
    label_lengths_kernel<<<ceil_div(B, 8), 256, 0, st>>>(d_labels, lab_lens, lab_flag, B, out_len, V);
    RPX_CUDA_OK(cudaGetLastError());
    RPX_CUDA_OK(cudaMemcpyAsync(&h[B + 1], lab_lens, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
    RPX_CUDA_OK(cudaMemcpyAsync(&h[2 * B + 1], lab_flag, 4, cudaMemcpyDeviceToHost, st));
  }
  if (d_attention_mask || d_labels) RPX_CUDA_OK(cudaStreamSynchronize(st));
  RPX_REQUIRE(h[B] == 0, RPX_ERR_MASK,
              "attention_mask must be a right-padded prefix of ones with at least one token per row");
  RPX_REQUIRE(h[2 * B + 1] == 0, RPX_ERR_INVALID, "labels must be -100 or ids in [0, %d)", V);

  auto& cu = dec->h_cu;
  cu.assign(3 * (size_t)B + 3, 0);
  p->max_enc = p->max_dec = 0;
  for (int b = 0; b < B; ++b) {
    cu[b + 1] = cu[b] + h[b];
    p->max_enc = h[b] > p->max_enc ? h[b] : p->max_enc;
    if (d_labels) {
      cu[B + 2 + b] = cu[B + 1 + b] + h[B + 1 + b];
      p->max_dec = h[B + 1 + b] > p->max_dec ? h[B + 1 + b] : p->max_dec;
    }
  }
  p->T_enc = cu[B];
  p->T_dec = cu[2 * B + 1];
  p->ew = carve(enc, base + pw.enc_off, p->T_enc, B);
  const Workspace& ew = p->ew;
  // the host vectors stay untouched until the next call, which synchronises before reusing them
  RPX_CUDA_OK(cudaMemcpyAsync(ew.cu_tokens, cu.data(), ((size_t)B + 1) * 4, cudaMemcpyHostToDevice, st));
  RPX_TRY(launch_pack_ids(d_input_ids, ew.cu_tokens, ew.ids, B, in_len, p->T_enc, V, ew.flag, st));

  // ---- encoder, then the cross K / V of every decoder layer, once per state
  RPX_TRY(forward(enc, ew, p->T_enc, B, p->max_enc, OutKind::kResidual, 0, nullptr, 0, st));
  if (search || p->T_dec > 0) {
    PdlScope pdl_scope(p->T_enc <= kPdlMaxTokens && p->T_dec <= kPdlMaxTokens);
    RPX_TRY(qkv_gemm(false, p->T_enc, ew.h16, dec->cross_kv, dec->n_kv, D,
                     RowScale{ew.ssA, enc->n_parts, p->T_enc, 1.0f / (float)D, c.ln_eps}, pw.cross_kv, nullptr, 0,
                     st));
  }
  return RPX_OK;
}

// Stage 2, the teacher-forced half: `_shift_right(labels)` through the decoder layers, the head and log-softmax; the
// per-row sums and counts into d_seq_logprob / d_seq_count, the logits into d_logits unless it is null.
int teacher_forced(const rpx_t5_decoder* dec, const rpx_encoder* enc, const Prefill& p, const __nv_bfloat16* cross_kv,
                   uint8_t* base, const SeqWs& sw, const int64_t* d_labels, int B, int out_len, float* d_logits,
                   double* d_seq_logprob, int32_t* d_seq_count, cudaStream_t st) {
  const rpx_t5_config& c = dec->cfg;
  const int D = c.d_model, V = c.vocab_size, P = dec->n_parts;
  const int T_enc = p.T_enc, T_dec = p.T_dec;
  const Workspace dw = carve(enc, base + sw.dec_off, T_dec > 0 ? T_dec : 1, B);
  RPX_CUDA_OK(cudaMemcpyAsync(dw.cu_tokens, dec->h_cu.data() + B + 1, ((size_t)B + 1) * 4, cudaMemcpyHostToDevice, st));
  if (T_dec > 0) {
    pack_decoder_kernel<<<ceil_div(T_dec, 256), 256, 0, st>>>(d_labels, dw.cu_tokens, dw.ids, sw.targets, B, out_len,
                                                              T_dec, dec->start_id);
    RPX_CUDA_OK(cudaGetLastError());
    PdlScope pdl_scope(T_dec <= kPdlMaxTokens && T_enc <= kPdlMaxTokens);
    RPX_TRY(launch_embed(dw.ids, dec->emb, dw.h32, dw.h16, dw.ssA, T_dec, P, T_dec, D, st));
    float* ss_in = dw.ssA;
    float* ss_other = dw.ssB;
    for (int l = 0; l < c.num_layers; ++l)
      RPX_TRY(decoder_layer(dec, dec->layers[l], l, dw, T_dec, B, p.max_dec, cross_kv, T_enc, p.ew.cu_tokens, &ss_in,
                            &ss_other, st));
    // ---- head
    RPX_TRY(head_gemm(T_dec, dw.h16, dec->head, V, D, RowScale{ss_in, P, T_dec, 1.0f / (float)D, c.ln_eps}, sw.logits,
                      st));
    token_logprob_kernel<<<ceil_div(T_dec, 8), 256, 0, st>>>(sw.logits, sw.targets, sw.tok_lp, T_dec, V);
    RPX_CUDA_OK(cudaGetLastError());
  }
  seq_logprob_kernel<<<ceil_div(B, 128), 128, 0, st>>>(sw.tok_lp, sw.targets, dw.cu_tokens, d_seq_logprob, d_seq_count,
                                                       B);
  RPX_CUDA_OK(cudaGetLastError());
  if (d_logits) {
    const int64_t rows = (int64_t)B * out_len;
    scatter_logits_kernel<<<(unsigned)ceil_div64(rows, 8), 256, 0, st>>>(sw.logits, dw.cu_tokens, d_logits, rows,
                                                                         out_len, V);
    RPX_CUDA_OK(cudaGetLastError());
  }
  return RPX_OK;
}

// Stage 3, the search half: beam or greedy search over the prefill's cross K / V, the results into d_sequences /
// d_scores; then one synchronisation, after which dec->h_poll holds [2] out_len, [3] the encoder's id-range flag,
// [4] the step at which the last search ended.  init_search must have run.
int search(rpx_t5_decoder* dec, const rpx_encoder* enc, const Prefill& p, uint8_t* base, const GenWs& g, int B, int nb,
           int num_return, int ML, double length_penalty, int eos_id, int64_t* d_sequences, float* d_scores,
           const rpx_generate_trace* trace, cudaStream_t st) {
  const int R = B * nb;
  const SearchShape sh{B, nb, dec->cfg.vocab_size, ML};
  const Workspace dw = carve(enc, base + g.dec_off, R, B);
  int32_t* cu_beam = dec->h_cu.data() + 2 * B + 2;  // the beams' query offsets, b nb
  for (int b = 0; b <= B; ++b) cu_beam[b] = b * nb;
  RPX_CUDA_OK(cudaMemcpyAsync(dw.cu_tokens, cu_beam, ((size_t)B + 1) * 4, cudaMemcpyHostToDevice, st));
  RPX_TRY(search_init(g.s, sh, dec->start_id, st));

  // ---- the steps, enqueued in blocks; the done-state count of the block before is read while a block runs
  const int states = sh.states();
  int t = 0, blk = 0;
  {
    PdlScope pdl_scope(true);
    while (t <= ML - 2) {
      const int t_end = t + kPollSteps < ML - 1 ? t + kPollSteps : ML - 1;
      for (; t < t_end; ++t) {
        RPX_TRY(decode_step(dec, enc, g, dw, p.ew.cu_tokens, p.T_enc, B, nb, ML, t, st));
        RPX_TRY(search_step(g.s, sh, g.logits, length_penalty, eos_id, trace, t, st));
      }
      RPX_CUDA_OK(cudaMemcpyAsync(dec->h_poll + (blk & 1), g.s.counters, 4, cudaMemcpyDeviceToHost, st));
      RPX_CUDA_OK(cudaEventRecord(dec->poll_ev[blk & 1], st));
      if (blk > 0) {
        RPX_CUDA_OK(cudaEventSynchronize(dec->poll_ev[(blk - 1) & 1]));
        if (dec->h_poll[(blk - 1) & 1] == states) break;
      }
      ++blk;
    }
  }
  RPX_TRY(search_finish(g.s, sh, num_return, dec->start_id, eos_id, d_sequences, d_scores, st));
  RPX_CUDA_OK(cudaMemcpyAsync(dec->h_poll + 2, g.s.counters + 1, 4, cudaMemcpyDeviceToHost, st));
  RPX_CUDA_OK(cudaMemcpyAsync(dec->h_poll + 3, p.ew.flag, 4, cudaMemcpyDeviceToHost, st));
  RPX_CUDA_OK(cudaMemcpyAsync(dec->h_poll + 4, g.s.counters + 2, 4, cudaMemcpyDeviceToHost, st));
  RPX_CUDA_OK(cudaStreamSynchronize(st));
  return RPX_OK;
}

}  // namespace
}  // namespace rpx

using namespace rpx;

extern "C" {

size_t rpx_t5_decoder_packed_bytes(const rpx_t5_config* cfg) {
  if (validate_dec_cfg(cfg) != RPX_OK) return 0;
  return dec_packed_layout(*cfg).total;
}

int rpx_t5_decoder_create(const rpx_t5_config* cfg, const rpx_t5_decoder_weights* w, int32_t scale_decoder_outputs,
                          int32_t start_token_id, void* d_packed, size_t packed_bytes, void* stream,
                          rpx_t5_decoder** out) {
  RPX_TRY(validate_dec_cfg(cfg));
  RPX_REQUIRE(w && d_packed && out, RPX_ERR_INVALID, "rpx_t5_decoder_create: null argument");
  RPX_REQUIRE(w->d_shared && w->d_rel_bias && w->d_final_ln && w->d_enc_final_ln && w->d_head, RPX_ERR_INVALID,
              "rpx_t5_decoder_create: null weight");
  RPX_REQUIRE(start_token_id >= 0 && start_token_id < cfg->vocab_size, RPX_ERR_INVALID,
              "rpx_t5_decoder_create: start_token_id=%d outside the vocabulary", start_token_id);
  DeviceInfo dev;
  RPX_TRY(get_device_info(&dev));
  const DecPackedLayout L = dec_packed_layout(*cfg);
  RPX_REQUIRE(packed_bytes >= L.total, RPX_ERR_WORKSPACE, "packed buffer too small: %zu < %zu", packed_bytes, L.total);
  RPX_REQUIRE((reinterpret_cast<uintptr_t>(d_packed) & 255) == 0, RPX_ERR_INVALID, "packed buffer must be 256-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* base = static_cast<uint8_t*>(d_packed);
  const int D = cfg->d_model, inner = cfg->num_heads * cfg->d_kv, F = cfg->d_ff, V = cfg->vocab_size;

  rpx_t5_decoder* d = new (std::nothrow) rpx_t5_decoder();
  RPX_REQUIRE(d != nullptr, RPX_ERR_INVALID, "out of host memory");
  d->cfg = *cfg;
  d->inner = inner;
  d->n_parts = ss_parts(D, false);
  d->n_kv = cfg->num_layers * 2 * inner;
  d->start_id = start_token_id;
  auto fail = [&](int code) {
    delete d;
    return code;
  };
#define TRY_D(expr)                    \
  do {                                 \
    int _s = (expr);                   \
    if (_s != RPX_OK) return fail(_s); \
  } while (0)
#define CUDA_D(expr)                                                                         \
  do {                                                                                       \
    cudaError_t _c = (expr);                                                                 \
    if (_c != cudaSuccess) {                                                                 \
      set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_c)); \
      return fail(RPX_ERR_CUDA);                                                             \
    }                                                                                        \
  } while (0)

  CUDA_D(cudaMemcpyAsync(base + L.emb, w->d_shared, (size_t)V * D * 4, cudaMemcpyDeviceToDevice, st));
  d->emb = reinterpret_cast<const float*>(base + L.emb);
  TRY_D(build_bias_lut(w->d_rel_bias, cfg->num_heads, cfg->rel_buckets, cfg->rel_max_distance, false,
                       reinterpret_cast<int32_t*>(base + L.bucket_tmp), reinterpret_cast<float*>(base + L.bias_lut), st));
  d->bias_lut = reinterpret_cast<const float*>(base + L.bias_lut);

  // head rows: W_head[v, k] * final_ln[k] (* d_model ** -0.5)
  const float* head_scale = w->d_final_ln;
  if (scale_decoder_outputs) {
    float* hs = reinterpret_cast<float*>(base + L.head_scale);
    scale_vec_kernel<<<ceil_div(D, 256), 256, 0, st>>>(w->d_final_ln, (float)(1.0 / sqrt((double)D)), hs, D);
    CUDA_D(cudaGetLastError());
    head_scale = hs;
  }
  __nv_bfloat16* head = reinterpret_cast<__nv_bfloat16*>(base + L.head);
  TRY_D(launch_pack_weight(w->d_head, head_scale, head, V, D, 0, V, V, st));
  d->head = head;

  __nv_bfloat16* ckv = reinterpret_cast<__nv_bfloat16*>(base + L.cross_kv);
  d->cross_kv = ckv;
  d->layers.resize(cfg->num_layers);
  for (int l = 0; l < cfg->num_layers; ++l) {
    // cross K / V of layer l, encoder.final_layer_norm folded along K
    TRY_D(launch_pack_weight(w->h_ck[l], w->d_enc_final_ln, ckv, inner, D, 2 * l * inner, inner, inner, st));
    TRY_D(launch_pack_weight(w->h_cv[l], w->d_enc_final_ln, ckv, inner, D, (2 * l + 1) * inner, inner, inner, st));
    uint8_t* lb = base + L.layer0 + L.layer_stride * l;
    auto at = [&](size_t off) { return reinterpret_cast<__nv_bfloat16*>(lb + off); };
    TRY_D(launch_pack_weight(w->h_q[l], w->h_ln0[l], at(L.qkv), inner, D, 0, inner, inner, st));
    TRY_D(launch_pack_weight(w->h_k[l], w->h_ln0[l], at(L.qkv), inner, D, inner, inner, inner, st));
    TRY_D(launch_pack_weight(w->h_v[l], w->h_ln0[l], at(L.qkv), inner, D, 2 * inner, inner, inner, st));
    TRY_D(launch_pack_weight(w->h_o[l], nullptr, at(L.o), D, inner, 0, D, D, st));
    TRY_D(launch_pack_weight(w->h_cq[l], w->h_ln1[l], at(L.cq), inner, D, 0, inner, inner, st));
    TRY_D(launch_pack_weight(w->h_co[l], nullptr, at(L.co), D, inner, 0, D, D, st));
    TRY_D(launch_pack_weight(w->h_wi0[l], w->h_ln2[l], at(L.wi), F, D, 0, 128, 256, st));
    TRY_D(launch_pack_weight(w->h_wi1[l], w->h_ln2[l], at(L.wi), F, D, 128, 128, 256, st));
    TRY_D(launch_pack_weight(w->h_wo[l], nullptr, at(L.wo), D, F, 0, D, D, st));
    d->layers[l] = DecLayerW{at(L.qkv), at(L.o), at(L.cq), at(L.co), at(L.wi), at(L.wo)};
  }
  CUDA_D(cudaStreamSynchronize(st));
#undef TRY_D
#undef CUDA_D
  *out = d;
  return RPX_OK;
}

int rpx_t5_decoder_destroy(rpx_t5_decoder* dec) {
  if (!dec) return RPX_OK;
  if (dec->h_poll) cudaFreeHost(dec->h_poll);
  for (cudaEvent_t ev : dec->poll_ev)
    if (ev) cudaEventDestroy(ev);
  delete dec;
  return RPX_OK;
}

size_t rpx_seq2seq_workspace_bytes(const rpx_t5_decoder* dec, const rpx_encoder* enc, int32_t batch, int32_t in_len,
                                   int32_t out_len) {
  if (!dec || !enc || batch <= 0 || in_len <= 0 || out_len <= 0 || check_pair(dec, enc) != RPX_OK) return 0;
  return carve_prefill(dec, enc, nullptr, batch, in_len).total + carve_seq(dec, enc, nullptr, batch, out_len).total;
}

int rpx_seq2seq_forward(rpx_t5_decoder* dec, rpx_encoder* enc, const int64_t* d_input_ids,
                        const int64_t* d_attention_mask, int32_t batch, int32_t in_len, const int64_t* d_labels,
                        int32_t out_len, float* d_logits, double* d_seq_logprob, int32_t* d_seq_count,
                        void* d_workspace, size_t workspace_bytes, void* stream) {
  RPX_REQUIRE(dec && enc && d_input_ids && d_labels && d_seq_logprob && d_seq_count && d_workspace, RPX_ERR_INVALID,
              "rpx_seq2seq_forward: null argument");
  RPX_TRY(check_pair(dec, enc));
  RPX_TRY(check_seq_args("rpx_seq2seq_forward", batch, in_len, out_len, d_logits));
  RPX_REQUIRE((reinterpret_cast<uintptr_t>(d_workspace) & 255) == 0, RPX_ERR_INVALID, "workspace must be 256-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* base = static_cast<uint8_t*>(d_workspace);
  const PrefillWs pw = carve_prefill(dec, enc, base, batch, in_len);
  uint8_t* tail = base + pw.total;
  const SeqWs sw = carve_seq(dec, enc, tail, batch, out_len);
  RPX_REQUIRE(pw.total + sw.total <= workspace_bytes, RPX_ERR_WORKSPACE, "workspace too small: need %zu, have %zu",
              pw.total + sw.total, workspace_bytes);
  const Workspace d_max = carve(enc, tail + sw.dec_off, (int64_t)batch * out_len, batch);

  Prefill p;
  RPX_TRY(prefill(dec, enc, d_input_ids, d_attention_mask, batch, in_len, d_labels, out_len, d_max.lens, d_max.flag,
                  base, pw, false, &p, st));
  RPX_TRY(teacher_forced(dec, enc, p, pw.cross_kv, tail, sw, d_labels, batch, out_len, d_logits, d_seq_logprob,
                         d_seq_count, st));
  // ids outside [0, vocab) are reported after the fact (the forward ran with id 0 in their place)
  int32_t flag = 0;
  RPX_CUDA_OK(cudaMemcpyAsync(&flag, p.ew.flag, 4, cudaMemcpyDeviceToHost, st));
  RPX_CUDA_OK(cudaStreamSynchronize(st));
  RPX_REQUIRE((flag & 2) == 0, RPX_ERR_INVALID, "input_ids contains ids outside [0, %d)", dec->cfg.vocab_size);
  return RPX_OK;
}

size_t rpx_seq2seq_generate_workspace_bytes(const rpx_t5_decoder* dec, const rpx_encoder* enc, int32_t batch,
                                            int32_t in_len, int32_t num_beams, int32_t max_length) {
  if (!dec || !enc || batch <= 0 || in_len <= 0 || num_beams <= 0 || num_beams > kMaxBeams || max_length < 2 ||
      check_pair(dec, enc) != RPX_OK)
    return 0;
  return carve_prefill(dec, enc, nullptr, batch, in_len).total +
         carve_gen(dec, enc, nullptr, nullptr, batch, num_beams, max_length).total;
}

int rpx_seq2seq_generate(rpx_t5_decoder* dec, rpx_encoder* enc, const int64_t* d_input_ids,
                         const int64_t* d_attention_mask, int32_t batch, int32_t in_len, int32_t num_beams,
                         int32_t num_return, int32_t max_length, double length_penalty, int32_t eos_id,
                         int64_t* d_sequences, float* d_scores, int32_t* h_out_len, int32_t* h_steps,
                         const rpx_generate_trace* trace, void* d_workspace, size_t workspace_bytes, void* stream) {
  RPX_REQUIRE(dec && enc && d_input_ids && d_sequences && h_out_len && d_workspace, RPX_ERR_INVALID,
              "rpx_seq2seq_generate: null argument");
  RPX_TRY(check_pair(dec, enc));
  RPX_TRY(check_gen_args("rpx_seq2seq_generate", batch, in_len, num_beams, num_return, max_length, eos_id, d_scores,
                         dec->cfg.vocab_size));
  RPX_REQUIRE((reinterpret_cast<uintptr_t>(d_workspace) & 255) == 0, RPX_ERR_INVALID, "workspace must be 256-byte aligned");
  RPX_REQUIRE(!trace || (trace->d_scores && trace->d_parents && trace->d_tokens && trace->max_steps >= 0),
              RPX_ERR_INVALID, "rpx_seq2seq_generate: incomplete trace");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* base = static_cast<uint8_t*>(d_workspace);
  const PrefillWs pw = carve_prefill(dec, enc, base, batch, in_len);
  uint8_t* tail = base + pw.total;
  const GenWs g = carve_gen(dec, enc, tail, pw.cross_kv, batch, num_beams, max_length);
  RPX_REQUIRE(pw.total + g.total <= workspace_bytes, RPX_ERR_WORKSPACE, "workspace too small: need %zu, have %zu",
              pw.total + g.total, workspace_bytes);
  RPX_TRY(init_search(dec));

  Prefill p;
  RPX_TRY(prefill(dec, enc, d_input_ids, d_attention_mask, batch, in_len, nullptr, 0, nullptr, nullptr, base, pw, true,
                  &p, st));
  RPX_TRY(search(dec, enc, p, tail, g, batch, num_beams, num_return, max_length, length_penalty, eos_id, d_sequences,
                 d_scores, trace, st));
  // ids outside [0, vocab) are reported after the fact (the search ran with id 0 in their place)
  RPX_REQUIRE((dec->h_poll[3] & 2) == 0, RPX_ERR_INVALID, "input_ids contains ids outside [0, %d)", dec->cfg.vocab_size);
  *h_out_len = dec->h_poll[2];
  if (h_steps) *h_steps = dec->h_poll[4];
  return RPX_OK;
}

size_t rpx_seq2seq_evaluate_workspace_bytes(const rpx_t5_decoder* dec, const rpx_encoder* enc, int32_t batch,
                                            int32_t in_len, int32_t out_len, int32_t num_beams, int32_t max_length) {
  if (!dec || !enc || batch <= 0 || in_len <= 0 || out_len <= 0 || num_beams <= 0 || num_beams > kMaxBeams ||
      max_length < 2 || check_pair(dec, enc) != RPX_OK)
    return 0;
  const size_t seq = carve_seq(dec, enc, nullptr, batch, out_len).total;
  const size_t gen = carve_gen(dec, enc, nullptr, nullptr, batch, num_beams, max_length).total;
  return carve_prefill(dec, enc, nullptr, batch, in_len).total + (seq > gen ? seq : gen);
}

int rpx_seq2seq_evaluate(rpx_t5_decoder* dec, rpx_encoder* enc, const int64_t* d_input_ids,
                         const int64_t* d_attention_mask, int32_t batch, int32_t in_len, const int64_t* d_labels,
                         int32_t out_len, float* d_logits, double* d_seq_logprob, int32_t* d_seq_count,
                         int32_t num_beams, int32_t num_return, int32_t max_length, double length_penalty,
                         int32_t eos_id, int64_t* d_sequences, float* d_scores, int32_t* h_out_len, int32_t* h_steps,
                         void* d_workspace, size_t workspace_bytes, void* stream) {
  RPX_REQUIRE(dec && enc && d_input_ids && d_labels && d_seq_logprob && d_seq_count && d_sequences && h_out_len &&
                  d_workspace,
              RPX_ERR_INVALID, "rpx_seq2seq_evaluate: null argument");
  RPX_TRY(check_pair(dec, enc));
  RPX_TRY(check_seq_args("rpx_seq2seq_evaluate", batch, in_len, out_len, d_logits));
  RPX_TRY(check_gen_args("rpx_seq2seq_evaluate", batch, in_len, num_beams, num_return, max_length, eos_id, d_scores,
                         dec->cfg.vocab_size));
  RPX_REQUIRE((reinterpret_cast<uintptr_t>(d_workspace) & 255) == 0, RPX_ERR_INVALID, "workspace must be 256-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* base = static_cast<uint8_t*>(d_workspace);
  const PrefillWs pw = carve_prefill(dec, enc, base, batch, in_len);
  // the two halves share the regions after the prefill's: the search starts after the teacher-forced half's last
  // kernel on the same stream, and reads nothing of it
  uint8_t* tail = base + pw.total;
  const SeqWs sw = carve_seq(dec, enc, tail, batch, out_len);
  const GenWs g = carve_gen(dec, enc, tail, pw.cross_kv, batch, num_beams, max_length);
  const size_t need = pw.total + (sw.total > g.total ? sw.total : g.total);
  RPX_REQUIRE(need <= workspace_bytes, RPX_ERR_WORKSPACE, "workspace too small: need %zu, have %zu", need,
              workspace_bytes);
  const Workspace d_max = carve(enc, tail + sw.dec_off, (int64_t)batch * out_len, batch);
  RPX_TRY(init_search(dec));

  Prefill p;
  RPX_TRY(prefill(dec, enc, d_input_ids, d_attention_mask, batch, in_len, d_labels, out_len, d_max.lens, d_max.flag,
                  base, pw, true, &p, st));
  RPX_TRY(teacher_forced(dec, enc, p, pw.cross_kv, tail, sw, d_labels, batch, out_len, d_logits, d_seq_logprob,
                         d_seq_count, st));
  RPX_TRY(search(dec, enc, p, tail, g, batch, num_beams, num_return, max_length, length_penalty, eos_id, d_sequences,
                 d_scores, nullptr, st));
  // ids outside [0, vocab) are reported once, after both halves ran with id 0 in their place
  RPX_REQUIRE((dec->h_poll[3] & 2) == 0, RPX_ERR_INVALID, "input_ids contains ids outside [0, %d)", dec->cfg.vocab_size);
  *h_out_len = dec->h_poll[2];
  if (h_steps) *h_steps = dec->h_poll[4];
  return RPX_OK;
}

int rpx_debug_decode_attention(const void* d_cache, const int32_t* d_lin, const float* d_lut, void* d_out, int32_t t,
                               int32_t rows, int32_t max_length, int32_t n_heads, int32_t rel_max_distance,
                               void* stream) {
  RPX_REQUIRE(d_cache && d_lut && d_out, RPX_ERR_INVALID, "rpx_debug_decode_attention: null argument");
  RPX_REQUIRE(rows > 0 && n_heads > 0 && t >= 0 && t < max_length, RPX_ERR_INVALID,
              "rpx_debug_decode_attention: t=%d rows=%d max_length=%d n_heads=%d", t, rows, max_length, n_heads);
  RPX_REQUIRE(rows <= INT32_MAX / max_length, RPX_ERR_UNSUPPORTED, "rpx_debug_decode_attention: rows=%d too many", rows);
  RPX_REQUIRE(rel_max_distance > 0 && rel_max_distance <= 2048, RPX_ERR_INVALID,
              "rpx_debug_decode_attention: rel_max_distance=%d", rel_max_distance);
  const int inner = n_heads * 64;
  DecodeAttnArgs a{static_cast<const __nv_bfloat16*>(d_cache), d_lin, d_lut, static_cast<__nv_bfloat16*>(d_out), nullptr,
                   t, rows, 3 * inner, inner, n_heads, max_length, rel_max_distance, 1};
  return launch_decode_attention(a, static_cast<cudaStream_t>(stream));
}

size_t rpx_debug_search_workspace_bytes(int32_t batch, int32_t num_beams, int32_t max_length) {
  if (batch <= 0 || num_beams <= 0 || num_beams > kMaxBeams || max_length < 2) return 0;
  Carver c{nullptr};
  carve_search(c, batch, (int64_t)batch * num_beams, max_length);
  return c.off;
}

int rpx_debug_search(const float* d_logits, int32_t batch, int32_t num_beams, int32_t vocab, int32_t num_return,
                     int32_t max_length, double length_penalty, int32_t eos_id, int32_t start_id,
                     int64_t* d_sequences, float* d_scores, int32_t* h_out_len, int32_t* h_steps,
                     const rpx_generate_trace* trace, void* d_workspace, size_t workspace_bytes, void* stream) {
  RPX_REQUIRE(d_logits && d_sequences && h_out_len && d_workspace, RPX_ERR_INVALID, "rpx_debug_search: null argument");
  RPX_REQUIRE(vocab > 0, RPX_ERR_INVALID, "rpx_debug_search: vocab=%d", vocab);
  RPX_TRY(check_gen_args("rpx_debug_search", batch, 1, num_beams, num_return, max_length, eos_id, d_scores, vocab));
  RPX_REQUIRE(start_id >= 0 && start_id < vocab, RPX_ERR_INVALID, "rpx_debug_search: start_id=%d outside [0, %d)",
              start_id, vocab);
  RPX_REQUIRE((reinterpret_cast<uintptr_t>(d_workspace) & 255) == 0, RPX_ERR_INVALID, "workspace must be 256-byte aligned");
  RPX_REQUIRE(!trace || (trace->d_scores && trace->d_parents && trace->d_tokens && trace->max_steps >= 0),
              RPX_ERR_INVALID, "rpx_debug_search: incomplete trace");
  const int64_t R = (int64_t)batch * num_beams;
  Carver c{static_cast<uint8_t*>(d_workspace)};
  const SearchBufs s = carve_search(c, batch, R, max_length);
  RPX_REQUIRE(c.off <= workspace_bytes, RPX_ERR_WORKSPACE, "workspace too small: need %zu, have %zu", c.off,
              workspace_bytes);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RPX_TRY(configure_search_step(kMaxStepSmem));
  const SearchShape sh{batch, num_beams, vocab, max_length};
  RPX_TRY(search_init(s, sh, start_id, st));
  for (int t = 0; t < max_length - 1; ++t)
    RPX_TRY(search_step(s, sh, d_logits + (size_t)t * R * vocab, length_penalty, eos_id, trace, t, st));
  RPX_TRY(search_finish(s, sh, num_return, start_id, eos_id, d_sequences, d_scores, st));
  int32_t counters[3];
  RPX_CUDA_OK(cudaMemcpyAsync(counters, s.counters, sizeof counters, cudaMemcpyDeviceToHost, st));
  RPX_CUDA_OK(cudaStreamSynchronize(st));
  *h_out_len = counters[1];
  if (h_steps) *h_steps = counters[2];
  return RPX_OK;
}

int rpx_debug_attention_ex(int32_t mode, const void* d_q, const void* d_kv, void* d_out, const int32_t* d_cu_q,
                           const int32_t* d_cu_kv, const float* d_lut, int32_t n_q_tokens, int32_t n_kv_tokens,
                           int32_t n_seqs, int32_t max_len, int32_t n_heads, int32_t rel_max_distance, void* stream) {
  RPX_REQUIRE(mode >= RPX_ATTN_BIDIRECTIONAL && mode <= RPX_ATTN_CROSS, RPX_ERR_INVALID, "rpx_debug_attention_ex: mode=%d",
              mode);
  const bool cross = mode == RPX_ATTN_CROSS;
  RPX_REQUIRE(d_q && d_out && d_cu_q && (cross ? d_kv && d_cu_kv : d_lut != nullptr), RPX_ERR_INVALID,
              "rpx_debug_attention_ex: null argument");
  RPX_REQUIRE(n_q_tokens > 0 && max_len > 0 && n_heads > 0 && n_seqs > 0 && (!cross || n_kv_tokens > 0),
              RPX_ERR_INVALID, "rpx_debug_attention_ex: empty problem");
  RPX_REQUIRE(n_seqs <= 65535, RPX_ERR_UNSUPPORTED, "rpx_debug_attention_ex: n_seqs=%d exceeds the 65535 grid limit", n_seqs);
  RPX_REQUIRE(cross || (rel_max_distance > 0 && rel_max_distance <= 2048), RPX_ERR_INVALID,
              "rpx_debug_attention_ex: rel_max_distance=%d", rel_max_distance);
  const int inner = n_heads * 64;
  const auto* q = static_cast<const __nv_bfloat16*>(d_q);
  AttnArgs a = cross ? AttnArgs{q, n_q_tokens, inner, 0, static_cast<const __nv_bfloat16*>(d_kv), n_kv_tokens, 2 * inner,
                                0, inner, static_cast<__nv_bfloat16*>(d_out), inner, d_cu_q, d_cu_kv, nullptr, n_seqs,
                                max_len, n_heads, 64, 0}
                     : AttnArgs{q, n_q_tokens, 3 * inner, 0, q, n_q_tokens, 3 * inner, inner, 2 * inner,
                                static_cast<__nv_bfloat16*>(d_out), inner, d_cu_q, d_cu_q, d_lut, n_seqs, max_len,
                                n_heads, 64, rel_max_distance};
  PdlScope pdl_scope(n_q_tokens <= kPdlMaxTokens);
  return launch_t5_attention_mode(static_cast<AttnMode>(mode), a, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
