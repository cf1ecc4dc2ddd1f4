// rpx_generate.cu — the two kernels generation adds to the decoder (rpx_decoder.cu runs them):
//
//   decode attention  one new query per (row, head) against the row's own keys p = 0..t, read from the KV cache
//                     through the lineage table: cache row p * R + lin[r][p] holds position p of row r's hypothesis
//   search step       one CTA per state: HF 5.5 `GenerationMixin._beam_search` (early_stopping=False) for one step,
//                     or greedy `_sample` when num_beams == 1
//
// Every K/V row is written once, at the step that produced it (the QKV GEMM writes straight into the cache), and is
// never moved: where HF reorders its cache by `beam_idx` every step, the search step gathers `lin` rows by parent.
#include <math.h>

#include "rpx_common.cuh"
#include "rpx_kernels.cuh"
#include "rpx_topk_common.cuh"

namespace rpx {
namespace {

constexpr int kDecAttnWarps = 4;
constexpr int kStepThreads = 1024;
constexpr float kMask = -1.0e9f;  // HF's "cannot be chosen" offset

// grid (R, heads), 4 warps.  Warp w takes the 32-key chunks w, w + 4, ...: lane j scores key 32 c + j (its k row
// loaded whole), then the warp folds the chunk into its own online softmax, lanes owning two of the 64 dims for the
// value sum.  The four warps are combined in warp order, so a row's result depends on t alone, not on R or on the
// other rows.
__global__ void __launch_bounds__(32 * kDecAttnWarps) decode_attention_kernel(DecodeAttnArgs a) {
  const int r = blockIdx.x, h = blockIdx.y;
  if (a.state_done && a.state_done[4 * (r / a.beams)] != 0) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t = a.t;
  __shared__ float q_s[64];
  __shared__ float m_s[kDecAttnWarps], l_s[kDecAttnWarps];
  __shared__ float acc_s[kDecAttnWarps][64];
  const __nv_bfloat16* q = a.cache + ((size_t)t * a.rows + r) * a.ld + h * 64;
  if (threadIdx.x < 64) q_s[threadIdx.x] = __bfloat162float(q[threadIdx.x]);
  __syncthreads();
  const int32_t* lin = a.lin ? a.lin + (size_t)r * a.max_length : nullptr;
  const float* lut = a.lut + (size_t)h * (2 * a.max_distance + 1) + a.max_distance;
  const size_t k_off = (size_t)a.inner + h * 64, v_off = 2 * (size_t)a.inner + h * 64 + 2 * lane;
  float m = -INFINITY, l = 0.f, acc0 = 0.f, acc1 = 0.f;
  for (int c = warp; 32 * c <= t; c += kDecAttnWarps) {
    const int p = 32 * c + lane;
    const bool valid = p <= t;
    int slot = r;
    float s = -INFINITY;
    if (valid) {
      if (lin) slot = lin[p];
      const uint4* k = reinterpret_cast<const uint4*>(a.cache + ((size_t)p * a.rows + slot) * a.ld + k_off);
      float dot = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const uint4 u = k[i];
        const uint32_t w4[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w4[j]));
          dot = fmaf(q_s[8 * i + 2 * j], f.x, dot);
          dot = fmaf(q_s[8 * i + 2 * j + 1], f.y, dot);
        }
      }
      const int delta = max(p - t, -a.max_distance);
      s = dot + lut[delta];
    }
    float cmax = s;
    for (int off = 16; off; off >>= 1) cmax = fmaxf(cmax, __shfl_xor_sync(kFullMask, cmax, off));
    const float m_new = fmaxf(m, cmax);
    const float scale = expf(m - m_new);
    const float pj = valid ? expf(s - m_new) : 0.f;
    float psum = pj;
    for (int off = 16; off; off >>= 1) psum += __shfl_xor_sync(kFullMask, psum, off);
    l = l * scale + psum;
    acc0 *= scale;
    acc1 *= scale;
    const int n_valid = min(32, t - 32 * c + 1);
    for (int j = 0; j < n_valid; ++j) {
      const float pk = __shfl_sync(kFullMask, pj, j);
      const int sl = __shfl_sync(kFullMask, slot, j);
      const float2 v = __bfloat1622float2(
          *reinterpret_cast<const __nv_bfloat162*>(a.cache + ((size_t)(32 * c + j) * a.rows + sl) * a.ld + v_off));
      acc0 = fmaf(pk, v.x, acc0);
      acc1 = fmaf(pk, v.y, acc1);
    }
    m = m_new;
  }
  if (lane == 0) {
    m_s[warp] = m;
    l_s[warp] = l;
  }
  acc_s[warp][2 * lane] = acc0;
  acc_s[warp][2 * lane + 1] = acc1;
  __syncthreads();
  if (threadIdx.x < 64) {
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < kDecAttnWarps; ++w) M = fmaxf(M, m_s[w]);
    float L = 0.f, o = 0.f;
#pragma unroll
    for (int w = 0; w < kDecAttnWarps; ++w) {
      if (l_s[w] == 0.f) continue;  // a warp that had no key
      const float e = expf(m_s[w] - M);
      L += l_s[w] * e;
      o += acc_s[w][threadIdx.x] * e;
    }
    a.out[(size_t)r * a.inner + h * 64 + threadIdx.x] = __float2bfloat16(o / L);
  }
}

// ---------------------------------------------------------------------------------------------- search step
// Block-wide exclusive prefix sum of one int per thread (kStepThreads threads); returns the total in *total.
__device__ int block_exclusive_scan(int v, int* warp_tot, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
  for (int off = 1; off < 32; off <<= 1) {
    const int y = __shfl_up_sync(kFullMask, x, off);
    if (lane >= off) x += y;
  }
  if (lane == 31) warp_tot[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int w = lane < (kStepThreads >> 5) ? warp_tot[lane] : 0;
    for (int off = 1; off < 32; off <<= 1) {
      const int y = __shfl_up_sync(kFullMask, w, off);
      if (lane >= off) w += y;
    }
    warp_tot[lane] = w;  // inclusive
  }
  __syncthreads();
  const int before = (warp ? warp_tot[warp - 1] : 0) + x - v;
  if (threadIdx.x == kStepThreads - 1) *total = before + v;
  __syncthreads();
  return before;
}

// One CTA per state over its [nb, V] logits.  Restates, for early_stopping=False and one EOS id:
//   log_softmax (fp32 result; max in fp32, sum of exp in fp64), + running scores            HF _beam_search
//   top 2 nb of nb V by (score desc, flat index asc), parent = i / V, token = i % V          _get_top_k_continuations
//   hits = token == eos or cur_len + 1 >= max_length                                         stopping criteria
//   running = top nb of (score + hits * -1e9)                                                _get_running_beams_...
//   candidates c < nb that hit: score / pen, + -1e9 unless the heuristic is unsatisfied, + -1e9 unless the
//   candidate finished; merged with the nb finished hypotheses, top nb kept                  _update_finished_beams
//   heuristic: running[0] / pen > the worst finished (or -1e9 while a slot is open)          _check_early_stop_heuristic
// with cur_len = t + 1 and pen = (t + 1) ** length_penalty, the same for the update and the heuristic.  Every
// selection ranks (score desc, position asc).  Then writes the running beams' next tokens, their lineage rows (the
// parent's lin row, plus position t + 1 in the row's own slot) and the finished hypotheses (double-buffered per
// state).  A state whose search is done returns at once: its finished hypotheses can no longer change.
__global__ void __launch_bounds__(kStepThreads) beam_step_kernel(BeamStepArgs a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  const int b = blockIdx.x;
  int32_t* st = a.state + 4 * b;  // done, unsat, parity, -
  if (st[0] != 0) return;
  const int nb = a.beams, V = a.vocab, N = nb * V, K = 2 * nb, t = a.t, ML = a.max_length;
  const int row0 = b * nb;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint32_t* keys = reinterpret_cast<uint32_t*>(smem_raw);  // [N]
  __shared__ int hist[256];
  __shared__ int warp_tot[32];
  __shared__ int s_total, s_count_gt, s_prefix_digit, s_kk;
  __shared__ uint64_t cand_key[256];
  __shared__ float cand_run[256], cand_fin[256];
  __shared__ int cand_rank[256];
  __shared__ float run_sc[128];
  __shared__ float fin_sc_old[128];
  __shared__ int merged_src[128];  // new finished slot k <- old slot (< nb) or candidate nb + c
  __shared__ int run_parent[128];
  __shared__ int s_unsat, s_par;

  if (tid < nb) run_sc[tid] = a.run_score[row0 + tid];
  if (tid == 0) {
    s_unsat = st[1];
    s_par = st[2];
  }
  __syncthreads();
  const int par = s_par;
  const float* fin_score_old = a.fin_score + (size_t)par * a.rows + row0;
  if (tid < nb) fin_sc_old[tid] = fin_score_old[tid];

  // 1. log_softmax per beam, + running score, as ordered keys
  for (int i = warp; i < nb; i += kStepThreads / 32) {
    const float* x = a.logits + (size_t)(row0 + i) * V;
    float mx = -INFINITY;
    for (int j = lane; j < V; j += 32) mx = fmaxf(mx, x[j]);
    for (int off = 16; off; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(kFullMask, mx, off));
    double s = 0.0;
    for (int j = lane; j < V; j += 32) s += exp((double)x[j] - (double)mx);
    for (int off = 16; off; off >>= 1) s += __shfl_xor_sync(kFullMask, s, off);
    const double ls = log(s);
    const float rs = run_sc[i];
    float* tr = a.trace_scores ? a.trace_scores + (size_t)(row0 + i) * V : nullptr;
    for (int j = lane; j < V; j += 32) {
      const float lp = (float)(((double)x[j] - (double)mx) - ls);
      if (tr) tr[j] = lp;
      keys[i * V + j] = fkey(__float_as_uint(lp + rs));
    }
  }
  if (tid == 0) {
    s_count_gt = 0;
    s_prefix_digit = 0;
    s_kk = K;
  }
  __syncthreads();

  // 2. radix select of the K-th largest key, 8 bits at a time
  uint32_t prefix = 0, pmask = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += kStepThreads) hist[i] = 0;
    __syncthreads();
    for (int i = tid; i < N; i += kStepThreads) {
      const uint32_t k = keys[i];
      if ((k & pmask) == prefix) atomicAdd(&hist[(k >> shift) & 255], 1);
    }
    __syncthreads();
    if (tid == 0) {
      int kk = s_kk, cum = 0, d = 255;
      for (; d > 0; --d) {
        if (cum + hist[d] >= kk) break;
        cum += hist[d];
      }
      s_kk = kk - cum;
      s_prefix_digit = d;
    }
    __syncthreads();
    prefix |= (uint32_t)s_prefix_digit << shift;
    pmask |= 255u << shift;
    __syncthreads();
  }
  const uint32_t thr = prefix;
  const int kk_eq = s_kk;  // how many keys equal to thr are taken: those of the lowest flat indices
  // 3. collect: every key above thr, then the kk_eq lowest indices equal to it
  for (int i = tid; i < N; i += kStepThreads) {
    const uint32_t k = keys[i];
    if (k > thr) {
      const int pos = atomicAdd(&s_count_gt, 1);
      cand_key[pos] = ((uint64_t)k << 32) | (uint64_t)(0xFFFFFFFFu - (uint32_t)i);
    }
  }
  const int per = (N + kStepThreads - 1) / kStepThreads;
  const int lo = min(N, tid * per), hi = min(N, lo + per);
  int n_eq = 0;
  for (int i = lo; i < hi; ++i) n_eq += keys[i] == thr;
  const int before = block_exclusive_scan(n_eq, warp_tot, &s_total);
  const int n_gt = K - kk_eq;
  if (before < kk_eq) {
    int pos = before;
    for (int i = lo; i < hi && pos < kk_eq; ++i)
      if (keys[i] == thr) cand_key[n_gt + pos++] = ((uint64_t)thr << 32) | (uint64_t)(0xFFFFFFFFu - (uint32_t)i);
  }
  __syncthreads();
  // rank the K candidates: (score desc, index asc) is key order
  if (tid < K) {
    const uint64_t me = cand_key[tid];
    int rank = 0;
    for (int j = 0; j < K; ++j) rank += cand_key[j] > me;
    cand_rank[tid] = rank;
  }
  __syncthreads();
  uint64_t my_key = 0;
  if (tid < K) my_key = cand_key[tid];
  __syncthreads();
  if (tid < K) cand_key[cand_rank[tid]] = my_key;  // sorted
  __syncthreads();

  // 4. per candidate c (rank order): hits, running value, finished value
  const bool at_max = t + 2 >= ML;
  if (tid < K) {
    const uint64_t key = cand_key[tid];
    const int idx = (int)(0xFFFFFFFFu - (uint32_t)(key & 0xFFFFFFFFull));
    const float s = __uint_as_float(unkey((uint32_t)(key >> 32)));
    const int token = idx % V;
    const bool hits = token == a.eos || at_max;
    cand_run[tid] = hits ? s + kMask : s;
    float f = s / a.penalty;
    if (!s_unsat) f = f + kMask;
    const bool did = hits && tid < nb;
    if (!did) f = f + kMask;
    cand_fin[tid] = f;
  }
  __syncthreads();
  // running: top nb of cand_run by (value desc, position asc)
  if (tid < K) {
    const float v = cand_run[tid];
    int rank = 0;
    for (int j = 0; j < K; ++j) {
      const float w = cand_run[j];
      rank += (w > v) || (w == v && j < tid);
    }
    if (rank < nb) {
      const uint64_t key = cand_key[tid];
      const int idx = (int)(0xFFFFFFFFu - (uint32_t)(key & 0xFFFFFFFFull));
      run_sc[rank] = v;
      run_parent[rank] = idx / V;
      const int row = row0 + rank;
      a.tokens[(size_t)(t + 1) * a.rows + row] = idx % V;
      a.run_score[row] = v;
      if (a.trace_parents) {
        a.trace_parents[row] = row0 + idx / V;
        a.trace_tokens[row] = idx % V;
      }
    }
  }
  // finished: top nb of [old finished (positions 0..nb), candidates (nb..nb + K)]
  const int M = nb + K;
  if (tid < M) {
    const float v = tid < nb ? fin_sc_old[tid] : cand_fin[tid - nb];
    int rank = 0;
    for (int j = 0; j < M; ++j) {
      const float w = j < nb ? fin_sc_old[j] : cand_fin[j - nb];
      rank += (w > v) || (w == v && j < tid);
    }
    if (rank < nb) merged_src[rank] = tid;
  }
  __syncthreads();

  // 5. lineage rows of the new running beams: the parent's positions 0..t, then position t + 1 in its own slot
  const int32_t* lin_old = a.lin + (size_t)(t & 1) * a.rows * ML;
  int32_t* lin_new = a.lin + (size_t)((t + 1) & 1) * a.rows * ML;
  const int w_rows = nb * (t + 2);
  for (int i = tid; i < w_rows; i += kStepThreads) {
    const int r = i / (t + 2), p = i % (t + 2);
    lin_new[(size_t)(row0 + r) * ML + p] = p <= t ? lin_old[(size_t)(row0 + run_parent[r]) * ML + p] : row0 + r;
  }
  // 6. finished hypotheses into the other buffer: generated tokens (positions 1..len), length, score, flag
  const int npar = par ^ 1;
  const size_t fo = (size_t)par * a.rows, fn = (size_t)npar * a.rows;
  for (int k = warp; k < nb; k += kStepThreads / 32) {
    const int src = merged_src[k];
    int32_t* dst = a.fin_seq + (fn + row0 + k) * ML;
    if (src < nb) {
      const int len = a.fin_len[fo + row0 + src];
      const int32_t* s = a.fin_seq + (fo + row0 + src) * ML;
      for (int p = lane; p < len; p += 32) dst[p] = s[p];
      if (lane == 0) {
        a.fin_len[fn + row0 + k] = len;
        a.fin_score[fn + row0 + k] = fin_sc_old[src];
        a.fin_flag[fn + row0 + k] = a.fin_flag[fo + row0 + src];
      }
    } else {
      const int c = src - nb;
      const uint64_t key = cand_key[c];
      const int idx = (int)(0xFFFFFFFFu - (uint32_t)(key & 0xFFFFFFFFull));
      const int parent = row0 + idx / V;
      for (int p = 1 + lane; p <= t; p += 32) dst[p - 1] = a.tokens[(size_t)p * a.rows + lin_old[(size_t)parent * ML + p]];
      if (lane == 0) {
        dst[t] = idx % V;
        a.fin_len[fn + row0 + k] = t + 1;
        a.fin_score[fn + row0 + k] = cand_fin[c];
        a.fin_flag[fn + row0 + k] = (c < nb) && (idx % V == a.eos || at_max);
      }
    }
  }
  __syncthreads();
  // 7. the early-stop heuristic and the state's done bit
  if (tid == 0) {
    const float best = run_sc[0] / a.penalty;
    float worst = INFINITY;
    for (int k = 0; k < nb; ++k) worst = fminf(worst, a.fin_score[fn + row0 + k]);
    bool improve = false;
    for (int k = 0; k < nb; ++k) improve |= best > (a.fin_flag[fn + row0 + k] ? worst : kMask);
    const int unsat = s_unsat && improve;
    st[1] = unsat;
    st[2] = npar;
    if (!unsat || at_max) {
      st[0] = 1;
      atomicAdd(a.done_count, 1);
      atomicMax(a.last_step, t + 1);
    }
  }
}

// (v, j) comes before (best, arg) in torch.argmax's order: a NaN above every number (the first NaN wins), then the
// larger value, then the lower id.
__device__ __forceinline__ bool argmax_before(float v, int j, float best, int arg) {
  if (isnan(v)) return !isnan(best) || j < arg;
  return v > best || (v == best && j < arg);
}

// num_beams == 1 (HF greedy `_sample`): one CTA per row, torch.argmax of the fp32 logits (the lowest id of the
// maximum; the first NaN if the row holds one); the row is done at EOS or max_length, and its later tokens are the
// pad id (the finishing kernel writes them).
__global__ void __launch_bounds__(256) greedy_step_kernel(BeamStepArgs a) {
  const int r = blockIdx.x;
  int32_t* st = a.state + 4 * r;
  if (st[0] != 0) return;
  const float* x = a.logits + (size_t)r * a.vocab;
  float best = -INFINITY;
  int arg = 0x7fffffff;  // any id of the row comes before it, -inf included
  for (int j = threadIdx.x; j < a.vocab; j += blockDim.x) {
    const float v = x[j];
    if (a.trace_scores) a.trace_scores[(size_t)r * a.vocab + j] = v;
    if (argmax_before(v, j, best, arg)) {
      best = v;
      arg = j;
    }
  }
  __shared__ float bv[8];
  __shared__ int bi[8];
  for (int off = 16; off; off >>= 1) {
    const float ov = __shfl_xor_sync(kFullMask, best, off);
    const int oi = __shfl_xor_sync(kFullMask, arg, off);
    if (argmax_before(ov, oi, best, arg)) {
      best = ov;
      arg = oi;
    }
  }
  if ((threadIdx.x & 31) == 0) {
    bv[threadIdx.x >> 5] = best;
    bi[threadIdx.x >> 5] = arg;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
      if (argmax_before(bv[w], bi[w], best, arg)) {
        best = bv[w];
        arg = bi[w];
      }
    a.tokens[(size_t)(a.t + 1) * a.rows + r] = arg;
    a.fin_len[r] = a.t + 1;
    if (a.trace_parents) {
      a.trace_parents[r] = r;
      a.trace_tokens[r] = arg;
    }
    if (arg == a.eos || a.t + 2 >= a.max_length) {
      st[0] = 1;
      atomicAdd(a.done_count, 1);
      atomicMax(a.last_step, a.t + 1);
    }
  }
}

__global__ void generate_init_kernel(GenerateInitArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int rows = a.rows;
  if (i < rows * a.max_length) a.tokens[i] = a.start_id;
  if (i < rows) {
    if (a.lin) a.lin[(size_t)i * a.max_length] = i;
    if (a.run_score) a.run_score[i] = (i % a.beams) == 0 ? 0.f : kMask;
    if (a.fin_score) a.fin_score[i] = kMask;  // parity 0
    a.fin_len[i] = 0;
    if (a.fin_flag) a.fin_flag[i] = 0;
  }
  if (i < a.states) {
    a.state[4 * i] = 0;
    a.state[4 * i + 1] = 1;
    a.state[4 * i + 2] = 0;
    a.state[4 * i + 3] = 0;
  }
  if (i == 0) {
    *a.done_count = 0;
    *a.out_len = 0;
    *a.last_step = 0;
  }
}

// One CTA per state: the first n_ret finished hypotheses (beam) or the row (greedy) as [start, tokens..., fill...]
// rows of width max_length, the scores, and the longest returned length + 1 (atomicMax into out_len).
__global__ void generate_finish_kernel(GenerateFinishArgs a) {
  const int b = blockIdx.x;
  const int ML = a.max_length;
  if (a.beams == 1) {
    const int len = a.fin_len[b];
    int64_t* dst = a.sequences + (size_t)b * ML;
    for (int p = threadIdx.x; p < ML; p += blockDim.x)
      dst[p] = p == 0 ? a.start_id : (p <= len ? a.tokens[(size_t)p * a.rows + b] : a.fill_id);
    if (threadIdx.x == 0) atomicMax(a.out_len, 1 + len);
    return;
  }
  const int par = a.state[4 * b + 2];
  for (int j = 0; j < a.n_ret; ++j) {
    const size_t slot = (size_t)par * a.rows + (size_t)b * a.beams + j;
    const int len = a.fin_len[slot];
    const int32_t* src = a.fin_seq + slot * ML;
    int64_t* dst = a.sequences + ((size_t)b * a.n_ret + j) * ML;
    for (int p = threadIdx.x; p < ML; p += blockDim.x) dst[p] = p == 0 ? a.start_id : (p <= len ? src[p - 1] : a.fill_id);
    if (threadIdx.x == 0) {
      a.scores[(size_t)b * a.n_ret + j] = a.fin_score[slot];
      atomicMax(a.out_len, 1 + len);
    }
  }
}

}  // namespace

int launch_decode_attention(const DecodeAttnArgs& a, cudaStream_t st) {
  decode_attention_kernel<<<dim3(a.rows, a.n_heads), 32 * kDecAttnWarps, 0, st>>>(a);
  RPX_CUDA_OK(cudaGetLastError());
  return RPX_OK;
}

size_t beam_step_smem_bytes(int beams, int vocab) { return (size_t)beams * vocab * 4; }

int configure_search_step(size_t max_smem) {
  RPX_CUDA_OK(cudaFuncSetAttribute(beam_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)max_smem));
  return RPX_OK;
}

int launch_search_step(const BeamStepArgs& a, int states, cudaStream_t st) {
  if (a.beams == 1) {
    greedy_step_kernel<<<states, 256, 0, st>>>(a);
  } else {
    beam_step_kernel<<<states, kStepThreads, beam_step_smem_bytes(a.beams, a.vocab), st>>>(a);
  }
  RPX_CUDA_OK(cudaGetLastError());
  return RPX_OK;
}

int launch_generate_init(const GenerateInitArgs& a, cudaStream_t st) {
  const int n = a.rows * a.max_length;
  generate_init_kernel<<<ceil_div(n, 256), 256, 0, st>>>(a);
  RPX_CUDA_OK(cudaGetLastError());
  return RPX_OK;
}

int launch_generate_finish(const GenerateFinishArgs& a, int states, cudaStream_t st) {
  generate_finish_kernel<<<states, 256, 0, st>>>(a);
  RPX_CUDA_OK(cudaGetLastError());
  return RPX_OK;
}

}  // namespace rpx
