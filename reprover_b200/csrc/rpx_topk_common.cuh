// rpx_topk_common.cuh — what the top-k kernels share (rpx_simtopk.cu: tensor-core path, rpx_smallq.cu:
// HBM-streaming path for 1-2 queries, rpx_exact.cu: exact fp64 fallback, rpx_bm25.cu: BM25 tiles) and their
// host-side entry points: the device-resident state of an index handle, the result writer, the key selection
// and the ranking every kernel ends with, and the exactness guard.
//
// Ordering contract (include/rpx.h): score descending, then index ascending, where score is the
// canonical fp64 dot product of the bf16 operands (dot64_canonical == oracle/rpx_oracle.c::
// rpx_oracle_dot64).  The fast paths rank by an fp32 score first; the EXACTNESS GUARD below decides
// whether that ranking can have missed a member of the true top-k and, if so, hands the query to the
// exact path.  Replaces common.py:307-308 (`Q @ E.T`, argsort) of the reference.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>

namespace rpx {

constexpr unsigned kFullMask = 0xffffffffu;

// Device-resident part of an index handle (rpx_index): zeroed by rpx_index_create, every kernel leaves
// the counters it used at zero again, so no per-call memset is needed.
struct IndexState {
  float norm2_max;          // upper bound of max_i sum_j E[i,j]^2 (fp32, rounded up)
  uint32_t ticket;          // small-Q kernel: CTAs finished (last one runs the final stage)
  uint32_t n_flagged;       // queries handed to the exact path by the guard of the current call
  uint32_t fb_count;        // exact path: candidates appended for the query in flight
  uint32_t bar_count;       // exact path: grid barrier
  uint32_t bar_gen;
  uint32_t max_err_bits;    // diagnostics: max |fp32 score - fp64 score| seen by a guard (float bits)
  uint32_t n_exact_total;   // diagnostics: queries that went through the exact path since creation
  uint32_t max_eps_bits;    // diagnostics: largest guard epsilon used (float bits)
  uint32_t pad[7];
};
static_assert(sizeof(IndexState) == 64, "IndexState layout");

// Per-query record the guard leaves for the exact path: the k-th best entry found so far.  Every member
// of the true top-k ranks at or before it, so the exact pass only has to look at rows that do.
struct ExactBound {
  double score;   // -inf: no bound (fewer than k candidates were re-scored)
  int64_t idx;    // local row index of that entry
};

// Monotone map float bits -> uint32 (a > b  <=>  fkey(a) > fkey(b), -0 < +0).
__device__ __forceinline__ uint32_t fkey(uint32_t u) { return u ^ ((u >> 31) ? 0xFFFFFFFFu : 0x80000000u); }
__device__ __forceinline__ uint32_t unkey(uint32_t k) { return (k & 0x80000000u) ? (k ^ 0x80000000u) : ~k; }
// Same for doubles.
__device__ __forceinline__ uint64_t dkey(double v) {
  const uint64_t u = (uint64_t)__double_as_longlong(v);
  return u ^ ((u >> 63) ? ~0ull : 0x8000000000000000ull);
}
__device__ __forceinline__ double undkey(uint64_t k) {
  const uint64_t u = (k & 0x8000000000000000ull) ? (k ^ 0x8000000000000000ull) : ~k;
  return __longlong_as_double((long long)u);
}
// Composite 64-bit key of an (fp32 score bits, row index) pair: larger key == better under
// (score desc, index asc).  Distinct rows have distinct keys; key 0 is never produced by a finite or
// infinite score (fkey(-inf) = 0x007FFFFF) and serves as "empty".
__device__ __forceinline__ uint64_t ckey32(uint32_t score_bits, uint32_t idx) {
  return ((uint64_t)fkey(score_bits) << 32) | (uint64_t)(0xFFFFFFFFu - idx);
}
__device__ __forceinline__ uint32_t ckey_idx(uint64_t key) { return 0xFFFFFFFFu - (uint32_t)(key & 0xFFFFFFFFull); }
__device__ __forceinline__ float ckey_score(uint64_t key) { return __uint_as_float(unkey((uint32_t)(key >> 32))); }

template <typename T, typename Op>
__device__ __forceinline__ T block_reduce(T v, T* red, Op op, T identity) {
  for (int off = 16; off; off >>= 1) v = op(v, __shfl_xor_sync(kFullMask, v, off));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  T r = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : identity;
  if (threadIdx.x < 32) {
    for (int off = 16; off; off >>= 1) r = op(r, __shfl_xor_sync(kFullMask, r, off));
    if (threadIdx.x == 0) red[0] = r;
  }
  __syncthreads();
  r = red[0];
  __syncthreads();
  return r;
}

// One selected candidate: dkey(fp64 score) and local row.
struct TopkCand {
  uint64_t key;  // 0 = empty slot
  uint64_t idx;
};

// Where a call's results go: k entries per query, ranked under the contract; ranks past the valid entries
// hold (-inf, -1).  All pointers are device pointers.
struct TopkOut {
  float* scores;        // [nq, k]  (null: not written)
  double* scores64;     // optional [nq, k]
  int64_t* idx;         // [nq, k]
  int32_t* count;       // optional [nq]: valid entries
  int64_t* packed;      // optional [nq, k, 2]: (fp64 score bits, index) — the all-gather payload
  int64_t idx_offset;   // added to every local row written

  __device__ __forceinline__ void put(int q, int k, int rank, double score, int64_t row) const {
    const size_t o = (size_t)q * k + rank;
    if (scores) scores[o] = (float)score;
    if (scores64) scores64[o] = score;
    idx[o] = row + idx_offset;
    if (packed) {
      packed[2 * o] = __double_as_longlong(score);
      packed[2 * o + 1] = row + idx_offset;
    }
  }
  // ranks [valid, k) of query q; thread `tid` of `nthreads` writes every nthreads-th of them, tid 0 the count
  __device__ __forceinline__ void pad(int q, int k, int valid, int tid, int nthreads) const {
    for (int r = valid + tid; r < k; r += nthreads) {
      const size_t o = (size_t)q * k + r;
      if (scores) scores[o] = -INFINITY;
      if (scores64) scores64[o] = -INFINITY;
      idx[o] = -1;
      if (packed) {
        packed[2 * o] = __double_as_longlong(-INFINITY);
        packed[2 * o + 1] = -1;
      }
    }
    if (count && tid == 0) count[q] = valid;
  }
  // the results of queries q0, q0 + 1, ...
  TopkOut at(int q0, int k) const {
    TopkOut o = *this;
    const size_t off = (size_t)q0 * k;
    o.scores = scores ? scores + off : nullptr;
    o.scores64 = scores64 ? scores64 + off : nullptr;
    o.idx = idx + off;
    o.count = count ? count + q0 : nullptr;
    o.packed = packed ? packed + 2 * off : nullptr;
    return o;
  }
};

// Rank of entry c among keys[0, n) under (key desc, idx asc), by counting.  Over distinct (key, idx) pairs
// the ranks are a permutation of 0..n-1.
template <typename K, typename I>
__device__ __forceinline__ int rank_desc(const K* keys, const I* idx, int n, int c) {
  const K kc = keys[c];
  const I ic = idx[c];
  int rank = 0;
  for (int j = 0; j < n; ++j) {
    const K kj = keys[j];
    rank += (kj > kc || (kj == kc && idx[j] < ic)) ? 1 : 0;
  }
  return rank;
}

struct SelectSmem {
  int hist[256];
  int bin, above;
};

struct KeyCut {
  uint64_t lo;   // every key >= lo is selected (n_above >= 0: every key > lo and need - n_above keys == lo)
  int n_above;   // -1, or the window narrowed to single key values: count(key > lo), lo is the need-th key
};

// Block-wide selection of the `need` largest of a set of 64-bit keys (need <= set size), called by all
// kThreads threads.  `for_each_key(f)` calls f(key) on the keys this thread holds, wherever they sit (shared
// memory, global memory, registers); every key lies in [kmin, kmax].  Returns lo with
// need <= count(key >= lo) <= need + slack, or, when ties at the need-th key hold that count higher, that key
// itself with n_above = count(key > lo).
// Radix descent over the window [base, win_hi] of the key space that still holds the boundary: 256 equal
// bins, a shared-memory histogram, warp 0 finds the bin where the count from the top crosses what is still
// needed; that bin becomes the next window.  The window is sized from (kmin, kmax), not from the digit
// positions, so keys that cluster in a narrow range take two or three levels.  `sm` is read until the call
// returns: a barrier must separate the call from the next write to it.
template <int kThreads, class ForEachKey>
__device__ __forceinline__ KeyCut select_keys(ForEachKey for_each_key, uint64_t kmin, uint64_t kmax, int need,
                                              int slack, SelectSmem& sm) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int taken = 0;  // keys above the window, all selected
  uint64_t base = kmin, win_hi = kmax;
  int shift = 64 - __clzll((long long)((kmax - kmin) | 1ull)) - 8;
  shift = shift < 0 ? 0 : shift;
  for (;;) {
    for (int b = tid; b < 256; b += kThreads) sm.hist[b] = 0;
    __syncthreads();
    for_each_key([&](uint64_t key) {
      if (key >= base && key <= win_hi) atomicAdd(&sm.hist[(int)((key - base) >> shift)], 1);
    });
    __syncthreads();
    if (warp == 0) {
      // lane l owns bins [8l, 8l + 8); suf = keys in the bins of lanes >= l
      int own = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) own += sm.hist[8 * lane + j];
      int suf = own;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int v = __shfl_down_sync(kFullMask, suf, off);
        if (lane + off < 32) suf += v;
      }
      // the crossing lane: suf >= need while the lanes above it hold fewer than need
      if (suf >= need && suf - own < need) {
        int above = suf - own, b = 8 * lane + 7;
        for (; b > 8 * lane; --b) {
          if (above + sm.hist[b] >= need) break;
          above += sm.hist[b];
        }
        sm.bin = b;
        sm.above = above;
      }
    }
    __syncthreads();
    const int b = sm.bin, above = sm.above, in_bin = sm.hist[b];
    const uint64_t lo = base + ((uint64_t)b << shift);
    if (above + in_bin <= need + slack) return KeyCut{lo, -1};
    if (shift == 0) return KeyCut{lo, taken + above};
    need -= above;
    taken += above;
    base = lo;
    win_hi = base + ((1ull << shift) - 1ull);
    shift = shift > 8 ? shift - 8 : 0;
    __syncthreads();  // hist / bin are rewritten by the next level
  }
}

// Canonical fp64 dot product (identical in oracle/rpx_oracle.c::rpx_oracle_dot64):
// lane l accumulates, in increasing j then e order, the elements d = (j*32 + l)*8 + e
// (e = 0..7) with acc = acc + a*b — the bf16 x bf16 product is exact (even in fp32), so this is
// one rounding per addition — and the 32 partials are combined by the xor butterfly
// 16, 8, 4, 2, 1 (p = p + p_partner).
__device__ __forceinline__ double dot64_canonical(const __nv_bfloat16* __restrict__ qrow,  // smem or global
                                                  const __nv_bfloat16* __restrict__ erow, int d, int lane) {
  double acc = 0.0;
  const int chunks = d >> 3;
  // all of this lane's 16-byte loads of the (cold, DRAM-resident) index row go out before the first
  // dependent fma; the summation order is unchanged
  constexpr int kMaxIter = 8;  // d <= 8 * 32 * 8 = 2048 takes the batched path
  if (chunks <= kMaxIter * 32) {
    uint4 ev[kMaxIter];
#pragma unroll
    for (int it = 0; it < kMaxIter; ++it) {
      const int ch = lane + it * 32;
      ev[it] = ch < chunks ? *reinterpret_cast<const uint4*>(erow + ch * 8) : make_uint4(0u, 0u, 0u, 0u);
    }
#pragma unroll
    for (int it = 0; it < kMaxIter; ++it) {
      const int ch = lane + it * 32;
      if (ch < chunks) {
        const uint4 qv = *reinterpret_cast<const uint4*>(qrow + ch * 8);
        const uint32_t ew[4] = {ev[it].x, ev[it].y, ev[it].z, ev[it].w};
        const uint32_t qw[4] = {qv.x, qv.y, qv.z, qv.w};
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          // bf16 x bf16 is exact in fp32 (8 + 8 significand bits), so the fp32 product converted to
          // fp64 equals the exact product: one F2F per element instead of two (the fp32->fp64
          // conversion pipe, not HBM, was the limiter of this kernel)
          const float p0 = __uint_as_float(qw[w] << 16) * __uint_as_float(ew[w] << 16);
          const float p1 = __uint_as_float(qw[w] & 0xFFFF0000u) * __uint_as_float(ew[w] & 0xFFFF0000u);
          acc += (double)p0;
          acc += (double)p1;
        }
      }
    }
  } else {
    for (int ch = lane; ch < chunks; ch += 32) {
      const uint4 ev = *reinterpret_cast<const uint4*>(erow + ch * 8);
      const uint4 qv = *reinterpret_cast<const uint4*>(qrow + ch * 8);
      const uint32_t ew[4] = {ev.x, ev.y, ev.z, ev.w};
      const uint32_t qw[4] = {qv.x, qv.y, qv.z, qv.w};
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        const float p0 = __uint_as_float(qw[w] << 16) * __uint_as_float(ew[w] << 16);
        const float p1 = __uint_as_float(qw[w] & 0xFFFF0000u) * __uint_as_float(ew[w] & 0xFFFF0000u);
        acc += (double)p0;
        acc += (double)p1;
      }
    }
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) acc += __shfl_xor_sync(kFullMask, acc, off);
  return acc;
}

// ------------------------------------------------------------------------------- exactness guard
// A fast path ranks rows by an fp32 score s32 that differs from the contract's fp64 score s64 by at
// most eps = c(d) * ||q||_2 * max_i ||e_i||_2  (|sum of products| and every partial sum are bounded
// by sum |q_j e_ij| <= ||q|| ||e_i||):
//   wgmma path     every K=16 instruction adds 16 exact products to the fp32 accumulator; each addend
//                  may lose < 1 ulp of the largest magnitude involved when it is aligned, and the
//                  result is rounded once more: <= 18 * 2^-23 * sum|p| per instruction, d/16
//                  instructions  ->  c = (18 d / 16 + 2) * 2^-23   (2.0e-4 for d = 1472)
//   streaming path per lane <= 8 ceil(d/256) fused multiply-adds + 5 butterfly additions, round to
//                  nearest: c = (8 ceil(d/256) + 8) * 2^-24      (3.3e-6 for d = 1472)
// both doubled for safety.  (The diagnostics counter max_err_bits records what the guards actually
// observe; tests assert it stays far below eps.)
//
// Let R be the re-scored set, (B, iB) its k-th best entry under the contract, and U the largest fp32
// score any row outside R can have (dropped by a threshold, cut by a compaction, or not selected for
// re-scoring).  A row outside R has s64 <= U + eps; if B > U + eps none of them can rank at or before
// the k-th entry of R, so the top-k of R is the top-k of the corpus.  Otherwise the query is flagged
// and the exact path (rpx_exact.cu) recomputes it from all rows that rank at or before (B, iB).
__host__ __device__ inline float guard_coeff_mma(int d) { return 2.0f * ((18.0f * d) / 16.0f + 2.0f) * 1.1920929e-7f; }
__host__ __device__ inline float guard_coeff_stream(int d) {
  return 2.0f * (8.0f * (float)((d + 255) / 256) + 8.0f) * 5.9604645e-8f;
}

struct GuardOut {
  IndexState* state;     // norm bound in, flag counters out
  uint32_t* flagged;     // [nq] list of flagged query numbers (first state->n_flagged entries valid)
  ExactBound* bounds;    // [nq]
};

// The guard's epsilon for one query (also recorded in the diagnostics).
__device__ __forceinline__ float guard_eps(const GuardOut& g, float q2, float coeff) {
  return coeff * sqrtf(q2 * g.state->norm2_max) * 1.0001f;
}

// Is the ranked result proven?  n_ranked = number of re-scored candidates, kth_score = the k-th best of
// them (valid when n_ranked >= k), u = the best fp32 score a row outside the re-scored set can have
// (-inf: nothing was left out).
__device__ __forceinline__ bool guard_proven(int k, int n_ranked, double kth_score, float u, float eps) {
  const bool nothing_left_out = (u == -INFINITY);
  if (n_ranked >= k) return nothing_left_out || kth_score > (double)u + (double)eps;
  return nothing_left_out;
}

// Hands query q to the exact path (called by ONE thread).
__device__ __forceinline__ void guard_flag(const GuardOut& g, int q, int k, int n_ranked, double kth_score,
                                           uint32_t kth_idx) {
  ExactBound b;
  b.score = n_ranked >= k ? kth_score : -INFINITY;
  b.idx = n_ranked >= k ? (int64_t)kth_idx : (int64_t)0x7FFFFFFF;
  g.bounds[q] = b;
  const uint32_t pos = atomicAdd(&g.state->n_flagged, 1u);
  g.flagged[pos] = (uint32_t)q;
}

// Called by ONE thread per query once the re-scored set has been ranked.  Returns true when proven.
__device__ __forceinline__ bool guard_decide(const GuardOut& g, int q, int k, int n_ranked, double kth_score,
                                             uint32_t kth_idx, float u, float q2, float coeff, float max_err) {
  const float eps = guard_eps(g, q2, coeff);
  atomicMax(&g.state->max_err_bits, __float_as_uint(max_err));   // non-negative floats order like their bits
  atomicMax(&g.state->max_eps_bits, __float_as_uint(eps));
  const bool proven = guard_proven(k, n_ranked, kth_score, u, eps);
  if (!proven) guard_flag(g, q, k, n_ranked, kth_score, kth_idx);
  return proven;
}

// ------------------------------------------------------------------------------- host entry points
// One similarity + top-k request (all pointers are device pointers).
struct TopkCall {
  const __nv_bfloat16* Q;   // [nq, d]
  int nq;
  const __nv_bfloat16* E;   // [n, d]
  int64_t n;
  int d, k;
  const uint32_t* mask;     // optional access bitmask [nq][mask_stride]
  int64_t mask_stride;
  TopkOut out;
  GuardOut guard;           // state of the index handle, [nq] guard scratch
  cudaStream_t st;
};
// re-score set size for k results (k + margin; the guard covers what the margin does not)
inline int topk_n_res(int k) { return k + (k / 8 > 12 ? k / 8 : 12); }
constexpr int kFastPathMaxK = 200;   // larger k goes through the exact path

int launch_row_norm_max(const __nv_bfloat16* E, int64_t n, int d, IndexState* state, cudaStream_t st);
size_t exact_cand_bytes(int64_t n);
int launch_exact_topk(const TopkCall& c, void* cand_ws, bool all_queries);
bool smallq_supported(int nq, int k, int d);
size_t smallq_workspace_bytes(int num_sms);
int launch_smallq_topk(const TopkCall& c, void* ws);
size_t mma_topk_workspace_bytes(int nq, int k, int d, int num_sms);
int run_mma_topk(const TopkCall& c, void* ws, size_t ws_bytes);
// k-way merge of per-shard results; `packed`: one [n_parts, nq, k, 2] (score bits, index) buffer.
int launch_topk_merge(const double* d_scores64, const int64_t* d_idx_or_packed, bool packed, int n_parts, int nq, int k,
                      float* d_out_scores, double* d_out_scores64, int64_t* d_out_idx, int32_t* d_out_count,
                      cudaStream_t st);

}  // namespace rpx
