// rpx_topk_common.cuh — device helpers shared by the three top-k paths
// (rpx_simtopk.cu: tensor-core path, rpx_smallq.cu: HBM-streaming path for <= 4 queries,
//  rpx_exact.cu: exact fp64 fallback) and the device-resident state of an index handle.
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

// Block-wide sum of per-thread counts with ONE barrier per call: warp REDUX, one shared-memory
// atomic per warp, three rotating counters (slot i % 3 is used by call i and cleared during call
// i + 1, well before call i + 3 adds to it again).  `slots` must be zero on the first call.
__device__ __forceinline__ int block_count(int m, int* slots, int iter) {
  m = __reduce_add_sync(kFullMask, m);
  int* cur = slots + iter % 3;
  if ((threadIdx.x & 31) == 0 && m != 0) atomicAdd(cur, m);
  __syncthreads();
  const int total = *cur;
  if (threadIdx.x == 0) slots[(iter + 2) % 3] = 0;
  return total;
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

}  // namespace rpx
