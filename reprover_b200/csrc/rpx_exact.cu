// rpx_exact.cu — the exact (fp64) top-k path and the row-norm pass of an index handle.
//
// Replaces, for the queries the fast paths cannot prove (see the exactness guard in
// rpx_topk_common.cuh) and for k beyond the fast paths' list sizes, the reference's
//     similarities = ctx_emb @ premise_emb.t();  idxs = similarities.argsort(descending=True)
// (common.py:307-308) with the contract's arithmetic itself: every admissible row is scored with the
// canonical fp64 dot product and the k best under (score desc, index asc) are selected exactly
// (select_keys on the monotone 64-bit score keys, then on the indices of the entries tied at the k-th key).
//
//   exact_topk_kernel   cooperative launch, one CTA per SM.  Per query: phase A — all warps stream the
//                       index (one row per warp trip, 16-byte coalesced loads, fp64 accumulation) and
//                       append the rows that rank at or before the guard's bound; grid barrier; phase B —
//                       CTA 0 selects and ranks; grid barrier.  With nothing flagged the kernel returns
//                       at once (~3 us), which is all the fast paths ever pay for it on ordinary data.
//   row_norm_max_kernel HBM-bound pass over the index: max_i sum_j E[i,j]^2 -> IndexState::norm2_max
//                       (the ||e|| factor of the guard's epsilon); runs once per rpx_index_create.
#include "rpx_common.cuh"
#include "rpx_topk_common.cuh"

namespace rpx {

namespace {

constexpr int kExactThreads = 512;
constexpr int kExactMaxK = 1024;

// Sense-reversing grid barrier (all CTAs co-resident: cooperative launch).  `count` returns to zero
// after every barrier, `gen` only ever increments, so nothing has to be reset between launches.
__device__ __forceinline__ void grid_barrier(IndexState* st) {
  __syncthreads();
  if (threadIdx.x == 0) {
    volatile uint32_t* gen = &st->bar_gen;
    const uint32_t g = *gen;  // cannot advance before this CTA has arrived
    __threadfence();
    if (atomicAdd(&st->bar_count, 1u) == gridDim.x - 1) {
      st->bar_count = 0u;
      __threadfence();
      atomicAdd(&st->bar_gen, 1u);
    } else {
      while (*gen == g) {
      }
    }
    __threadfence();
  }
  __syncthreads();
}

struct ExactParams {
  const __nv_bfloat16* Q;
  const __nv_bfloat16* E;
  int64_t n;
  int d, k, nq;
  const uint32_t* mask;
  int64_t mask_stride;
  TopkOut out;
  GuardOut guard;
  TopkCand* cand;    // [n]
  int all_queries;   // 1: every query 0..nq-1 goes through this path (no guard ran)
};

__global__ void __launch_bounds__(kExactThreads, 1) exact_topk_kernel(ExactParams p) {
  extern __shared__ __align__(16) uint8_t sm_raw[];
  __nv_bfloat16* sq = reinterpret_cast<__nv_bfloat16*>(sm_raw);                                   // [d]
  uint64_t* sel_key = reinterpret_cast<uint64_t*>(sm_raw + (((size_t)p.d * 2 + 15) & ~(size_t)15));  // [kExactMaxK]
  uint32_t* sel_idx = reinterpret_cast<uint32_t*>(sel_key + kExactMaxK);                            // [kExactMaxK]
  __shared__ SelectSmem sel;
  __shared__ int n_sel;

  const int tid = threadIdx.x, lane = tid & 31;
  const int n_f = p.all_queries ? p.nq : (int)*reinterpret_cast<volatile uint32_t*>(&p.guard.state->n_flagged);
  if (n_f == 0) return;
  const int64_t gwarp = (int64_t)blockIdx.x * (kExactThreads / 32) + (tid >> 5);
  const int64_t n_warps = (int64_t)gridDim.x * (kExactThreads / 32);

  for (int f = 0; f < n_f; ++f) {
    const int q = p.all_queries ? f : (int)p.guard.flagged[f];
    ExactBound bound;
    bound.score = -INFINITY;
    bound.idx = 0x7FFFFFFF;
    if (!p.all_queries) bound = p.guard.bounds[q];
    const bool unbounded = bound.score == -INFINITY;
    for (int i = tid; i < p.d / 8; i += kExactThreads)
      reinterpret_cast<uint4*>(sq)[i] = reinterpret_cast<const uint4*>(p.Q + (size_t)q * p.d)[i];
    __syncthreads();
    // ---- phase A: score every admissible row, keep those that rank at or before the bound
    const uint32_t* mrow = p.mask ? p.mask + (size_t)q * p.mask_stride : nullptr;
    for (int64_t row = gwarp; row < p.n; row += n_warps) {
      if (mrow != nullptr && !((mrow[row >> 5] >> (row & 31)) & 1u)) continue;  // warp-uniform
      const double s = dot64_canonical(sq, p.E + (size_t)row * p.d, p.d, lane);
      const bool keep = unbounded || s > bound.score || (s == bound.score && row <= bound.idx);
      if (lane == 0 && keep) {
        const uint32_t pos = atomicAdd(&p.guard.state->fb_count, 1u);
        TopkCand c;
        c.key = dkey(s);
        c.idx = (uint64_t)row;
        p.cand[pos] = c;
      }
    }
    grid_barrier(p.guard.state);
    // ---- phase B: exact selection + ranking by CTA 0
    if (blockIdx.x == 0) {
      const int C = (int)*reinterpret_cast<volatile uint32_t*>(&p.guard.state->fb_count);
      const int k = p.k;
      if (tid == 0) n_sel = 0;
      // the k best: every key above T, and of the keys equal to T those with index <= idx_cut
      uint64_t T = 0ull, idx_cut = ~0ull;
      if (C > k) {
        const auto each_key = [&](auto f) {
          for (int i = tid; i < C; i += kExactThreads) f(__ldcg(&p.cand[i].key));
        };
        const KeyCut cut = select_keys<kExactThreads>(each_key, 0ull, ~0ull, k, 0, sel);
        T = cut.lo;
        if (cut.n_above >= 0) {
          // more entries equal T than the top k has room for: the k - n_above smallest indices among them
          const auto each_tied = [&](auto f) {
            for (int i = tid; i < C; i += kExactThreads)
              if (__ldcg(&p.cand[i].key) == T) f(0xFFFFFFFFull - __ldcg(&p.cand[i].idx));
          };
          __syncthreads();  // `sel` is rewritten
          idx_cut = 0xFFFFFFFFull - select_keys<kExactThreads>(each_tied, 0ull, 0xFFFFFFFFull, k - cut.n_above, 0, sel).lo;
        }
      }
      __syncthreads();  // n_sel
      for (int i = tid; i < C; i += kExactThreads) {
        const uint64_t key = __ldcg(&p.cand[i].key);
        if (key < T) continue;
        const uint64_t ix = __ldcg(&p.cand[i].idx);
        if (key > T || ix <= idx_cut) {
          const int pos = atomicAdd(&n_sel, 1);
          if (pos < kExactMaxK) {
            sel_key[pos] = key;
            sel_idx[pos] = (uint32_t)ix;
          }
        }
      }
      __syncthreads();
      const int ns = n_sel < k ? n_sel : k;  // == k whenever C > k
      for (int c = tid; c < ns; c += kExactThreads)
        p.out.put(q, k, rank_desc(sel_key, sel_idx, ns, c), undkey(sel_key[c]), sel_idx[c]);
      p.out.pad(q, k, ns, tid, kExactThreads);
      __syncthreads();
      if (tid == 0) p.guard.state->fb_count = 0u;
    }
    grid_barrier(p.guard.state);
  }
  if (blockIdx.x == 0 && tid == 0) {
    if (!p.all_queries) p.guard.state->n_flagged = 0u;
    atomicAdd(&p.guard.state->n_exact_total, (uint32_t)n_f);
  }
}

// max over rows of sum e^2 (fp32), one warp per row trip, two rows in flight per warp.
__global__ void __launch_bounds__(256) row_norm_max_kernel(const __nv_bfloat16* __restrict__ E, int64_t n, int d,
                                                           IndexState* __restrict__ state) {
  const int lane = threadIdx.x & 31;
  const int64_t gwarp = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int64_t n_warps = (int64_t)gridDim.x * 8;
  const int chunks = d >> 3;
  float best = 0.f;
  for (int64_t row = gwarp; row < n; row += n_warps) {
    const uint4* src = reinterpret_cast<const uint4*>(E + (size_t)row * d);
    float acc = 0.f;
    for (int ch = lane; ch < chunks; ch += 32) {
      const uint4 v = __ldcs(src + ch);  // streamed once
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float a = __uint_as_float(w[i] << 16), b = __uint_as_float(w[i] & 0xFFFF0000u);
        acc = fmaf(a, a, acc);
        acc = fmaf(b, b, acc);
      }
    }
    for (int off = 16; off; off >>= 1) acc += __shfl_xor_sync(kFullMask, acc, off);
    best = fmaxf(best, acc);
  }
  __shared__ float red[8];
  if (lane == 0) red[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) best = fmaxf(best, red[w]);
    // fp32 accumulation of <= d non-negative terms: relative error <= d * 2^-24; round the bound up
    best *= 1.0f + 1.2e-7f * (float)d + 1e-6f;
    atomicMax(reinterpret_cast<uint32_t*>(&state->norm2_max), __float_as_uint(best));
  }
}

}  // namespace

size_t exact_cand_bytes(int64_t n) { return align_up((size_t)(n > 0 ? n : 1) * sizeof(TopkCand), 256); }

int launch_row_norm_max(const __nv_bfloat16* E, int64_t n, int d, IndexState* state, cudaStream_t st) {
  if (n <= 0) return RPX_OK;
  DeviceInfo dev;
  RPX_TRY(get_device_info(&dev));
  int64_t blocks = ceil_div64(n, 8);
  if (blocks > (int64_t)dev.num_sms * 8) blocks = (int64_t)dev.num_sms * 8;
  row_norm_max_kernel<<<(unsigned)blocks, 256, 0, st>>>(E, n, d, state);
  RPX_CUDA_OK(cudaGetLastError());
  return RPX_OK;
}

int launch_exact_topk(const TopkCall& c, void* cand_ws, bool all_queries) {
  RPX_REQUIRE(c.k >= 1 && c.k <= kExactMaxK, RPX_ERR_UNSUPPORTED, "top-k: k=%d outside [1, %d]", c.k, kExactMaxK);
  DeviceInfo dev;
  RPX_TRY(get_device_info(&dev));
  ExactParams p;
  p.Q = c.Q;
  p.E = c.E;
  p.n = c.n;
  p.d = c.d;
  p.k = c.k;
  p.nq = c.nq;
  p.mask = c.mask;
  p.mask_stride = c.mask_stride;
  p.out = c.out;
  p.guard = c.guard;
  p.cand = static_cast<TopkCand*>(cand_ws);
  p.all_queries = all_queries ? 1 : 0;
  const size_t smem = (((size_t)c.d * 2 + 15) & ~(size_t)15) + (size_t)kExactMaxK * (sizeof(uint64_t) + sizeof(uint32_t));
  static thread_local int configured = -1;
  if (configured != dev.device) {
    RPX_CUDA_OK(cudaFuncSetAttribute(exact_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    configured = dev.device;
  }
  RPX_REQUIRE(smem <= 64 * 1024, RPX_ERR_UNSUPPORTED, "exact top-k: d=%d too wide", c.d);
  // the kernel spins on a grid barrier: its CTAs must be co-resident
  void* args[] = {&p};
  RPX_CUDA_OK(cudaLaunchCooperativeKernel((const void*)exact_topk_kernel, dim3(dev.num_sms), dim3(kExactThreads), args, smem,
                                          c.st));
  return RPX_OK;
}

}  // namespace rpx
