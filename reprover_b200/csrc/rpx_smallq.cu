// rpx_smallq.cu — similarity + top-k for 1 or 2 queries as ONE HBM-bound streaming kernel.
//
// This is the shape the reference's only production call has: `PremiseRetriever.retrieve`
// (retrieval/model.py:338-375, called per proof state from prover/tactic_generator.py:286-292)
// scores ONE state against the whole index (`Q @ E.T`, common.py:307) and sorts all N scores
// (:308).  With a handful of queries the contraction is a matrix-vector product: 2 flop per index
// byte, far below the tensor-core ridge, so the bound is the 2*N*d bytes of the bf16 index
// (SURVEY.md §8d) and the kernel is written as a byte streamer, not as a GEMM:
//
//   * persistent grid, one 512-thread CTA per SM; a warp owns row pairs  g = cta + grid*(warp + 16 j):
//     neighbouring rows (near-duplicate premises sit next to each other in a Lean file) land on
//     different SMs, every warp load is 512 contiguous bytes of one row (16 B per lane, streaming /
//     evict-first), two rows = up to 16 loads per lane in flight before the first use;
//   * the queries live in shared memory as packed bf16; bf16 x bf16 products are exact in fp32 and are
//     accumulated with fp32 FMAs, lane partials are combined with the xor butterfly;
//   * rows the access bitmask (common.py:313-318) hides from every query are never read;
//   * per-query candidate heap in registers, one (score, index) key per lane, kept by warp shuffles
//     (REDUX min + ballot); at the end each warp hands its 8 best to the CTA, the CTA its 16 best to
//     global memory — 2368 keys per query instead of N scores;
//   * every CTA re-scores its 16 rows in fp64 in the canonical order (one warp per row, all SMs in
//     parallel) before it leaves; the LAST CTA to finish (ticket counter) runs the tail on those exact
//     scores: selects the k best, ranks them under (score desc, index asc), writes the results and runs
//     the exactness guard (rpx_topk_common.cuh) against everything the fp32 heaps dropped.
// No sampling pass, no memsets, no second launch (the exact-path kernel that follows returns at once
// unless the guard flagged a query).
#include "rpx_common.cuh"
#include "rpx_topk_common.cuh"

namespace rpx {

namespace {

constexpr int kSqThreads = 512;
constexpr int kSqWarps = kSqThreads / 32;
constexpr int kSqWarpKeep = 8;    // keys a warp hands to its CTA
constexpr int kSqCtaKeep = 16;    // keys a CTA hands to the tail
constexpr int kSqSelMax = 288;    // >= n_res + selection slack for k <= 200
constexpr int kSqSelSlack = 16;

struct SmallQParams {
  const __nv_bfloat16* Q;
  const __nv_bfloat16* E;
  int64_t n;
  int d, k;
  const uint32_t* mask;
  int64_t mask_stride;
  TopkOut out;
  GuardOut guard;
  TopkCand* cta_cand;  // [grid][NQ][kSqCtaKeep] exact (fp64 score, row) of each CTA's best rows
  uint64_t* cta_thr;   // [grid][NQ] best key that CTA dropped (0: none)
  float guard_coeff;
};

__device__ __forceinline__ float dot8_acc(const uint4& e, const uint4& q, float acc) {
  const uint32_t ew[4] = {e.x, e.y, e.z, e.w};
  const uint32_t qw[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
  for (int w = 0; w < 4; ++w) {
    acc = fmaf(__uint_as_float(ew[w] << 16), __uint_as_float(qw[w] << 16), acc);
    acc = fmaf(__uint_as_float(ew[w] & 0xFFFF0000u), __uint_as_float(qw[w] & 0xFFFF0000u), acc);
  }
  return acc;
}

__device__ __forceinline__ uint64_t shfl_u64(uint64_t v, int src) {
  const uint32_t lo = __shfl_sync(kFullMask, (uint32_t)v, src);
  const uint32_t hi = __shfl_sync(kFullMask, (uint32_t)(v >> 32), src);
  return ((uint64_t)hi << 32) | lo;
}

// One key per lane; `hmin` / `hlane` (warp-uniform) are the smallest key of the heap and its lane.
struct WarpHeap {
  uint64_t key = 0ull;
  uint64_t hmin = 0ull;
  int hlane = 0;
  __device__ __forceinline__ void offer(uint64_t cand, int lane) {  // warp-uniform `cand`
    if (cand <= hmin) return;
    if (lane == hlane) key = cand;
    const uint32_t hi = (uint32_t)(key >> 32), lo = (uint32_t)key;
    const uint32_t mhi = __reduce_min_sync(kFullMask, hi);
    const uint32_t mlo = __reduce_min_sync(kFullMask, hi == mhi ? lo : 0xFFFFFFFFu);
    hmin = ((uint64_t)mhi << 32) | mlo;
    hlane = __ffs(__ballot_sync(kFullMask, hi == mhi && lo == mlo)) - 1;
  }
};

// NQ queries (1 or 2), ITS = 16-byte chunks per lane per row (ceil(d / 256)).
template <int NQ, int ITS>
__global__ void __launch_bounds__(kSqThreads, 1) smallq_topk_kernel(const SmallQParams p) {
  extern __shared__ __align__(16) uint8_t sm_raw[];
  const int d = p.d, CH = d >> 3;
  uint4* sQ = reinterpret_cast<uint4*>(sm_raw);  // [NQ][CH] packed bf16
  uint64_t* wkeys = reinterpret_cast<uint64_t*>(sQ + (size_t)NQ * CH);  // [NQ][kSqWarps * kSqWarpKeep]
  uint64_t* ckeys = wkeys + NQ * kSqWarps * kSqWarpKeep;                  // [NQ][kSqCtaKeep]
  uint64_t* cdrop = ckeys + NQ * kSqCtaKeep;                              // [NQ]
  uint8_t* tail_smem = reinterpret_cast<uint8_t*>(cdrop + NQ);            // tail only
  __shared__ int is_last;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < NQ * CH; i += kSqThreads) sQ[i] = reinterpret_cast<const uint4*>(p.Q)[i];
  for (int i = tid; i < NQ * (kSqWarps * kSqWarpKeep + kSqCtaKeep + 1); i += kSqThreads) wkeys[i] = 0ull;
  __syncthreads();

  // ------------------------------------------------------------------ streaming pass
  WarpHeap heap[NQ];
  const int64_t groups = (p.n + 1) >> 1;
  const int64_t gstride = (int64_t)gridDim.x * kSqWarps;
  for (int64_t g = (int64_t)blockIdx.x + (int64_t)gridDim.x * warp; g < groups; g += gstride) {
    const int64_t r0 = 2 * g;
    uint32_t acc_bits[NQ];
    uint32_t any = 0u;
    const uint32_t live = (r0 + 1 < p.n) ? 3u : 1u;
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
      uint32_t w = 3u;
      if (p.mask != nullptr) w = p.mask[(size_t)q * p.mask_stride + (size_t)(r0 >> 5)] >> (r0 & 31);
      acc_bits[q] = w & live;
      any |= acc_bits[q];
    }
    if (any == 0u) continue;  // warp-uniform: nobody may see these rows, do not read them
    const uint4* e0 = reinterpret_cast<const uint4*>(p.E + (size_t)r0 * d);
    const uint4* e1 = e0 + CH;
    uint4 v0[ITS], v1[ITS];
#pragma unroll
    for (int it = 0; it < ITS; ++it) {
      const int ch = lane + 32 * it;
      v0[it] = (ch < CH && (any & 1u)) ? __ldcs(e0 + ch) : make_uint4(0u, 0u, 0u, 0u);
    }
#pragma unroll
    for (int it = 0; it < ITS; ++it) {
      const int ch = lane + 32 * it;
      v1[it] = (ch < CH && (any & 2u)) ? __ldcs(e1 + ch) : make_uint4(0u, 0u, 0u, 0u);
    }
    float a0[NQ], a1[NQ];
#pragma unroll
    for (int q = 0; q < NQ; ++q) a0[q] = a1[q] = 0.f;
#pragma unroll
    for (int it = 0; it < ITS; ++it) {
      const int ch = lane + 32 * it;
      if (ch < CH) {
#pragma unroll
        for (int q = 0; q < NQ; ++q) {
          const uint4 qv = sQ[q * CH + ch];
          a0[q] = dot8_acc(v0[it], qv, a0[q]);
          a1[q] = dot8_acc(v1[it], qv, a1[q]);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
#pragma unroll
      for (int off = 16; off; off >>= 1) {
        a0[q] += __shfl_xor_sync(kFullMask, a0[q], off);
        a1[q] += __shfl_xor_sync(kFullMask, a1[q], off);
      }
      if (acc_bits[q] & 1u) heap[q].offer(ckey32(__float_as_uint(a0[q]), (uint32_t)r0), lane);
      if (acc_bits[q] & 2u) heap[q].offer(ckey32(__float_as_uint(a1[q]), (uint32_t)r0 + 1u), lane);
    }
  }

  // ------------------------------------------------------------------ warp -> CTA -> global
#pragma unroll
  for (int q = 0; q < NQ; ++q) {
    const uint64_t mine = heap[q].key;
    int rank = 0;
    for (int j = 0; j < 32; ++j) rank += shfl_u64(mine, j) > mine ? 1 : 0;
    if (mine != 0ull) {
      if (rank < kSqWarpKeep) wkeys[q * (kSqWarps * kSqWarpKeep) + warp * kSqWarpKeep + rank] = mine;
      else if (rank == kSqWarpKeep) atomicMax(reinterpret_cast<unsigned long long*>(&cdrop[q]), (unsigned long long)mine);
    }
  }
  __syncthreads();
  constexpr int kPerQ = kSqWarps * kSqWarpKeep;  // 128
  for (int t = tid; t < NQ * kPerQ; t += kSqThreads) {
    const int q = t / kPerQ, i = t - q * kPerQ;
    const uint64_t mine = wkeys[q * kPerQ + i];
    if (mine == 0ull) continue;
    int rank = 0;
    for (int j = 0; j < kPerQ; ++j) rank += wkeys[q * kPerQ + j] > mine ? 1 : 0;
    if (rank < kSqCtaKeep) ckeys[q * kSqCtaKeep + rank] = mine;
    else if (rank == kSqCtaKeep) atomicMax(reinterpret_cast<unsigned long long*>(&cdrop[q]), (unsigned long long)mine);
  }
  __syncthreads();
  // ---- every CTA re-scores ITS candidates in fp64 (canonical order), one warp per row: 148 CTAs x 16 rows
  // in parallel, while the rows are still warm — the tail then ranks exact scores and never touches the index
  float err = 0.f;
  for (int t = warp; t < NQ * kSqCtaKeep; t += kSqWarps) {
    const int q = t / kSqCtaKeep;
    const uint64_t key = ckeys[t];
    TopkCand c;
    c.key = 0ull;
    c.idx = ~0ull;
    if (key != 0ull) {
      const uint32_t row = ckey_idx(key);
      const double s = dot64_canonical(reinterpret_cast<const __nv_bfloat16*>(sQ + (size_t)q * CH), p.E + (size_t)row * d, d, lane);
      c.key = dkey(s);
      c.idx = row;
      err = fmaxf(err, fabsf((float)(s - (double)ckey_score(key))));
    }
    if (lane == 0) p.cta_cand[(size_t)blockIdx.x * NQ * kSqCtaKeep + t] = c;
  }
  if (lane == 0 && err > 0.f) atomicMax(&p.guard.state->max_err_bits, __float_as_uint(err));
  if (tid < NQ) p.cta_thr[(size_t)blockIdx.x * NQ + tid] = cdrop[tid];
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const uint32_t t = atomicAdd(&p.guard.state->ticket, 1u);
    is_last = (t == gridDim.x - 1) ? 1 : 0;
    if (is_last) p.guard.state->ticket = 0u;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();

  // ------------------------------------------------------------------ tail (last CTA only)
  // exact (fp64 score, index) pairs of every CTA's candidates: select the k best, rank, write, guard
  const int G = (int)gridDim.x * kSqCtaKeep;  // candidates per query
  uint64_t* k64 = reinterpret_cast<uint64_t*>((reinterpret_cast<uintptr_t>(tail_smem) + 15) & ~(uintptr_t)15);  // [G]
  uint32_t* ix = reinterpret_cast<uint32_t*>(k64 + G);                                                            // [G]
  uint64_t* sel_key = reinterpret_cast<uint64_t*>((reinterpret_cast<uintptr_t>(ix + G) + 15) & ~(uintptr_t)15);   // [kSqSelMax]
  uint32_t* sel_idx = reinterpret_cast<uint32_t*>(sel_key + kSqSelMax);                                            // [kSqSelMax]
  __shared__ uint64_t red64[32];
  __shared__ float redf[32];
  __shared__ int redi[32];
  __shared__ SelectSmem sel;
  __shared__ int n_sel;
  __shared__ double kth_score;
  __shared__ uint32_t kth_idx;

  for (int q = 0; q < NQ; ++q) {
    uint64_t kmin = ~0ull, kmax = 0ull, udrop = 0ull;
    int valid = 0;
    for (int i = tid; i < G; i += kSqThreads) {
      const int cta = i / kSqCtaKeep, s = i - cta * kSqCtaKeep;
      const TopkCand* src = &p.cta_cand[((size_t)cta * NQ + q) * kSqCtaKeep + s];
      const uint64_t key = __ldcg(&src->key);
      k64[i] = key;
      ix[i] = (uint32_t)__ldcg(&src->idx);
      if (key != 0ull) {
        ++valid;
        kmin = key < kmin ? key : kmin;
        kmax = key > kmax ? key : kmax;
      }
    }
    for (int c = tid; c < (int)gridDim.x; c += kSqThreads) {
      const uint64_t t = __ldcg(&p.cta_thr[(size_t)c * NQ + q]);
      udrop = t > udrop ? t : udrop;
    }
    if (tid == 0) n_sel = 0;
    kmin = block_reduce<uint64_t>(kmin, red64, [](uint64_t a, uint64_t b) { return a < b ? a : b; }, ~0ull);
    kmax = block_reduce<uint64_t>(kmax, red64, [](uint64_t a, uint64_t b) { return a > b ? a : b; }, 0ull);
    udrop = block_reduce<uint64_t>(udrop, red64, [](uint64_t a, uint64_t b) { return a > b ? a : b; }, 0ull);
    const int total = block_reduce<int>(valid, redi, [](int a, int b) { return a + b; }, 0);
    const int k = p.k;
    // threshold on the fp64 keys: count(key >= lo) in [k, k + slack] unless ties hold it higher (empty slots,
    // key 0, lie below kmin)
    uint64_t lo = total > 0 ? kmin : 1ull;
    if (total > k + kSqSelSlack) {
      const auto each_key = [&](auto f) {
        for (int i = tid; i < G; i += kSqThreads) f(k64[i]);
      };
      lo = select_keys<kSqThreads>(each_key, kmin, kmax, k, kSqSelSlack, sel).lo;
    }
    for (int i = tid; i < G; i += kSqThreads) {
      const uint64_t key = k64[i];
      if (key != 0ull && key >= lo) {
        const int pos = atomicAdd(&n_sel, 1);
        if (pos < kSqSelMax) {
          sel_key[pos] = key;
          sel_idx[pos] = ix[i];
        }
      }
    }
    float q2 = 0.f;
    const __nv_bfloat16* sq = reinterpret_cast<const __nv_bfloat16*>(sQ + (size_t)q * CH);
    for (int i = tid; i < d; i += kSqThreads) {
      const float v = __bfloat162float(sq[i]);
      q2 = fmaf(v, v, q2);
    }
    q2 = block_reduce<float>(q2, redf, [](float a, float b) { return a + b; }, 0.f);  // (also orders n_sel / sel_*)
    // more exact ties at the k-th score than the ranking buffer holds: let the exact path do it
    const bool overflow = n_sel > kSqSelMax;
    const int ns = overflow ? kSqSelMax : n_sel;
    for (int c = tid; c < ns; c += kSqThreads) {
      const int rank = rank_desc(sel_key, sel_idx, ns, c);
      if (rank < k) {
        const double sc = undkey(sel_key[c]);
        p.out.put(q, k, rank, sc, sel_idx[c]);
        if (rank == k - 1) {
          kth_score = sc;
          kth_idx = sel_idx[c];
        }
      }
    }
    const int nvalid = ns < k ? ns : k;
    p.out.pad(q, k, nvalid, tid, kSqThreads);
    __syncthreads();
    if (tid == 0) {
      // the candidates were ranked by their exact scores; what can still be missing is a row a warp or
      // CTA heap dropped on its fp32 score (udrop = the best such key)
      const float u = udrop != 0ull ? ckey_score(udrop) : -INFINITY;
      guard_decide(p.guard, q, k, overflow ? 0 : ns, kth_score, kth_idx, overflow ? INFINITY : u, q2, p.guard_coeff,
                   0.f);
    }
    __syncthreads();
  }
}

size_t smallq_smem_bytes(int nq, int d, int grid) {
  const size_t CH = (size_t)d >> 3;
  size_t b = (size_t)nq * CH * 16;
  b += (size_t)nq * (kSqWarps * kSqWarpKeep + kSqCtaKeep + 1) * 8;
  b += 16 + (size_t)grid * kSqCtaKeep * (8 + 4);           // tail: fp64 keys + rows
  b += 16 + (size_t)kSqSelMax * (8 + 4);                    // tail: ranking buffer
  return b;
}

template <int NQ, int ITS>
int launch_one(const SmallQParams& p, int grid, size_t smem, cudaStream_t st, int device) {
  auto kern = smallq_topk_kernel<NQ, ITS>;
  static thread_local int configured = -1;
  if (configured != device) {
    RPX_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    configured = device;
  }
  kern<<<grid, kSqThreads, smem, st>>>(p);
  RPX_CUDA_OK(cudaGetLastError());
  return RPX_OK;
}

template <int NQ>
int launch_its(const SmallQParams& p, int its, int grid, size_t smem, cudaStream_t st, int device) {
  if (its <= 1) return launch_one<NQ, 1>(p, grid, smem, st, device);
  if (its <= 2) return launch_one<NQ, 2>(p, grid, smem, st, device);
  if (its <= 4) return launch_one<NQ, 4>(p, grid, smem, st, device);
  if (its <= 6) return launch_one<NQ, 6>(p, grid, smem, st, device);
  return launch_one<NQ, 8>(p, grid, smem, st, device);
}

}  // namespace

bool smallq_supported(int nq, int k, int d) { return nq >= 1 && nq <= 2 && k >= 1 && k <= 200 && d % 8 == 0 && d <= 2048; }

size_t smallq_workspace_bytes(int num_sms) {
  return align_up((size_t)num_sms * 2 * kSqCtaKeep * sizeof(TopkCand), 256) + align_up((size_t)num_sms * 2 * 8, 256);
}

// one launch, instantiated for NQ = nq
int launch_smallq_topk(const TopkCall& c, void* ws) {
  RPX_REQUIRE(smallq_supported(c.nq, c.k, c.d), RPX_ERR_UNSUPPORTED, "small-Q top-k: nq=%d k=%d d=%d", c.nq, c.k, c.d);
  DeviceInfo dev;
  RPX_TRY(get_device_info(&dev));
  const int grid = dev.num_sms;
  const int its = ((c.d >> 3) + 31) >> 5;
  uint8_t* base = static_cast<uint8_t*>(ws);
  SmallQParams p;
  p.Q = c.Q;
  p.E = c.E;
  p.n = c.n;
  p.d = c.d;
  p.k = c.k;
  p.mask = c.mask;
  p.mask_stride = c.mask_stride;
  p.out = c.out;
  p.guard = c.guard;
  p.cta_cand = reinterpret_cast<TopkCand*>(base);
  p.cta_thr = reinterpret_cast<uint64_t*>(base + align_up((size_t)grid * 2 * kSqCtaKeep * sizeof(TopkCand), 256));
  p.guard_coeff = guard_coeff_stream(c.d);
  const size_t smem = smallq_smem_bytes(c.nq, c.d, grid);
  RPX_REQUIRE(smem <= 160 * 1024, RPX_ERR_UNSUPPORTED, "small-Q top-k: %zu B of shared memory", smem);
  return c.nq == 2 ? launch_its<2>(p, its, grid, smem, c.st, dev.device) : launch_its<1>(p, its, grid, smem, c.st, dev.device);
}

}  // namespace rpx
