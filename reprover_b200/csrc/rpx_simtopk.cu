// rpx_simtopk.cu — fused similarity + top-k, the device half of
// `Corpus.get_nearest_premises` (reference common.py:299-326):
//     similarities = ctx_emb @ premise_emb.T        (:307)
//     argsort(descending) ... first k accessible    (:308-322)
//
// Stage 1  sim_topk (gemm_tc_kernel<..., EpiSimTopk, M_FASTEST>):
//   wgmma of a 128-query block against 128-premise tiles streamed once from HBM
//   by TMA; the [Q, N] score matrix is never written.  Each epilogue thread owns one
//   query row of the accumulator tile, compares its 128 scores against that query's running threshold
//   and appends the few survivors (score, index) to a per-(CTA, query) candidate list.
//   When a list fills up, the warp compacts it: a warp-shuffle bisection finds a
//   threshold that keeps ~KEEP best entries, and the threshold rises.
// Stage 2  select_rescore_kernel (one CTA per query):
//   gathers the query's lists from the CTAs that served its block, selects the KEEP
//   best by (fp32 score, index), re-scores those in fp64 with the canonical summation
//   order (bf16 products are exact in fp64) and emits the k best ordered by
//   (fp64 score desc, index asc) — the ordering contract in include/rpx.h.
// Stage 3  topk_merge_kernel: the k-way merge after the multi-GPU all-gather.
#include <math.h>

#include "rpx_gemm_launch.cuh"
#include "rpx_kernels.cuh"
#include "rpx_topk_common.cuh"

namespace rpx {

namespace {

constexpr int kSimBlockN = 128;
#ifndef RPX_SIM_SAMPLE_TILES
#define RPX_SIM_SAMPLE_TILES 64
#endif
#ifndef RPX_SIM_SEL_SLACK
#define RPX_SIM_SEL_SLACK 16
#endif
constexpr int kSampleTiles = RPX_SIM_SAMPLE_TILES;  // 64 x 128 = 8192 sampled premises
constexpr int kSelSlack = RPX_SIM_SEL_SLACK;        // stage 2 re-scores between n_res and n_res + kSelSlack rows
constexpr unsigned kFull = kFullMask;

// EPL = candidate entries per lane: a list holds CAP = 32*EPL entries and is compacted back to
// about KEEP (<= CAP/2) when it fills.  KEEP is the size of the candidate superset a CTA
// guarantees for its slice of the corpus.
// Stage-1 epilogue parameters (shared by every EpiSimTopk instantiation).
struct SimTopkParams {
  uint2* cand;           // [grid][128][CAP]  (score bits, local index)
  int32_t* cnt;          // [grid][128]
  float* thr_out;        // [grid][128] final pass threshold of each list: nothing above it was ever dropped
  uint32_t* gthr;        // [tiles_m*128] shared per-query threshold (monotone key, atomicMax)
  uint32_t* gmin;        // [tiles_m*128] min over CTAs of their first published rank_r-th best key
  uint32_t* gcnt;        // [tiles_m*128] number of CTAs that have published into gmin
  int n_seg;             // CTAs per query block
  int rank_r;            // ceil(KEEP / n_seg)
  int final_max;         // longest list stage 2 accepts (CAP: no final compaction; else KEEP+SLACK)
  const uint32_t* mask;  // optional access bitmask [nq][mask_stride]
  int64_t mask_stride;
  int nq;
  int n;
  int tiles_m;
};

template <int EPL, int KEEP_>
struct EpiSimTopk {
  static constexpr int CAP = 32 * EPL;
  static constexpr int KEEP = KEEP_;
  static constexpr int SLACK = 16;
  static_assert(KEEP + SLACK + 32 <= CAP, "list too small");
  using Params = SimTopkParams;
  static constexpr size_t kSmemBytes = 0;
  static constexpr int kWarps = 4;  // one warp per lane group: a query's list has one writer

  Params p;
  float thr;        // pass rule: score > thr
  uint2* wptr;      // next free entry of this thread's list
  uint2* buf;       // this thread's (query's) list
  uint2* warp_buf;  // list of lane 0's query; lane l's list is warp_buf + l*CAP
  int q, lane, slot;
  bool active;
  bool published = false;  // this list has contributed to gmin
  bool have_gmin = false;  // the all-CTA bound has been adopted

  __device__ EpiSimTopk(const Params& p_, uint8_t*, int row, int) : p(p_) {
    lane = row & 31;
    const int cta = blockIdx.x;
    q = (cta % p.tiles_m) * kBlockM + row;
    active = q < p.nq;
    thr = -INFINITY;
    warp_buf = p.cand + ((size_t)cta * kBlockM + (row & ~31)) * CAP;
    buf = warp_buf + (size_t)lane * CAP;
    wptr = buf;
    slot = cta * kBlockM + row;
  }
  __device__ __forceinline__ int count() const { return (int)(wptr - buf); }

  // Branch-free conditional append: every lane executes the same three instructions, the store
  // and the pointer bump are predicated.  (A branchy append serialises the warp once per lane
  // that appends, which made the epilogue ~4x slower than the MMA it has to keep up with.)
  __device__ __forceinline__ void append_if_gt(uint32_t bits, uint32_t idx) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.gt.f32 p, %1, %2;\n"
        "@p st.global.v2.b32 [%0], {%3, %4};\n"
        "@p add.s64 %0, %0, 8;\n"
        "}\n"
        : "+l"(wptr)
        : "f"(__uint_as_float(bits)), "f"(thr), "r"(bits), "r"(idx)
        : "memory");
  }
  __device__ __forceinline__ void append_if_gt_masked(uint32_t bits, uint32_t idx, uint32_t bit) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.gt.f32 p, %1, %2;\n"
        "setp.ne.and.u32 p, %5, 0, p;\n"
        "@p st.global.v2.b32 [%0], {%3, %4};\n"
        "@p add.s64 %0, %0, 8;\n"
        "}\n"
        : "+l"(wptr)
        : "f"(__uint_as_float(bits)), "f"(thr), "r"(bits), "r"(idx), "r"(bit)
        : "memory");
  }

  // Loads lane-strided entries [i*32 + lane] of list `b` (count c) into registers.
  __device__ __forceinline__ void load_list(const uint2* b, int c, uint2 (&e)[EPL]) const {
#pragma unroll
    for (int i = 0; i < EPL; ++i) {
      const int pos = i * 32 + lane;
      e[i] = pos < c ? b[pos] : make_uint2(0u, 0u);
    }
  }

  // Largest T with count(key >= T) >= target, by bisection on [lo, hi) with
  // count(>= lo) >= target > count(>= hi).  Returns T and the count at T.
  __device__ __forceinline__ uint32_t kth_key(const uint32_t (&key)[EPL], int c, int target, int slack,
                                              uint64_t lo, uint64_t hi, int count_lo, int* count_out) const {
    while (count_lo > target + slack && hi - lo > 1) {
      const uint32_t mid = (uint32_t)(lo + (hi - lo) / 2);
      int m = 0;
#pragma unroll
      for (int i = 0; i < EPL; ++i) m += (i * 32 + lane < c && key[i] >= mid) ? 1 : 0;
      m = __reduce_add_sync(kFull, m);
      if (m >= target) {
        lo = mid;
        count_lo = m;
      } else {
        hi = mid;
      }
    }
    *count_out = count_lo;
    return (uint32_t)lo;
  }

  // Warp-cooperative compaction of every list in this warp that holds more than `min_count`
  // entries: a bisection over the monotone score keys finds a threshold that keeps between KEEP
  // and KEEP+SLACK entries (exactly KEEP, lowest indices first, when many scores tie).  The next
  // list's entries are fetched while the current one is processed.
  __device__ void compact_warp(int min_count) {
    const int my_cnt = count();
    unsigned todo = __ballot_sync(kFull, my_cnt > min_count);
    if (todo == 0u) return;
    uint2 e[EPL], en[EPL];
    int src = __ffs(todo) - 1;
    todo &= todo - 1;
    int c = __shfl_sync(kFull, my_cnt, src);
    load_list(warp_buf + (size_t)src * CAP, c, e);
    while (src >= 0) {
      const int nsrc = todo ? __ffs(todo) - 1 : -1;
      todo &= todo - 1;
      int cn = 0;
      if (nsrc >= 0) {
        cn = __shfl_sync(kFull, my_cnt, nsrc);
        load_list(warp_buf + (size_t)nsrc * CAP, cn, en);
      }
      uint2* b = warp_buf + (size_t)src * CAP;
      uint32_t key[EPL];
      uint32_t kmin = 0xFFFFFFFFu, kmax = 0u;
#pragma unroll
      for (int i = 0; i < EPL; ++i) {
        if (i * 32 + lane < c) {
          key[i] = fkey(e[i].x);
          kmin = min(kmin, key[i]);
          kmax = max(kmax, key[i]);
        } else {
          key[i] = 0u;
        }
      }
      kmin = __reduce_min_sync(kFull, kmin);
      kmax = __reduce_max_sync(kFull, kmax);
      // invariant: count(key >= lo) = count_lo >= KEEP ; count(key >= hi) < KEEP
      int count_lo;
      const uint32_t lo32 = kth_key(key, c, KEEP, SLACK, kmin, (uint64_t)kmax + 1, c, &count_lo);
      // one-time global bound: the R-th best of this list (R = ceil(KEEP / #CTAs of the block)); once
      // every CTA of the query block has published one, >= KEEP entries exceed their minimum.
      const bool publish = __shfl_sync(kFull, (int)!published, src) != 0;
      uint32_t rth = 0u;
      if (publish) {
        int dummy;
        rth = kth_key(key, c, p.rank_r, 0, lo32, (uint64_t)kmax + 1, count_lo, &dummy);
      }
      const bool tie_mode = count_lo > KEEP + SLACK;  // > SLACK entries share the key `lo`
      int need_eq = 0;
      if (tie_mode) {
        int gt = 0;
#pragma unroll
        for (int i = 0; i < EPL; ++i) gt += (i * 32 + lane < c && key[i] > lo32) ? 1 : 0;
        gt = __reduce_add_sync(kFull, gt);
        need_eq = KEEP - gt;  // > 0 by the invariant (count(>= lo+1) < KEEP)
      }
      const unsigned lt_mask = (1u << lane) - 1u;
      int out = 0, eq_seen = 0;
#pragma unroll
      for (int i = 0; i < EPL; ++i) {
        const bool valid = i * 32 + lane < c;
        bool keep;
        if (tie_mode) {
          // lists are filled in increasing index order, so "first" == lowest index
          const bool eq = valid && key[i] == lo32;
          const unsigned eqb = __ballot_sync(kFull, eq);
          keep = valid && (key[i] > lo32 || (eq && eq_seen + __popc(eqb & lt_mask) < need_eq));
          eq_seen += __popc(eqb);
        } else {
          keep = valid && key[i] >= lo32;
        }
        const unsigned kb = __ballot_sync(kFull, keep);
        if (keep) b[out + __popc(kb & lt_mask)] = e[i];
        out += __popc(kb);
      }
      if (lane == src) {
        wptr = buf + out;
        // pass rule is `score > thr`: ties of `lo` are shut out in tie mode (later ones have
        // higher indices than the KEEP entries held), admitted otherwise.
        const float t_new = __uint_as_float(unkey(tie_mode ? lo32 : lo32 - 1u));
        thr = fmaxf(thr, t_new);
        // This CTA holds >= KEEP entries with key >= lo, so no entry with key < lo can be in the
        // query's global top-KEEP: publish the bound for the other CTAs serving this query block.
        atomicMax(p.gthr + q, lo32 - 1u);
        if (publish) {
          atomicMin(p.gmin + q, rth);
          __threadfence();
          atomicAdd(p.gcnt + q, 1u);
          published = true;
        }
      }
      src = nsrc;
      c = cn;
#pragma unroll
      for (int i = 0; i < EPL; ++i) e[i] = en[i];
    }
    __syncwarp();
  }

  __device__ void before_wait(const TileCtx&) {}
  __device__ void tile(const TileCtx& t) {
    // adopt the best bound any CTA of this query block has published so far
    if (active) {
      uint32_t g = __ldcg(p.gthr + q);
      if (!have_gmin && __ldcg(p.gcnt + q) >= (uint32_t)p.n_seg) {
        __threadfence();
        const uint32_t gm = __ldcg(p.gmin + q);  // every CTA holds >= rank_r entries with key >= gm
        g = max(g, gm - 1u);
        have_gmin = true;
      }
      if (g > fkey(__float_as_uint(thr))) thr = __uint_as_float(unkey(g));
    }
    for (int c = 0; c < t.n_cols; c += 32) {
      // only the lists that are actually about to overflow are compacted: after the warm-up (when
      // all 32 fill together) that is typically a single lane, so the other warps are not held up
      if (__any_sync(kFull, count() > CAP - 32)) compact_warp(CAP - 64);
      uint32_t v[32];
      acc_ld32(t.acc + c, v);
      const int base = t.n0 + c;
      uint32_t word = 0xFFFFFFFFu;
      if (p.mask != nullptr && active) word = p.mask[(size_t)q * p.mask_stride + (base >> 5)];
      if (base + 32 > p.n) word &= (1u << (p.n - base)) - 1u;  // ragged corpus tail (n - base in 1..31)
      if (!active) word = 0u;
      if (__all_sync(kFull, word == 0xFFFFFFFFu)) {
#pragma unroll
        for (int j = 0; j < 32; ++j) append_if_gt(v[j], (uint32_t)(base + j));
      } else if (__any_sync(kFull, word != 0u)) {
#pragma unroll
        for (int j = 0; j < 32; ++j) append_if_gt_masked(v[j], (uint32_t)(base + j), (word >> j) & 1u);
      }
    }
  }

  __device__ void finish() {
    // stage 2 keeps all lists of a query in shared memory: shorten them only if they would not fit
    if (p.final_max < CAP && __any_sync(kFull, count() > p.final_max)) compact_warp(p.final_max);
    p.cnt[slot] = count();
    p.thr_out[slot] = thr;
  }
};

// ------------------------------------------------------------------------------------ stage 0
// Sampling pass: scores of every query against a strided sample of corpus tiles (n_blk_stride > 1)
// are written out ([rows][ld] fp32, -inf where masked / out of range); sample_threshold_kernel
// then takes, per query, the n_res-th best sample score as the starting threshold of stage 1.
// With ~8k sampled premises the main pass admits ~1.4 % of the scores, so its lists hardly ever
// need compacting.  (A threshold from a sample is always valid: at least n_res premises — the
// sampled ones — score at or above it.)
struct EpiSampleScores {
  struct Params {
    float* S;
    int ld;
    const uint32_t* mask;
    int64_t mask_stride;
    int nq;
    int n;
  };
  static constexpr size_t kSmemBytes = 0;
  static constexpr int kWarps = 4;
  Params p;
  __device__ EpiSampleScores(const Params& p_, uint8_t*, int, int) : p(p_) {}
  __device__ void before_wait(const TileCtx&) {}
  __device__ void tile(const TileCtx& t) {
    const int q = t.m0 + t.row;
    const bool active = q < p.nq;
    float* dst = p.S + (size_t)q * p.ld + (size_t)t.n_blk * kSimBlockN;
    for (int c = 0; c < kSimBlockN; c += 32) {
      uint32_t v[32];
      if (c < t.n_cols) {
        acc_ld32(t.acc + c, v);
      }
      const int base = t.n0 + c;
      uint32_t word = 0u;
      if (c < t.n_cols) {
        word = 0xFFFFFFFFu;
        if (p.mask != nullptr && active) word = p.mask[(size_t)q * p.mask_stride + (base >> 5)];
        if (base + 32 > p.n) word &= (1u << (p.n - base)) - 1u;
      }
      if (active) {
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          float4 o;
          o.x = ((word >> (j + 0)) & 1u) ? __uint_as_float(v[j + 0]) : -INFINITY;
          o.y = ((word >> (j + 1)) & 1u) ? __uint_as_float(v[j + 1]) : -INFINITY;
          o.z = ((word >> (j + 2)) & 1u) ? __uint_as_float(v[j + 2]) : -INFINITY;
          o.w = ((word >> (j + 3)) & 1u) ? __uint_as_float(v[j + 3]) : -INFINITY;
          *reinterpret_cast<float4*>(dst + c + j) = o;
        }
      }
    }
  }
  __device__ void finish() {}
};

// One CTA per query: gthr[q] = T - 1 for a key value T with count(sample key >= T) >= n_res (any such T is
// a valid starting bound: that many premises reach it), or 0 when fewer than n_res sampled premises are
// admissible.  T comes from a 1024-bin histogram of the keys between the smallest and the largest valid
// sample key: one pass over the scores, one pass over shared memory, one block scan (instead of the
// dozen block-wide probes of a bisection).  T is the lower edge of the
// bin in which the n_res-th best key falls, so stage 1 admits at most that bin's extra keys.
// The kernel also resets the per-query bookkeeping stage 1 starts from (list counts, final thresholds, the
// shared gmin / gcnt bound) — three memset launches less per call.
struct StageOneReset {
  int32_t* cnt;        // [grid][128]
  float* thr_out;      // [grid][128]: NaN = "no list here", skipped by stage 2's fmaxf reduction
  uint32_t* gcnt;      // [tiles_m * 128]
  uint32_t* gmin;      // [tiles_m * 128]
  int n_seg, tiles_m;
};
constexpr int kThrBins = 1024;
__global__ void __launch_bounds__(256)
sample_threshold_kernel(const float* __restrict__ S, int ld, int n_cols, int n_res, uint32_t* __restrict__ gthr,
                        const StageOneReset rs) {
  {
    const int q = blockIdx.x, q_blk = q / kBlockM, row = q % kBlockM;
    for (int s = threadIdx.x; s < rs.n_seg; s += 256) {
      const int slot = (q_blk + s * rs.tiles_m) * kBlockM + row;
      rs.cnt[slot] = 0;
      rs.thr_out[slot] = __uint_as_float(0xFFFFFFFFu);
    }
    if (threadIdx.x == 0) {
      rs.gcnt[q] = 0u;
      rs.gmin[q] = 0xFFFFFFFFu;
    }
  }
  extern __shared__ __align__(16) uint8_t sm_raw[];
  uint32_t* keys = reinterpret_cast<uint32_t*>(sm_raw);
  __shared__ int hist[kThrBins];
  __shared__ int redi[32];
  __shared__ uint32_t redu[32];
  __shared__ int wsum[8];
  const int q = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t kNegInf = fkey(0xFF800000u);
  uint32_t kmax = 0u, kmin = 0xFFFFFFFFu;
  int valid = 0;
  for (int i = tid; i < kThrBins; i += 256) hist[i] = 0;
  for (int i = tid; i < n_cols; i += 256) {
    const uint32_t k = fkey(__float_as_uint(S[(size_t)q * ld + i]));
    keys[i] = k;
    if (k > kNegInf) {
      ++valid;
      kmax = max(kmax, k);
      kmin = min(kmin, k);
    }
  }
  valid = block_reduce<int>(valid, redi, [](int a, int b) { return a + b; }, 0);
  kmax = block_reduce<uint32_t>(kmax, redu, [](uint32_t a, uint32_t b) { return a > b ? a : b; }, 0u);
  kmin = block_reduce<uint32_t>(kmin, redu, [](uint32_t a, uint32_t b) { return a < b ? a : b; }, 0xFFFFFFFFu);
  if (valid < n_res) {
    if (tid == 0) gthr[q] = 0u;
    return;
  }
  // bin = (key - kmin) >> shift, in [0, kThrBins)
  const uint32_t span = kmax - kmin;
  int shift = 0;
  while ((span >> shift) >= (uint32_t)kThrBins) ++shift;
  for (int i = tid; i < n_cols; i += 256) {
    const uint32_t k = keys[i];
    if (k > kNegInf) atomicAdd(&hist[(k - kmin) >> shift], 1);
  }
  __syncthreads();
  // thread t owns bins [1023 - 4t - 3, 1023 - 4t] (descending): suffix counts from the top bin down
  int mine[4], tot = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    mine[j] = hist[kThrBins - 1 - (4 * tid + j)];
    tot += mine[j];
  }
  int incl = tot;  // inclusive scan over threads (thread 0 = top bins)
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int v = __shfl_up_sync(kFull, incl, off);
    if (lane >= off) incl += v;
  }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  int before = 0;
  for (int w = 0; w < warp; ++w) before += wsum[w];
  incl += before;
  const int excl = incl - tot;
  if (excl < n_res && incl >= n_res) {  // exactly one thread: the n_res-th best key falls in one of its bins
    int c = excl, bin = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (c < n_res && c + mine[j] >= n_res) bin = kThrBins - 1 - (4 * tid + j);
      c += mine[j];
    }
    const uint32_t T = kmin + ((uint32_t)bin << shift);  // lower edge of that bin: count(key >= T) >= n_res
    gthr[q] = T - 1u;
  }
}

// ------------------------------------------------------------------------------------ stage 2

// Threads per query in stage 2: many when few queries are in flight (one query's latency is what
// matters), 256 when there are enough queries to fill the GPU (more CTAs per SM overlap the staging /
// selection / gather phases of different queries).
constexpr int kSelThreadsLatency = 1024, kSelThreadsThroughput = 256, kSelThroughputMinQueries = 512;
constexpr int kSelMax = 288;  // >= largest re-score set (k + margin + selection slack)

__device__ __forceinline__ uint64_t ckey(uint2 e) { return ckey32(e.x, e.y); }

// One CTA per query.  The query's candidate lists (one per stage-1 CTA that served its block,
// each <= list_max entries) are staged in shared memory as 64-bit composite keys; a bisection
// picks the `n_res` best (+ <= 16), which are re-scored in fp64 and ranked exactly.  The exactness
// guard (rpx_topk_common.cuh) then compares the k-th re-scored entry with the best fp32 score any
// row outside the re-scored set can have — the largest final threshold of the query's lists
// (`thr_out`: everything stage 1 dropped scored at or below it) or the selection threshold — and
// flags the query for the exact path when the gap is inside the tensor-core error bound.
struct SelectOut {
  float* scores;
  double* scores64;
  int64_t* idx;
  int32_t* count;
  int64_t* packed;
  int64_t idx_offset;
  GuardOut guard;
  float guard_coeff;
  int q_base;  // number of query 0 of this launch within the call
};

template <int kSelThreads>
__global__ void __launch_bounds__(kSelThreads)
select_rescore_kernel(const uint2* __restrict__ cand, const int32_t* __restrict__ cnt, const float* __restrict__ thr_out,
                      int cap, int list_max, int n_res, int grid_sim, int tiles_m, const __nv_bfloat16* __restrict__ Q,
                      const __nv_bfloat16* __restrict__ E, int d, int k, const SelectOut o) {
  extern __shared__ __align__(16) uint8_t sm_raw[];
  const int n_seg = grid_sim / tiles_m;
  __nv_bfloat16* sq = reinterpret_cast<__nv_bfloat16*>(sm_raw);                                  // [d]
  double* sel_score = reinterpret_cast<double*>(sm_raw + (((size_t)d * 2 + 15) & ~(size_t)15));   // [kSelMax]
  uint32_t* sel_idx = reinterpret_cast<uint32_t*>(sel_score + kSelMax);                            // [kSelMax]
  float* sel_s32 = reinterpret_cast<float*>(sel_idx + kSelMax);                                    // [kSelMax]
  int* seg_off = reinterpret_cast<int*>(sel_s32 + kSelMax);                                        // [n_seg + 1]
  uint64_t* keys = reinterpret_cast<uint64_t*>(
      (reinterpret_cast<uintptr_t>(seg_off + n_seg + 1) + 15) & ~(uintptr_t)15);                   // [n_seg * list_max]
  __shared__ uint64_t red64[32];
  __shared__ float redf[32];
  __shared__ int hist[256];
  __shared__ int sel_bin, sel_above;
  __shared__ int n_sel;
  __shared__ double kth_score;
  __shared__ uint32_t kth_idx;

  const int q = blockIdx.x;
  const int q_blk = q / kBlockM, row = q % kBlockM;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  for (int i = tid; i < d / 8; i += kSelThreads)
    reinterpret_cast<uint4*>(sq)[i] = reinterpret_cast<const uint4*>(Q + (size_t)q * d)[i];
  if (tid == 0) n_sel = 0;
  // list lengths and final thresholds of the query's segments (independent loads, one per thread)
  float tdrop = -INFINITY;
  for (int s = tid; s < n_seg; s += kSelThreads) {
    const int slot = (q_blk + s * tiles_m) * kBlockM + row;
    const int c = cnt[slot];
    seg_off[s + 1] = c < list_max ? c : list_max;  // (stage 1 guarantees c <= list_max)
    tdrop = fmaxf(tdrop, thr_out[slot]);
  }
  tdrop = block_reduce<float>(tdrop, redf, [](float a, float b) { return fmaxf(a, b); }, -INFINITY);
  if (tid == 0) {
    int acc = 0;
    for (int s = 0; s < n_seg; ++s) {
      const int c = seg_off[s + 1];
      seg_off[s] = acc;
      acc += c;
    }
    seg_off[n_seg] = acc;
  }
  __syncthreads();
  const int total = seg_off[n_seg];

  // ---- stage the composite keys
  uint64_t kmin = ~0ull, kmax = 0ull;
  for (int s = warp; s < n_seg; s += kSelThreads / 32) {
    const int slot = (q_blk + s * tiles_m) * kBlockM + row;
    const int o0 = seg_off[s], c = seg_off[s + 1] - o0;
    const uint2* b = cand + (size_t)slot * cap;
    for (int i = lane; i < c; i += 32) {
      const uint64_t key = ckey(b[i]);
      keys[o0 + i] = key;
      kmin = key < kmin ? key : kmin;
      kmax = key > kmax ? key : kmax;
    }
  }
  kmin = block_reduce<uint64_t>(kmin, red64, [](uint64_t a, uint64_t b) { return a < b ? a : b; }, ~0ull);
  kmax = block_reduce<uint64_t>(kmax, red64, [](uint64_t a, uint64_t b) { return a > b ? a : b; }, 0ull);

  // ---- threshold: count(key >= lo) in [n_res, n_res + kSelSlack] (keys are distinct, so it exists).
  // Radix descent over the window [base, win_hi] of the key space that still holds the boundary: 256
  // equal bins, a shared-memory histogram, a warp scan from the top bin down to the bin where the count
  // crosses what is still needed; that bin becomes the next window.  Candidate keys cluster in a narrow
  // score range, so the window is sized from (kmin, kmax) instead of the 64-bit digit positions: two or
  // three levels where a bisection takes ~30 counting rounds.
  uint64_t lo = kmin;
  if (total > n_res + kSelSlack) {
    uint64_t base = kmin, win_hi = kmax;
    int need = n_res;  // keys still to take from the window; everything above the window is taken
    int shift = 64 - __clzll((long long)((kmax - kmin) | 1ull)) - 8;
    shift = shift < 0 ? 0 : shift;
    for (;;) {
      for (int b = tid; b < 256; b += kSelThreads) hist[b] = 0;
      __syncthreads();
      for (int i = tid; i < total; i += kSelThreads) {
        const uint64_t key = keys[i];
        if (key >= base && key <= win_hi) atomicAdd(&hist[(int)((key - base) >> shift)], 1);
      }
      __syncthreads();
      if (warp == 0) {
        // lane l owns bins [8l, 8l + 8); suf = keys in the bins of lanes >= l
        int own = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) own += hist[8 * lane + j];
        int suf = own;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
          const int v = __shfl_down_sync(kFull, suf, off);
          if (lane + off < 32) suf += v;
        }
        // the crossing lane: suf >= need while the lanes above it hold fewer than need
        if (suf >= need && suf - own < need) {
          int above = suf - own, b = 8 * lane + 7;
          for (; b > 8 * lane; --b) {
            if (above + hist[b] >= need) break;
            above += hist[b];
          }
          sel_bin = b;
          sel_above = above;
        }
      }
      __syncthreads();
      const int b = sel_bin, above = sel_above, in_bin = hist[b];
      lo = base + ((uint64_t)b << shift);
      if (above + in_bin <= need + kSelSlack || shift == 0) break;
      need -= above;
      base = lo;
      win_hi = base + ((1ull << shift) - 1ull);
      shift = shift > 8 ? shift - 8 : 0;
      __syncthreads();  // hist / sel_bin are rewritten by the next level
    }
  }
  // ---- collect the selected candidates
  for (int i = tid; i < total; i += kSelThreads) {
    const uint64_t key = keys[i];
    if (key >= lo) {
      const int pos = atomicAdd(&n_sel, 1);
      if (pos < kSelMax) {
        sel_idx[pos] = ckey_idx(key);
        sel_s32[pos] = ckey_score(key);
      }
    }
  }
  __syncthreads();
  int ns = n_sel < kSelMax ? n_sel : kSelMax;

  float q2 = 0.f;
  for (int i = tid; i < d; i += kSelThreads) {
    const float v = __bfloat162float(sq[i]);
    q2 = fmaf(v, v, q2);
  }
  q2 = block_reduce<float>(q2, redf, [](float a, float b) { return a + b; }, 0.f);
  const float eps = guard_eps(o.guard, q2, o.guard_coeff);

  // Two rounds at most.  Round 0 re-scores the n_res best by fp32 score.  If the guard cannot prove that
  // set only because list entries just below the selection threshold might still belong (the common case
  // on ordinary data: a handful of scores within epsilon of the k-th), round 1 takes in every list entry
  // whose fp32 score is within 2 epsilon of the k-th exact score and ranks again — then everything left out
  // is more than epsilon below the k-th.  Only what stage 1 itself dropped (tdrop) needs the exact path.
  float err = 0.f;
  float u = -INFINITY;
  int first_new = 0;
  bool proven = false;
  for (int round = 0; round < 2; ++round) {
    // ---- exact fp64 re-scoring of the candidates added this round, one warp per candidate
    for (int c = first_new + warp; c < ns; c += kSelThreads / 32) {
      const double s = dot64_canonical(sq, E + (size_t)sel_idx[c] * d, d, lane);
      if (lane == 0) {
        sel_score[c] = s;
        err = fmaxf(err, fabsf((float)(s - (double)sel_s32[c])));
      }
    }
    __syncthreads();
    // ---- rank by counting under (score desc, index asc); ranks are a permutation
    for (int c = tid; c < ns; c += kSelThreads) {
      const double sc = sel_score[c];
      const uint32_t ic = sel_idx[c];
      int rank = 0;
      for (int j = 0; j < ns; ++j) {
        const double sj = sel_score[j];
        rank += (sj > sc || (sj == sc && sel_idx[j] < ic)) ? 1 : 0;
      }
      if (rank < k) {
        const size_t oo = (size_t)q * k + rank;
        o.scores[oo] = (float)sc;
        if (o.scores64) o.scores64[oo] = sc;
        o.idx[oo] = (int64_t)ic + o.idx_offset;
        if (o.packed) {
          o.packed[2 * oo] = __double_as_longlong(sc);
          o.packed[2 * oo + 1] = (int64_t)ic + o.idx_offset;
        }
      }
      if (rank == k - 1) {
        kth_score = sc;
        kth_idx = ic;
      }
    }
    __syncthreads();
    u = tdrop;                                             // dropped by a stage-1 threshold / compaction
    if (total > ns) u = fmaxf(u, ckey_score(lo));          // staged but not selected for re-scoring
    proven = guard_proven(k, ns, kth_score, u, eps);
    if (proven || round == 1 || ns < k || total <= ns) break;
    // ---- widen: every staged entry with fp32 score >= kth - 2 eps joins the re-scored set
    const float t_new = __double2float_rd(kth_score - 2.0 * (double)eps);
    if (!(tdrop < t_new)) break;                           // stage 1 dropped rows that close: exact path
    const uint64_t lo2 = (uint64_t)fkey(__float_as_uint(t_new)) << 32;
    if (lo2 >= lo) break;                                  // (cannot happen: kth <= best unselected + eps)
    int extra = 0;
    for (int i = tid; i < total; i += kSelThreads) extra += (keys[i] >= lo2 && keys[i] < lo) ? 1 : 0;
    extra = block_reduce<int>(extra, reinterpret_cast<int*>(redf), [](int a, int b) { return a + b; }, 0);
    if (ns + extra > kSelMax) break;                       // too many near-ties for this buffer: exact path
    first_new = ns;
    for (int i = tid; i < total; i += kSelThreads) {
      const uint64_t key = keys[i];
      if (key >= lo2 && key < lo) {
        const int pos = atomicAdd(&n_sel, 1);
        sel_idx[pos] = ckey_idx(key);
        sel_s32[pos] = ckey_score(key);
      }
    }
    __syncthreads();
    ns = n_sel;
    lo = lo2;
  }

  const int valid = ns < k ? ns : k;
  for (int r = valid + tid; r < k; r += kSelThreads) {
    const size_t oo = (size_t)q * k + r;
    o.scores[oo] = -INFINITY;
    if (o.scores64) o.scores64[oo] = -INFINITY;
    o.idx[oo] = -1;
    if (o.packed) {
      o.packed[2 * oo] = __double_as_longlong(-INFINITY);
      o.packed[2 * oo + 1] = -1;
    }
  }
  err = block_reduce<float>(err, redf, [](float a, float b) { return fmaxf(a, b); }, 0.f);
  if (tid == 0) {
    if (o.count) o.count[q] = valid;
    atomicMax(&o.guard.state->max_err_bits, __float_as_uint(err));
    atomicMax(&o.guard.state->max_eps_bits, __float_as_uint(eps));
    if (!proven) guard_flag(o.guard, o.q_base + q, k, ns, kth_score, kth_idx);
  }
}

// ------------------------------------------------------------------------------------ stage 3
// PACKED: the parts arrive as one [n_parts, nq, k, 2] int64 buffer of (fp64 score bits, index) records —
// exactly what the all-gather of every rank's `out_packed` delivers — instead of two planes.
template <bool PACKED>
__global__ void __launch_bounds__(256)
topk_merge_kernel(const double* __restrict__ scores, const int64_t* __restrict__ idx, int n_parts, int nq, int k,
                  float* __restrict__ out_scores, double* __restrict__ out_scores64, int64_t* __restrict__ out_idx,
                  int32_t* __restrict__ out_count) {
  extern __shared__ __align__(16) uint8_t sm_raw[];
  const int n = n_parts * k;
  double* s = reinterpret_cast<double*>(sm_raw);
  int64_t* ix = reinterpret_cast<int64_t*>(s + n);
  __shared__ int n_valid;
  const int q = blockIdx.x, tid = threadIdx.x;
  if (tid == 0) n_valid = 0;
  __syncthreads();
  int local_valid = 0;
  for (int i = tid; i < n; i += blockDim.x) {
    const int part = i / k, r = i % k;
    const size_t src = ((size_t)part * nq + q) * k + r;
    if (PACKED) {
      const longlong2 rec = reinterpret_cast<const longlong2*>(idx)[src];
      s[i] = __longlong_as_double(rec.x);
      ix[i] = rec.y;
    } else {
      s[i] = scores[src];
      ix[i] = idx[src];
    }
    local_valid += ix[i] >= 0 ? 1 : 0;
  }
  atomicAdd(&n_valid, local_valid);
  __syncthreads();
  // Every part is already sorted under the contract (valid entries first), so the global rank of
  // an entry is its position in its own part plus, for every other part, the number of entries that
  // beat it — found by binary search (R * log2 k steps instead of R * k).
  for (int c = tid; c < n; c += blockDim.x) {
    const int64_t ic = ix[c];
    if (ic < 0) continue;
    const double sc = s[c];
    const int own = c / k;
    int rank = c - own * k;
    for (int p2 = 0; p2 < n_parts; ++p2) {
      if (p2 == own) continue;
      const double* ps = s + p2 * k;
      const int64_t* pi = ix + p2 * k;
      int lo = 0, hi = k;  // first position whose entry does NOT beat (sc, ic)
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        const int64_t im = pi[mid];
        const bool beats = im >= 0 && (ps[mid] > sc || (ps[mid] == sc && im < ic));
        if (beats) lo = mid + 1; else hi = mid;
      }
      rank += lo;
    }
    if (rank < k) {
      const size_t o = (size_t)q * k + rank;
      out_scores[o] = (float)sc;
      if (out_scores64) out_scores64[o] = sc;
      out_idx[o] = ic;
    }
  }
  const int valid = n_valid < k ? n_valid : k;
  for (int r = valid + tid; r < k; r += blockDim.x) {
    const size_t o = (size_t)q * k + r;
    out_scores[o] = -INFINITY;
    if (out_scores64) out_scores64[o] = -INFINITY;
    out_idx[o] = -1;
  }
  if (out_count && tid == 0) out_count[q] = valid;
}

struct SimPlan {
  int epl, cap, keep, list_max, n_res;
  size_t sel_smem;
  int tiles_m, grid;
  size_t cand_bytes, cnt_bytes, gthr_bytes, sample_bytes, total;
  int sample_tiles;  // corpus tiles scored by the sampling pass (0 = no sampling pass)
};

constexpr size_t kSelSmemBudget = 200 * 1024;

size_t sel_smem_bytes(int d, int n_seg, int list_max) {
  return (((size_t)d * 2 + 15) & ~(size_t)15) + kSelMax * (sizeof(double) + sizeof(uint32_t) + sizeof(float)) +
         ((size_t)n_seg + 1) * sizeof(int) + 16 + (size_t)n_seg * list_max * sizeof(uint64_t);
}

int plan_sim(int nq, int k, int d, int num_sms, SimPlan* pl) {
  RPX_REQUIRE(k >= 1 && k <= kFastPathMaxK, RPX_ERR_UNSUPPORTED, "sim_topk: k=%d outside [1, %d]", k, kFastPathMaxK);
  RPX_REQUIRE(nq >= 1, RPX_ERR_INVALID, "sim_topk: nq=%d", nq);
  // per-CTA candidate superset KEEP >= re-score set n_res = k + margin; the margin absorbs most
  // fp32 (tensor-core) vs fp64 rank flips at the k-th place, the guard in stage 2 catches the rest
  pl->n_res = topk_n_res(k);
  pl->keep = k <= 100 ? 128 : 256;
  pl->epl = 16;
  pl->cap = 32 * pl->epl;
  int chunk_q = nq < num_sms * kBlockM ? nq : num_sms * kBlockM;  // queries per launch
  pl->tiles_m = ceil_div(chunk_q, kBlockM);
  int n_seg = num_sms / pl->tiles_m;
  if (n_seg < 1) n_seg = 1;
  // stage 2 keeps one query's lists in shared memory: full-length lists if they fit, else lists
  // compacted to KEEP+16 at the end of stage 1, else fewer stage-1 CTAs per query block
  // (short lists => small stage-2 footprint => several stage-2 CTAs per SM to hide the gather latency)
  pl->list_max = pl->cap;
  while (pl->list_max > pl->keep + 16 && sel_smem_bytes(d, n_seg, pl->list_max) > (size_t)46 << 10) pl->list_max -= 8;
  while (n_seg > 1 && sel_smem_bytes(d, n_seg, pl->list_max) > kSelSmemBudget) --n_seg;
  pl->grid = n_seg * pl->tiles_m;
  pl->sel_smem = sel_smem_bytes(d, n_seg, pl->list_max);
  pl->cand_bytes = align_up((size_t)pl->grid * kBlockM * pl->cap * sizeof(uint2), 256);
  pl->cnt_bytes = align_up((size_t)pl->grid * kBlockM * sizeof(int32_t), 256);  // also the size of thr_out
  pl->gthr_bytes = align_up((size_t)pl->tiles_m * kBlockM * sizeof(uint32_t), 256);
  // sampling pass: up to kSampleTiles tiles of kSimBlockN premises, score matrix capped at 64 MB
  pl->sample_tiles = kSampleTiles;
  while (pl->sample_tiles > 4 &&
         (size_t)pl->tiles_m * kBlockM * pl->sample_tiles * kSimBlockN * sizeof(float) > (size_t)64 << 20)
    pl->sample_tiles /= 2;
  pl->sample_bytes = align_up((size_t)pl->tiles_m * kBlockM * pl->sample_tiles * kSimBlockN * sizeof(float), 256);
  pl->total = pl->cand_bytes + 2 * pl->cnt_bytes + 3 * pl->gthr_bytes + pl->sample_bytes;  // + thr_out; gthr, gmin, gcnt
  return RPX_OK;
}

// Launch of stage 1 with the plan's (fixed) tiles_m / grid.  The A tensor map covers the true
// nq rows, so query rows beyond nq are zero-filled by TMA and flagged inactive in the epilogue.
// `tiles_n_override` / `stride`: visit only tiles 0, stride, 2*stride, ... (the sampling pass).
template <class Epi>
int launch_sim_epi(const __nv_bfloat16* Q, int nq, const __nv_bfloat16* E, int64_t n, int d,
                   const typename Epi::Params& ep, const SimPlan& pl, cudaStream_t st, int tiles_n_override = 0,
                   int stride = 1) {
  using Cfg = GemmCfg<kSimBlockN, kGemmStages>;
  DeviceInfo dev;
  RPX_TRY(get_device_info(&dev));
  CUtensorMap tmA, tmB;
  RPX_TRY(make_tmap_bf16_2d(&tmA, Q, (uint64_t)nq, (uint64_t)d, (uint64_t)d, kBlockM));
  RPX_TRY(make_tmap_bf16_2d(&tmB, E, (uint64_t)n, (uint64_t)d, (uint64_t)d, kSimBlockN));
  const int tiles_n = tiles_n_override > 0 ? tiles_n_override : (int)ceil_div64(n, kSimBlockN);
  const size_t smem = Cfg::smem_bytes(Epi::kSmemBytes);
  auto kern = gemm_tc_kernel<kSimBlockN, kGemmStages, Epi, true>;
  static thread_local int configured_dev = -1;
  if (configured_dev != dev.device) {
    RPX_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured_dev = dev.device;
  }
  int64_t tiles = (int64_t)pl.tiles_m * tiles_n;
  const int grid = tiles < pl.grid ? (int)tiles : pl.grid;  // stays a multiple of tiles_m
  kern<<<grid, gemm_threads<Epi>(), smem, st>>>(tmA, tmB, pl.tiles_m * kBlockM, (int)n, d, pl.tiles_m, tiles_n, stride,
                                                ep, L2Prefetch{nullptr, 0u, grid, nullptr});
  RPX_CUDA_OK(cudaGetLastError());
  return RPX_OK;
}

}  // namespace

size_t mma_topk_workspace_bytes(int nq, int k, int d, int num_sms) {
  SimPlan pl;
  if (plan_sim(nq, k, d, num_sms, &pl) != RPX_OK) return 0;
  return pl.total + 256;
}

// The tensor-core path: [stage 0 sampling pass + threshold] -> stage 1 (fused MMA + top-k epilogue) ->
// stage 2 (select, fp64 re-score, rank, guard).  `ws` is this path's private workspace.
int run_mma_topk(const TopkCall& c, void* ws, size_t ws_bytes) {
  const int nq = c.nq, d = c.d, k = c.k;
  const int64_t n = c.n;
  RPX_REQUIRE(n >= 0 && n < (int64_t)INT32_MAX - 512, RPX_ERR_UNSUPPORTED, "sim_topk: n=%lld out of range", (long long)n);
  RPX_REQUIRE(d > 0 && d % 64 == 0 && d <= 8192, RPX_ERR_UNSUPPORTED, "sim_topk: d=%d must be a multiple of 64 (<= 8192)", d);
  DeviceInfo dev;
  RPX_TRY(get_device_info(&dev));
  SimPlan pl;
  RPX_TRY(plan_sim(nq, k, d, dev.num_sms, &pl));
  RPX_REQUIRE(pl.total <= ws_bytes, RPX_ERR_WORKSPACE, "sim_topk: workspace %zu < %zu", ws_bytes, pl.total);
  RPX_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255) == 0, RPX_ERR_INVALID, "workspace must be 256-byte aligned");
  cudaStream_t st = c.st;
  uint8_t* base = static_cast<uint8_t*>(ws);
  uint2* cand = reinterpret_cast<uint2*>(base);
  float* thr_out = reinterpret_cast<float*>(base + pl.cand_bytes);
  int32_t* cnt = reinterpret_cast<int32_t*>(base + pl.cand_bytes + pl.cnt_bytes);
  uint32_t* gthr = reinterpret_cast<uint32_t*>(base + pl.cand_bytes + 2 * pl.cnt_bytes);
  uint32_t* gcnt = gthr + pl.gthr_bytes / 4;
  uint32_t* gmin = gcnt + pl.gthr_bytes / 4;
  float* sample = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(gmin) + pl.gthr_bytes);
  const int n_seg = pl.grid / pl.tiles_m;
  const int rank_r = ceil_div(pl.keep, n_seg);
  const __nv_bfloat16* Q = c.Q;
  const __nv_bfloat16* E = c.E;
  static thread_local int sel_configured = -1;
  if (sel_configured != dev.device) {
    RPX_CUDA_OK(cudaFuncSetAttribute(select_rescore_kernel<kSelThreadsLatency>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kSelSmemBudget + 8 * 1024)));
    RPX_CUDA_OK(cudaFuncSetAttribute(select_rescore_kernel<kSelThreadsThroughput>,
                                     cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kSelSmemBudget + 8 * 1024)));
    sel_configured = dev.device;
  }
  const int chunk_q = pl.tiles_m * kBlockM;
  for (int q0 = 0; q0 < nq; q0 += chunk_q) {
    const int nq_c = nq - q0 < chunk_q ? nq - q0 : chunk_q;
    // (only the last chunk can be smaller; its tiles_m may shrink but the plan's grid stays valid
    //  because we keep tiles_m fixed and let the surplus query blocks be empty)
    const uint32_t* mask_c = c.mask ? c.mask + (size_t)q0 * c.mask_stride : nullptr;
    const int64_t tiles_n_all = ceil_div64(n, kSimBlockN);
    if (tiles_n_all >= 4 * (int64_t)pl.sample_tiles) {
      // stage 0: starting thresholds from a strided sample of the corpus (writes gthr, resets the rest)
      const int ld = pl.sample_tiles * kSimBlockN;
      EpiSampleScores::Params sp{sample, ld, mask_c, c.mask_stride, nq_c, (int)n};
      RPX_TRY((launch_sim_epi<EpiSampleScores>(Q + (size_t)q0 * d, nq_c, E, n, d, sp, pl, st, pl.sample_tiles,
                                                (int)(tiles_n_all / pl.sample_tiles))));
      const StageOneReset rs{cnt, thr_out, gcnt, gmin, n_seg, pl.tiles_m};
      sample_threshold_kernel<<<nq_c, 256, (size_t)ld * sizeof(uint32_t), st>>>(sample, ld, ld, pl.n_res, gthr, rs);
      RPX_CUDA_OK(cudaGetLastError());
    } else {
      // small corpus, no sampling pass: plain resets.  Lists no stage-1 CTA visits keep count 0 and must not
      // contribute a threshold: 0xFF bytes are a NaN, which the fmaxf() reduction in stage 2 skips
      RPX_CUDA_OK(cudaMemsetAsync(cnt, 0, pl.cnt_bytes + 2 * pl.gthr_bytes, st));  // cnt, gthr, gcnt are adjacent
      RPX_CUDA_OK(cudaMemsetAsync(gmin, 0xFF, pl.gthr_bytes, st));
      RPX_CUDA_OK(cudaMemsetAsync(thr_out, 0xFF, pl.cnt_bytes, st));
    }
    if (n > 0) {
      SimTopkParams ep{cand, cnt, thr_out, gthr, gmin, gcnt, n_seg, rank_r, pl.list_max, mask_c, c.mask_stride, nq_c, (int)n, pl.tiles_m};
      if (pl.keep == 128) {
        RPX_TRY((launch_sim_epi<EpiSimTopk<16, 128>>(Q + (size_t)q0 * d, nq_c, E, n, d, ep, pl, st)));
      } else {
        RPX_TRY((launch_sim_epi<EpiSimTopk<16, 256>>(Q + (size_t)q0 * d, nq_c, E, n, d, ep, pl, st)));
      }
    }
    SelectOut so;
    so.scores = c.out_scores + (size_t)q0 * k;
    so.scores64 = c.out_scores64 ? c.out_scores64 + (size_t)q0 * k : nullptr;
    so.idx = c.out_idx + (size_t)q0 * k;
    so.count = c.out_count ? c.out_count + q0 : nullptr;
    so.packed = c.out_packed ? c.out_packed + (size_t)q0 * k * 2 : nullptr;
    so.idx_offset = c.idx_offset;
    so.guard.state = c.state;
    so.guard.flagged = c.flagged;
    so.guard.bounds = c.bounds;
    so.guard_coeff = guard_coeff_mma(d);
    so.q_base = q0;
    if (nq_c >= kSelThroughputMinQueries) {
      select_rescore_kernel<kSelThreadsThroughput><<<nq_c, kSelThreadsThroughput, pl.sel_smem, st>>>(
          cand, cnt, thr_out, pl.cap, pl.list_max, pl.n_res, pl.grid, pl.tiles_m, Q + (size_t)q0 * d, E, d, k, so);
    } else {
      select_rescore_kernel<kSelThreadsLatency><<<nq_c, kSelThreadsLatency, pl.sel_smem, st>>>(
          cand, cnt, thr_out, pl.cap, pl.list_max, pl.n_res, pl.grid, pl.tiles_m, Q + (size_t)q0 * d, E, d, k, so);
    }
    RPX_CUDA_OK(cudaGetLastError());
  }
  return RPX_OK;
}

int launch_topk_merge(const double* d_scores64, const int64_t* d_idx_or_packed, bool packed, int n_parts, int nq, int k,
                      float* d_out_scores, double* d_out_scores64, int64_t* d_out_idx, int32_t* d_out_count,
                      cudaStream_t st) {
  RPX_REQUIRE(n_parts >= 1 && nq >= 1 && k >= 1, RPX_ERR_INVALID, "rpx_topk_merge: bad sizes");
  const size_t smem = (size_t)n_parts * k * 16;
  RPX_REQUIRE(smem <= 96 * 1024, RPX_ERR_UNSUPPORTED, "rpx_topk_merge: n_parts*k=%d too large", n_parts * k);
  DeviceInfo dev;
  RPX_TRY(get_device_info(&dev));
  static thread_local int configured = -1;
  if (configured != dev.device) {
    RPX_CUDA_OK(cudaFuncSetAttribute(topk_merge_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    RPX_CUDA_OK(cudaFuncSetAttribute(topk_merge_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    configured = dev.device;
  }
  if (packed)
    topk_merge_kernel<true><<<nq, 256, smem, st>>>(nullptr, d_idx_or_packed, n_parts, nq, k, d_out_scores, d_out_scores64,
                                                   d_out_idx, d_out_count);
  else
    topk_merge_kernel<false><<<nq, 256, smem, st>>>(d_scores64, d_idx_or_packed, n_parts, nq, k, d_out_scores,
                                                    d_out_scores64, d_out_idx, d_out_count);
  RPX_CUDA_OK(cudaGetLastError());
  return RPX_OK;
}

}  // namespace rpx
