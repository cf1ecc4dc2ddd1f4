// rpx_gemm.cuh — the wgmma / TMA contraction core shared by the encoder GEMMs and the
// similarity kernel.
//
//   D[M, N] (fp32) = A[M, K] * B[N, K]^T        A, B bf16, K contiguous
//
// Structure (one persistent CTA per SM, 160 + 32 * Epi::kWarps threads):
//   warps 0-3   : MMA warpgroup  — wgmma.mma_async (M = 64 per instruction, one instruction per
//                 64-row half of the tile, N = BLOCK_N, K = 16) x4 per stage, the fp32 accumulator in
//                 registers; a stage goes back to the producer (`empty[]`) once the wgmma group that read
//                 it has retired.  After the last k-block the accumulator is written to a shared-memory
//                 tile (`acc`, one row of BLOCK_N floats per output row) and published (`tfull`).
//   warp 4      : TMA producer   — cp.async.bulk.tensor A/B tiles into a STAGES-deep
//                 128B-swizzled shared-memory ring, completion on `full[]` mbarriers
//   warps 5..   : epilogue       — read the accumulator tile (one row per thread) and run the fused
//                 epilogue functor; `tempty` hands the tile back.  The MMA warpgroup runs the mainloop of
//                 tile i+1 while the epilogue works on tile i; it only waits for `tempty` before it writes
//                 the next accumulator.
//
// `n_blk_stride` > 1 makes the kernel visit only every stride-th B tile (the similarity
// kernel's sampling pass); it is 1 everywhere else.
//
// Tiles are visited in n-fastest order so that concurrently resident CTAs share
// the same A row-block through L2 (the B operand — the weights — is small and
// L2-resident).  The similarity kernel uses M_FASTEST instead: A is the (small)
// query block, B the streamed corpus, and a grid that is a multiple of tiles_m
// pins every CTA to one query block for its whole life.
//
// The reference has no counterpart: it calls torch `@` / nn.Linear (cuBLAS) —
// SURVEY.md §2.1 K3/K8/K9/K11.
#pragma once
#include "rpx_ptx.cuh"

namespace rpx {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;  // 64 bf16 = 128 B = one swizzle atom row
constexpr int kMmaK = 16;
#ifndef RPX_EPI_WARPS
#define RPX_EPI_WARPS 4
#endif
constexpr int kMmaThreads = 128;  // warps 0-3: the MMA warpgroup
constexpr int kProducerWarp = 4;
constexpr int kEpiWarp0 = 5;      // first epilogue warp
// threads of a launch: MMA warpgroup + TMA warp + Epi::kWarps epilogue warps (4 or 8)
template <class Epi>
constexpr int gemm_threads() { return kMmaThreads + 32 + 32 * Epi::kWarps; }

template <int BLOCK_N, int STAGES, int BM = kBlockM>
struct GemmCfg {
  static_assert(BM == 64 || BM == 128, "tile rows: one or two 64-row wgmma blocks");
  static_assert(BLOCK_N == 64 || BLOCK_N == 128, "wgmma N of a tile: 64 or 128");
  static_assert(2 * STAGES + 2 <= 30, "barrier block holds at most 14 stages");
  static constexpr int kABytes = BM * kBlockK * 2;
  static constexpr int kBBytes = BLOCK_N * kBlockK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  // accumulator tile: BM rows of BLOCK_N floats, rows padded by 4 floats so that the eight rows a
  // quarter-warp reads at once (16 B each) fall into distinct banks
  static constexpr int kAccStride = BLOCK_N + 4;
  static constexpr int kAccBytes = BM * kAccStride * 4;
  // ring + accumulator + 1 KB alignment slack + barriers
  static constexpr int kBarBytes = 256;
  static constexpr size_t smem_bytes(size_t epi_extra) {
    return (size_t)STAGES * kStageBytes + kAccBytes + 1024 + kBarBytes + epi_extra;
  }
};

// Kernel argument of gemm_tc_kernel: CTAs [0, work_ctas) run the GEMM (persistent over the tiles with that
// stride); CTAs beyond prefetch `bytes` at `ptr` into L2 and leave.  work_ctas == gridDim.x: no helpers.
struct L2Prefetch {
  const void* ptr;
  uint32_t bytes;
  int work_ctas;
  unsigned long long* timeline;  // debug (rpx_debug_set_timeline): 8 %globaltimer stamps of CTA 0, or null
};

RPX_DEVICE unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define RPX_STAMP(pf, i)                                                   \
  do {                                                                     \
    if ((pf).timeline != nullptr && blockIdx.x == 0) (pf).timeline[i] = global_ns(); \
  } while (0)

// What an epilogue functor sees for one output tile.
struct TileCtx {
  const float* acc;  // this thread's row of the accumulator tile (shared memory), column 0
  int m0, n0;      // tile origin in the output
  int n_cols;      // valid columns in this tile (multiple of 32)
  int row;         // this thread's row inside the tile, 0..127
  int m_blk, n_blk;
  int M, N;
  int next_m0, next_n0;  // origin of the next tile this CTA will process (next_m0 < 0: none)
  int next_cols;         // its width
  int part, split;       // this warp handles the 32-column chunks with (chunk % split) == part
  int rows_per_warp;     // tile rows held by one lane group: 32 (M = 128 tiles) or 16 (M = 64: lanes 16-31 idle)
};

// 32 consecutive accumulator columns of this thread's row.
RPX_DEVICE void acc_ld32(const float* src, uint32_t (&v)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 x = reinterpret_cast<const float4*>(src)[i];
    v[4 * i] = __float_as_uint(x.x);
    v[4 * i + 1] = __float_as_uint(x.y);
    v[4 * i + 2] = __float_as_uint(x.z);
    v[4 * i + 3] = __float_as_uint(x.w);
  }
}

// Epi must provide:
//   struct Params;                       (trivially copyable kernel argument)
//   static constexpr size_t kSmemBytes;  (extra dynamic shared memory, may be 0)
//   static constexpr int kWarps;         (4 or 8 epilogue warps; with 8, two warps share a lane
//                                         group and split the tile's 32-column chunks between them)
//   __device__ Epi(const Params&, uint8_t* smem_extra, int row /*tile row this thread owns, 0..127*/,
//                  int part /*column share of this warp, 0..kWarps/4-1*/);
//   __device__ void before_wait(const TileCtx&);  (work that may run while the MMAs of this tile are
//                                                  still in flight, e.g. prefetching)
//   __device__ void tile(const TileCtx&);     (all epilogue threads, warp-converged)
//   __device__ void finish();
// SPLIT_B (the gated FFN up-projection): the B tile is two boxes of BLOCK_N/2 rows — the gate rows and the
// linear-branch rows of the same BLOCK_N/2 hidden units.  The packed weight interleaves wi_0 / wi_1 in
// 128-row blocks (rows [256j, 256j+128) gate, [256j+128, 256j+256) linear, see rpx_encoder.cu), so n-tile t
// (units u0 = t * BLOCK_N/2) takes rows 256 (u0/128) + u0 % 128 and the same + 128; tmB must then be encoded
// with a box of BLOCK_N/2 rows.
//
// PAIR: the kernel runs as clusters of two CTAs that work in lockstep on vertically adjacent tiles — the same
// n-tile, m-tiles 2j and 2j+1 — and share the B tile: each CTA's producer loads one half of it (BLOCK_N/2 rows,
// tmB encoded with that box) and multicasts it into both CTAs, so every B byte crosses L2 once per pair.  A
// stage is refilled only after the MMA warpgroups of BOTH CTAs have released it (the empty barriers count the
// peer's arrivals too), since the refill writes into the peer's shared memory as well.  Grid = 2 x pairs.
//
// BM = 64 (latency path): 64-row tiles, one wgmma row block.  An epilogue warp then owns 16 rows (row r of the
// tile belongs to lane r % 16 of lane group r / 16) and its upper 16 lanes idle.  A CTA takes in half the
// activation bytes per k-block and the ring holds more stages — what a narrow GEMM's time is made of (see
// rpx_encoder.cu).
template <int BLOCK_N, int STAGES, class Epi, bool M_FASTEST = false, bool SPLIT_B = false, int BM = kBlockM,
          bool PAIR = false>
__global__ void __launch_bounds__(gemm_threads<Epi>(), 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               int M, int N, int K, int tiles_m, int tiles_n, int n_blk_stride, typename Epi::Params ep,
               L2Prefetch pf) {
  using Cfg = GemmCfg<BLOCK_N, STAGES, BM>;
  constexpr int kSub = BM / 64;  // 64-row wgmma blocks per tile
  static_assert(!PAIR || (!M_FASTEST && !SPLIT_B), "paired tiles: plain n-fastest order, one B box per CTA");
  if (threadIdx.x == 0) RPX_STAMP(pf, 0);
  if ((int)blockIdx.x >= pf.work_ctas) {
    // Helper CTA (latency path): the GEMM itself keeps only a fraction of the SMs busy, so the launch is
    // widened to the whole GPU and the surplus CTAs pull the NEXT layer's weights into L2 while this
    // layer computes — its GEMMs then stream their B operand at L2 instead of DRAM latency.
    pdl_launch_dependents();
    const int n_help = (int)gridDim.x - pf.work_ctas;
    const size_t lines = ((size_t)pf.bytes + 127) >> 7;
    const char* base = static_cast<const char*>(pf.ptr);
    for (size_t i = (size_t)((int)blockIdx.x - pf.work_ctas) * blockDim.x + threadIdx.x; i < lines;
         i += (size_t)n_help * blockDim.x)
      asm volatile("prefetch.global.L2 [%0];" ::"l"(base + (i << 7)));
    return;
  }
  extern __shared__ uint8_t smem_raw[];
  // 128B swizzle needs 1024-byte aligned tile bases.
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024 - (raw_addr & 1023)) & 1023);
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * Cfg::kABytes;
  float* sAcc = reinterpret_cast<float*>(smem + STAGES * Cfg::kStageBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::kStageBytes + Cfg::kAccBytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + STAGES;
  uint64_t* tfull = bars + 2 * STAGES;
  uint64_t* tempty = bars + 2 * STAGES + 1;
  uint8_t* smem_extra = smem + STAGES * Cfg::kStageBytes + Cfg::kAccBytes + Cfg::kBarBytes;

  const int warp = threadIdx.x >> 5;
  const int num_kb = K / kBlockK;
  // Work units: tiles, or (PAIR) tile pairs; this CTA takes units unit0, unit0 + unit_step, ...
  const uint32_t rank = PAIR ? cluster_ctarank() : 0u;
  const int num_units = PAIR ? ((tiles_m + 1) / 2) * tiles_n : tiles_m * tiles_n;
  const int unit0 = PAIR ? (int)blockIdx.x >> 1 : (int)blockIdx.x;
  const int unit_step = PAIR ? pf.work_ctas >> 1 : pf.work_ctas;
  auto unit_m = [&](int u) { return PAIR ? 2 * (u / tiles_n) + (int)rank : (M_FASTEST ? u % tiles_m : u / tiles_n); };
  auto unit_n = [&](int u) { return PAIR ? u % tiles_n : (M_FASTEST ? u / tiles_m : u % tiles_n); };

  if (warp == kProducerWarp) {
    if (elect_one()) {
      tma_prefetch_desc(&tmA);
      tma_prefetch_desc(&tmB);
      for (int s = 0; s < STAGES; ++s) {
        mbar_init(&full[s], 1);
        mbar_init(&empty[s], PAIR ? 2 * kMmaThreads : kMmaThreads);
      }
      mbar_init(tfull, kMmaThreads);
      mbar_init(tempty, 32 * Epi::kWarps);
      fence_mbar_init();
    }
    __syncwarp();
  }
  __syncthreads();
  if (PAIR) cluster_sync_all();  // the peer's barriers are initialised before anything multicasts or arrives on them
  // Everything above touched only this CTA's shared memory.  Under programmatic dependent launch
  // (rpx_ptx.cuh) the preceding kernel may still be running: the A operand and whatever the epilogue reads
  // from global memory are its outputs and must wait for it (pdl_wait), but the B operand — the weights —
  // is never written by a kernel of the chain, so the producer streams the first ring's worth of B tiles
  // BEFORE it waits: by the time the predecessor retires, part of this CTA's weights are already on chip.
  pdl_launch_dependents();
  if (threadIdx.x == 0) RPX_STAMP(pf, 1);

  if (warp == kProducerWarp) {
    // ------------------------------------------------------------------ TMA producer
    if (elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      int pre = 0;  // stages of the first tile whose barrier is armed and whose B tile is already in flight
      auto load_b = [&](int st, int n_blk, int kb) {
        if (M_FASTEST) {
          tma_load_2d_hint(sB + st * Cfg::kBBytes, &tmB, &full[st], kb * kBlockK, n_blk * n_blk_stride * BLOCK_N, kEvictFirst);
        } else if (PAIR) {
          constexpr int H = BLOCK_N / 2;
          tma_load_2d_multicast(sB + st * Cfg::kBBytes + rank * H * kBlockK * 2, &tmB, &full[st], kb * kBlockK,
                                n_blk * BLOCK_N + (int)rank * H, (uint16_t)0x3);
        } else if (SPLIT_B) {
          constexpr int H = BLOCK_N / 2;
          const int u0 = n_blk * H;
          const int gate_row = (u0 / 128) * 256 + (u0 % 128);
          tma_load_2d(sB + st * Cfg::kBBytes, &tmB, &full[st], kb * kBlockK, gate_row);
          tma_load_2d(sB + st * Cfg::kBBytes + H * kBlockK * 2, &tmB, &full[st], kb * kBlockK, gate_row + 128);
        } else {
          tma_load_2d(sB + st * Cfg::kBBytes, &tmB, &full[st], kb * kBlockK, n_blk * n_blk_stride * BLOCK_N);
        }
      };
      if (!M_FASTEST && !PAIR && unit0 < num_units) {
        const int n_blk0 = unit_n(unit0);
        pre = num_kb < STAGES ? num_kb : STAGES;
        for (int kb = 0; kb < pre; ++kb) {  // fresh barriers: every stage is free
          mbar_arrive_expect_tx(&full[kb], Cfg::kStageBytes);
          load_b(kb, n_blk0, kb);
        }
      }
      pdl_wait();
      RPX_STAMP(pf, 2);
      for (int u = unit0; u < num_units; u += unit_step) {
        const int n_blk = unit_n(u);
        const int m_blk = unit_m(u);
        for (int kb = 0; kb < num_kb; ++kb) {
          if (pre > 0) {
            --pre;  // armed, B in flight: only the A tile is missing
          } else {
            mbar_wait(&empty[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full[stage], Cfg::kStageBytes);
            load_b(stage, n_blk, kb);
          }
          // L2 eviction hints for the similarity kernel: the streamed operand (corpus) evict-first, the
          // re-used operand (query block, re-read by every tile) evict-last.
          if (M_FASTEST) {
            tma_load_2d_hint(sA + stage * Cfg::kABytes, &tmA, &full[stage], kb * kBlockK, m_blk * BM, kEvictLast);
          } else {
            tma_load_2d(sA + stage * Cfg::kABytes, &tmA, &full[stage], kb * kBlockK, m_blk * BM);
          }
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else if (warp < kProducerWarp) {
    // ------------------------------------------------------------------ MMA warpgroup
    const int lane = threadIdx.x & 31;
    float acc[kSub][BLOCK_N / 2];
    int stage = 0;
    uint32_t phase = 0;
    uint32_t tphase = 0;
    auto release = [&](int st) {
      mbar_arrive(&empty[st]);
      if (PAIR) mbar_arrive_cluster(&empty[st], rank ^ 1u);
    };
    for (int u = unit0; u < num_units; u += unit_step) {
      int prev = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full[stage], phase);
        if (kb == 0 && u == unit0 && threadIdx.x == 0) RPX_STAMP(pf, 3);
        const uint64_t a_desc = make_smem_desc_kmajor_sw128(smem_u32(sA + stage * Cfg::kABytes));
        const uint64_t b_desc = make_smem_desc_kmajor_sw128(smem_u32(sB + stage * Cfg::kBBytes));
#pragma unroll
        for (int s = 0; s < kSub; ++s) wgmma_fence_operand(acc[s]);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / kMmaK; ++k) {
#pragma unroll
          for (int s = 0; s < kSub; ++s) {
            // +32 bytes (>>4 = 2) per K=16 step inside the swizzle atom; +8 KB (>>4 = 512) per 64 A rows
            if constexpr (BLOCK_N == 128)
              wgmma_m64n128k16_ss(acc[s], a_desc + 512 * s + 2 * k, b_desc + 2 * k, (kb | k) != 0);
            else
              wgmma_m64n64k16_ss(acc[s], a_desc + 512 * s + 2 * k, b_desc + 2 * k, (kb | k) != 0);
          }
        }
        wgmma_commit();
        // the group of the previous k-block has retired once at most this one is in flight: its stage is free
        if (kb > 0) {
          wgmma_wait<1>();
          release(prev);
        }
        prev = stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int s = 0; s < kSub; ++s) wgmma_fence_operand(acc[s]);
      release(prev);
      if (u == unit0 && threadIdx.x == 0) RPX_STAMP(pf, 4);
      // accumulator -> shared memory, once the epilogue has finished reading the previous tile
      mbar_wait(tempty, tphase ^ 1);
      const int r0 = (warp * 16 + (lane >> 2)) * Cfg::kAccStride + 2 * (lane & 3);
#pragma unroll
      for (int s = 0; s < kSub; ++s) {
        float* dst = sAcc + s * 64 * Cfg::kAccStride + r0;
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(acc[s][4 * j], acc[s][4 * j + 1]);
          *reinterpret_cast<float2*>(dst + 8 * Cfg::kAccStride + 8 * j) = make_float2(acc[s][4 * j + 2], acc[s][4 * j + 3]);
        }
      }
      mbar_arrive(tfull);
      tphase ^= 1;
    }
  } else {
    // ------------------------------------------------------------------ epilogue
    const int lane_grp = (warp - kEpiWarp0) & 3;              // which 32 (or 16) rows of the tile
    const int lane = threadIdx.x & 31;
    // row of the tile this thread owns; with 64-row tiles lanes 16-31 of a group hold nothing: their row lies
    // beyond every matrix, so the functors' `m < M` tests switch them off (they read a duplicate row)
    const int row = BM == kBlockM ? lane_grp * 32 + lane : (lane < 16 ? lane_grp * 16 + lane : (1 << 28));
    const int acc_row = BM == kBlockM ? lane_grp * 32 + lane : lane_grp * 16 + (lane & 15);
    const int part = (warp - kEpiWarp0) >> 2;                 // which share of the columns (0 when 4 warps)
    pdl_wait();  // the epilogue reads (row scales, residual stream) and overwrites the predecessor's outputs
    Epi epi(ep, smem_extra, lane_grp * 32 + lane, part);      // (the functor's staging is per lane group)
    uint32_t tphase = 0;
    for (int u = unit0; u < num_units; u += unit_step) {
      TileCtx t;
      t.n_blk = unit_n(u);
      t.m_blk = unit_m(u);
      t.m0 = t.m_blk * BM;
      t.rows_per_warp = BM / 4;
      t.n0 = t.n_blk * n_blk_stride * BLOCK_N;  // (n_blk stays the logical tile index)
      int n_this = N - t.n0;
      if (n_this > BLOCK_N) n_this = BLOCK_N;
      t.n_cols = n_this;
      t.row = row;
      t.part = part;
      t.split = Epi::kWarps / 4;
      t.M = M;
      t.N = N;
      t.acc = sAcc + acc_row * Cfg::kAccStride;
      {
        const int nu = u + unit_step;
        if (nu < num_units) {
          t.next_m0 = unit_m(nu) * BM;
          t.next_n0 = unit_n(nu) * BLOCK_N;
          t.next_cols = N - t.next_n0 < BLOCK_N ? N - t.next_n0 : BLOCK_N;
        } else {
          t.next_m0 = -1;
          t.next_n0 = 0;
          t.next_cols = 0;
        }
      }
      epi.before_wait(t);
      mbar_wait(tfull, tphase);
      if (threadIdx.x == 32 * kEpiWarp0 && u == unit0) RPX_STAMP(pf, 5);
      epi.tile(t);
      if (threadIdx.x == 32 * kEpiWarp0 && u == unit0) RPX_STAMP(pf, 6);
      mbar_arrive(tempty);
      tphase ^= 1;
    }
    epi.finish();
  }

  __syncthreads();
  // the peer may still multicast into this CTA's ring or arrive on its barriers until it is done too
  if (PAIR) cluster_sync_all();
  if (threadIdx.x == 0) RPX_STAMP(pf, 7);
}

// ============================================================================ epilogues

// Row scale shared by the epilogues that consume an RMSNorm'd operand: the
// RMSNorm weight is folded into the GEMM's B operand at load time, so all that
// is left is rs[m] = rsqrt(mean_k(x[m,k]^2) + eps), applied to the fp32 accumulator.
// sumsq is delivered as `n_parts` partial sums per row (written by the producing
// epilogue, one per output n-block), summed here in a fixed order -> deterministic.
struct RowScale {
  const float* ss_parts;  // [n_parts][M] or nullptr (scale 1)
  int n_parts;
  int part_stride;        // elements between parts (>= M)
  float inv_dim;          // 1 / d_model
  float eps;
  __device__ float get(int m) const {
    if (ss_parts == nullptr) return 1.0f;
    float s = 0.f;
    // loads in batches of 24 (independent, all in flight together), additions in part order: the latency
    // path has 46 parts per row and would pay one L2 round trip per part with a plain loop
    constexpr int kBatch = 24;
    for (int p = 0; p < n_parts; p += kBatch) {
      float v[kBatch];
#pragma unroll
      for (int j = 0; j < kBatch; ++j) v[j] = p + j < n_parts ? ss_parts[(size_t)(p + j) * part_stride + m] : 0.f;
#pragma unroll
      for (int j = 0; j < kBatch; ++j)
        if (p + j < n_parts) s += v[j];
    }
    return rsqrtf(s * inv_dim + eps);
  }
};

// C[m, n] = acc (fp32).  Generic; used by tests.
struct EpiStoreF32 {
  struct Params {
    float* C;
    int ldc;
  };
  static constexpr size_t kSmemBytes = 0;
  static constexpr int kWarps = RPX_EPI_WARPS;
  Params p;
  __device__ EpiStoreF32(const Params& p_, uint8_t*, int, int) : p(p_) {}
  __device__ void before_wait(const TileCtx&) {}
  __device__ void tile(const TileCtx& t) {
    const int m = t.m0 + t.row;
    const bool ok = m < t.M;
    for (int c = 32 * t.part; c < t.n_cols; c += 32 * t.split) {
      uint32_t v[32];
      acc_ld32(t.acc + c, v);
      if (ok) {
        float4* dst = reinterpret_cast<float4*>(p.C + (size_t)m * p.ldc + t.n0 + c);
#pragma unroll
        for (int i = 0; i < 8; ++i)
          dst[i] = make_float4(__uint_as_float(v[4 * i]), __uint_as_float(v[4 * i + 1]),
                               __uint_as_float(v[4 * i + 2]), __uint_as_float(v[4 * i + 3]));
      }
    }
  }
  __device__ void finish() {}
};

// C[m, n] = bf16(acc * rs[m]).  QKV projection (RMSNorm folded: prologue of K3).
struct EpiStoreBF16 {
  struct Params {
    __nv_bfloat16* C;
    int ldc;
    RowScale rs;
  };
  static constexpr size_t kSmemBytes = 0;
  static constexpr int kWarps = RPX_EPI_WARPS;
  Params p;
  float rs = 0.f;  // this thread's row scale for the tile in flight
  __device__ EpiStoreBF16(const Params& p_, uint8_t*, int, int) : p(p_) {}
  // the row scale does not depend on the accumulator: its partial sums (up to 23 L2 round trips on the latency
  // path) are fetched while the MMAs of the tile are still running
  __device__ void before_wait(const TileCtx& t) {
    const int m = t.m0 + t.row;
    rs = m < t.M ? p.rs.get(m) : 0.f;
  }
  __device__ void tile(const TileCtx& t) {
    const int m = t.m0 + t.row;
    const bool ok = m < t.M;
    for (int c = 32 * t.part; c < t.n_cols; c += 32 * t.split) {
      uint32_t v[32];
      acc_ld32(t.acc + c, v);
      if (ok) {
        uint4* dst = reinterpret_cast<uint4*>(p.C + (size_t)m * p.ldc + t.n0 + c);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          uint4 o;
          o.x = pack_bf16x2(__uint_as_float(v[8 * i + 0]) * rs, __uint_as_float(v[8 * i + 1]) * rs);
          o.y = pack_bf16x2(__uint_as_float(v[8 * i + 2]) * rs, __uint_as_float(v[8 * i + 3]) * rs);
          o.z = pack_bf16x2(__uint_as_float(v[8 * i + 4]) * rs, __uint_as_float(v[8 * i + 5]) * rs);
          o.w = pack_bf16x2(__uint_as_float(v[8 * i + 6]) * rs, __uint_as_float(v[8 * i + 7]) * rs);
          dst[i] = o;
        }
      }
    }
  }
  __device__ void finish() {}
};

// Residual update (attention output projection K8 and FFN down projection K9) of the latency path:
//   h32[m, n] += acc;  h16[m, n] = bf16(h32[m, n]);  ss_out[n / 32][m] = sum over the 32-column chunk of h32[m, n]^2
// The fp32 copy is the residual stream; the bf16 copy is the next GEMM's A operand;
// ss_out feeds the next RMSNorm (see RowScale).  One partial sum per 32-column chunk: the latency path uses 32- or
// 64-wide tiles depending on the token count and must hand the next RMSNorm the same partial sums either way.
// The throughput path runs EpiWsResidual (rpx_gemm_ws.cuh).
//
// The accumulator arrives one ROW per thread, which is the worst possible layout for global
// memory: a warp-wide 16-byte access would touch 32 different 128-byte lines.  Each warp
// therefore transposes its 32x32 fp32 block through a swizzled shared-memory tile and does the
// read-modify-write with lanes running along the row: one instruction covers 4 rows x 128
// contiguous bytes (4 L1 wavefronts instead of 32).  Residual loads run one chunk ahead.
// (RPX_EPI_WARPS=8 — two warps per lane group splitting the chunks — is off by default.)
struct EpiResidualParams {
  float* h32;
  __nv_bfloat16* h16;
  int ld;
  float* ss_out;  // [n_parts][ss_stride], n_parts = ss_parts(ld, latency) of rpx_encoder.cu
  int ss_stride;
};
struct EpiResidualChunkSS {
  using Params = EpiResidualParams;
  static constexpr int kWarps = RPX_EPI_WARPS;
  static constexpr size_t kSmemBytes = kWarps * 32 * 32 * sizeof(float);  // one 32x32 tile per warp
  Params p;
  float4* stg;  // this warp's staging tile: row r = 8 float4, stored at slot (j ^ (r & 7))
  int lane, grp;
  float4 h[8];  // residual values of the chunk in flight (loaded one chunk ahead)
  __device__ EpiResidualChunkSS(const Params& p_, uint8_t* smem_extra, int row, int part) : p(p_) {
    lane = row & 31;
    grp = row >> 5;
    stg = reinterpret_cast<float4*>(smem_extra) + (part * 4 + grp) * 32 * 8;
  }
  __device__ __forceinline__ void load_chunk(const TileCtx& t, int c, int row_base, int sub, int col4,
                                             float4 (&hh)[8]) const {
    const size_t col = (size_t)t.n0 + c + col4;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int r = sub + 4 * i, m = row_base + r;
      if (r < t.rows_per_warp && m < t.M) hh[i] = *reinterpret_cast<const float4*>(p.h32 + (size_t)m * p.ld + col);
      else hh[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  // the first chunk's residual values do not depend on the accumulator: they are fetched while the MMAs of
  // the tile are still running (on the latency path that L2 round trip was a third of the epilogue)
  __device__ void before_wait(const TileCtx& t) {
    const int c = 32 * t.part;
    if (c < t.n_cols) load_chunk(t, c, t.m0 + grp * t.rows_per_warp, lane >> 3, (lane & 7) * 4, h);
  }
  __device__ void tile(const TileCtx& t) {
    const int sub = lane >> 3;        // row within a group of 4
    const int j4 = lane & 7;          // which float4 of the 32-column chunk
    const int col4 = j4 * 4;
    const int row_base = t.m0 + grp * t.rows_per_warp;
    const int step = 32 * t.split;
    float ss[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) ss[i] = 0.f;
    float4 hn[8];
    int c = 32 * t.part;
    for (; c < t.n_cols; c += step) {
      uint32_t v[32];
      acc_ld32(t.acc + c, v);
      // next chunk's residual loads go out before this chunk is consumed
      if (c + step < t.n_cols) load_chunk(t, c + step, row_base, sub, col4, hn);
      const size_t col = (size_t)t.n0 + c + col4;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        stg[lane * 8 + (j ^ (lane & 7))] =
            make_float4(__uint_as_float(v[4 * j]), __uint_as_float(v[4 * j + 1]), __uint_as_float(v[4 * j + 2]),
                        __uint_as_float(v[4 * j + 3]));
      __syncwarp();
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = sub + 4 * i;
        const int m = row_base + r;
        const float4 a = stg[r * 8 + (j4 ^ (r & 7))];
        h[i].x += a.x;
        h[i].y += a.y;
        h[i].z += a.z;
        h[i].w += a.w;
        ss[i] += h[i].x * h[i].x + h[i].y * h[i].y + h[i].z * h[i].z + h[i].w * h[i].w;
        if (r < t.rows_per_warp && m < t.M) {
          *reinterpret_cast<float4*>(p.h32 + (size_t)m * p.ld + col) = h[i];
          *reinterpret_cast<uint2*>(p.h16 + (size_t)m * p.ld + col) =
              make_uint2(pack_bf16x2(h[i].x, h[i].y), pack_bf16x2(h[i].z, h[i].w));
        }
      }
      __syncwarp();
#pragma unroll
      for (int i = 0; i < 8; ++i) h[i] = hn[i];
      write_ss(t, ss, row_base, sub, (t.n0 + c) >> 5);
#pragma unroll
      for (int i = 0; i < 8; ++i) ss[i] = 0.f;
    }
  }
  // a row's partial sums sit in the 8 lanes that share `sub`
  __device__ __forceinline__ void write_ss(const TileCtx& t, float (&ss)[8], int row_base, int sub, int part_idx) const {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float v = ss[i];
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      v += __shfl_xor_sync(0xffffffffu, v, 4);
      const int r = sub + 4 * i, m = row_base + r;
      if ((lane & 7) == 0 && r < t.rows_per_warp && m < t.M) p.ss_out[(size_t)part_idx * p.ss_stride + m] = v;
    }
  }
  __device__ void finish() {}
};

// gelu_new (tanh form) — HF activations.py NewGELUActivation, used by T5 "gated-gelu".
__device__ __forceinline__ float gelu_new(float x) {
  const float k0 = 0.7978845608028654f;  // sqrt(2/pi)
  const float k1 = 0.044715f;
  float u = k0 * (x + k1 * x * x * x);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
  return 0.5f * x * (1.0f + t);
}

// Gated-GELU FFN up projection (K9) of the latency path: accumulator columns [0, HALF) are the gate and
// [HALF, 2*HALF) the linear branch of the same HALF hidden units (HALF = 64 / 32: the SPLIT_B tiles).  The
// throughput path runs EpiWsGeGLU (rpx_gemm_ws.cuh).
//   out[m, n_blk*HALF + j] = bf16( gelu_new(acc[j]*rs) * (acc[HALF+j]*rs) )
template <int HALF>
struct EpiGeGLUT {
  struct Params {
    __nv_bfloat16* out;  // [M, N/2]
    int ldo;
    RowScale rs;
  };
  static constexpr size_t kSmemBytes = 0;
  static constexpr int kWarps = RPX_EPI_WARPS;
  Params p;
  float rs = 0.f;  // (fetched ahead of the accumulator: see EpiStoreBF16)
  __device__ EpiGeGLUT(const Params& p_, uint8_t*, int, int) : p(p_) {}
  __device__ void before_wait(const TileCtx& t) {
    const int m = t.m0 + t.row;
    rs = m < t.M ? p.rs.get(m) : 0.f;
  }
  __device__ void tile(const TileCtx& t) {
    const int m = t.m0 + t.row;
    const bool ok = m < t.M;
    for (int c = 32 * t.part; c < HALF; c += 32 * t.split) {
      uint32_t g[32], u[32];
      acc_ld32(t.acc + c, g);
      acc_ld32(t.acc + HALF + c, u);
      if (ok) {
        uint4* dst = reinterpret_cast<uint4*>(p.out + (size_t)m * p.ldo + t.n_blk * HALF + c);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float r[8];
#pragma unroll
          for (int j = 0; j < 8; ++j)
            r[j] = gelu_new(__uint_as_float(g[8 * i + j]) * rs) * (__uint_as_float(u[8 * i + j]) * rs);
          uint4 o;
          o.x = pack_bf16x2(r[0], r[1]);
          o.y = pack_bf16x2(r[2], r[3]);
          o.z = pack_bf16x2(r[4], r[5]);
          o.w = pack_bf16x2(r[6], r[7]);
          dst[i] = o;
        }
      }
    }
  }
  __device__ void finish() {}
};

}  // namespace rpx
