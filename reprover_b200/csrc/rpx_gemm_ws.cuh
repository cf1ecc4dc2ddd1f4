// rpx_gemm_ws.cuh — the throughput-path GEMM core: 128 x 256 tiles, two consumer warpgroups, epilogues run
// straight from the accumulator registers.
//
//   D[M, N] (fp32) = A[M, K] * B[N, K]^T        A, B bf16, K contiguous, K % 64 == 0
//
// Structure (one persistent CTA per SM, 384 threads, tiles visited n-fastest like gemm_tc_kernel):
//   warpgroup 0     : TMA producers, which give their registers away (setmaxnreg.dec to 40).
//                     warp 0: one elected thread streams 128 x 64 A and 256 x 64 B tiles into a STAGES-deep
//                     128B-swizzled ring (48 KB per stage), completion on `full[]`.  It keeps filling the ring
//                     across tile boundaries, so the next tile's first k-blocks land while the consumers run the
//                     epilogue.  With CLUSTER = 2 (see below) it loads its own A tile and one half of the shared
//                     B tile, which it multicasts into both CTAs.
//                     warps 1, 2 (residual epilogues, Epi::kResBufs > 0): warp 1 + w streams the fp32 residual
//                     block of consumer w's rows into that consumer's ring of kResBufs chunk buffers (64 rows x
//                     32 columns, 8 KB, 128B-swizzled), completion on `rfull[]`, released on `rempty[]`.  A tile's
//                     chunks are requested as soon as a buffer is free, i.e. while its mainloop still runs.
//   warpgroups 1, 2 : consumers — consumer w owns rows [64w, 64w + 64) of the tile and issues wgmma.m64n256k16
//                     (128 fp32 accumulator registers per thread, setmaxnreg.inc to 232); a stage goes back to
//                     the producer (`empty[]`) once the wgmma group that read it has retired: lane 0 of each
//                     consumer warp arrives once for its warp.  After the last k-block each consumer runs the
//                     epilogue functor on its own fragment.
//                     The last n-tile of an N that is not a multiple of 256 runs its k-loop on m64nWk16 with W its
//                     column count rounded up to 64 (the accumulator prefix acc[0, W/2)), chosen once per tile:
//                     the B rows past N are still loaded as TMA zero-fill, but only those below W reach the
//                     tensor cores.  The order of the additions over k, and so every output bit, is that of the
//                     full-width MMA.
//
// CLUSTER = 2: the CTAs run as clusters of two on vertically adjacent tiles.  A work unit is an (m-tile pair,
// n-tile), units visited n-fastest; rank r of the cluster takes m-tile 2 (u / tiles_n) + r.  Both need the same
// 256 x 64 B tile per k-block, so rank r loads its rows [128r, 128r + 128) once from L2 and multicasts them
// into the same offset of both CTAs' stage (tmB encoded with a 128-row box): a CTA pulls 32 KB per k-block
// through L2 instead of 48 KB.  The B tile in shared memory is laid out as with CLUSTER = 1.  Since a refill
// writes into the peer's shared memory, a stage goes back to the producer only once the consumer warps of both
// CTAs have released it (each warp also arrives on the peer's `empty[]`).  When tiles_m is odd, the last pair's
// rank-1 tile lies wholly past M: that CTA still runs the pipeline (TMA zero-fills its A and counts the full
// box), and its epilogues store nothing.
// Against gemm_tc_kernel (128 x 128 tiles, accumulator handed to epilogue warps through a 66 KB shared-memory
// tile): a k-block brings 48 KB for 4.2 MFLOP instead of 32 KB for 2.1 MFLOP, every m64n256k16 reads its A
// slice once per 256 columns, and no shared memory is held for the hand-off.  The epilogue no longer overlaps
// the MMAs of the next tile inside the CTA, so no epilogue thread waits on a global load: what the epilogue
// reads either arrives in shared memory ahead of it (the residual stream) or is fetched during the first
// k-block (Epi::prefetch).
//
// Shared memory: STAGES x 48 KB of operand ring + 2 x kResBufs x 8 KB of residual chunks within the 227 KB an
// H100 block may use; the residual GEMMs choose the split per site (rpx_encoder.cu, residual_gemm).
//
// Fragment layout (rpx_ptx.cuh): the thread with lane l of warp v (0..3) of consumer w holds rows
// r0 = 64w + 16v + l/4 and r0 + 8 of the tile; acc[4j], acc[4j+1] are row r0, columns 8j + 2(l%4) + {0, 1}, and
// acc[4j+2], acc[4j+3] the same columns of row r0 + 8, for j = 0..31.  A quad of lanes holds 8 contiguous
// columns of a row: fp32 accesses from the fragment fill whole 32-byte sectors.
#pragma once
#include <type_traits>

#include "rpx_gemm.cuh"

namespace rpx {

constexpr int kWsBlockN = 256;
constexpr int kWsThreads = 384;
constexpr int kResChunkCols = 32;                                  // one 128-byte swizzle row of fp32
constexpr int kResChunkBytes = 64 * kResChunkCols * 4;             // 8 KB: a consumer's 64 rows

template <int STAGES, int RES_BUFS>
struct WsCfg {
  static_assert(2 * STAGES + 4 * RES_BUFS <= 32, "barrier block holds 32 mbarriers");
  static constexpr int kABytes = kBlockM * kBlockK * 2;    // 16 KB
  static constexpr int kBBytes = kWsBlockN * kBlockK * 2;  // 32 KB
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kRingBytes = STAGES * kStageBytes;
  static constexpr int kResBytes = 2 * RES_BUFS * kResChunkBytes;
  // ring + residual chunks + 1 KB alignment slack + barriers
  static constexpr size_t kSmemBytes = (size_t)kRingBytes + kResBytes + 1024 + 256;
};

// What a register-fragment epilogue sees for one output tile.
struct FragCtx {
  int m0, n0;  // tile origin in the output
  int n_blk;   // n-tile index
  int n_cols;  // valid columns in this tile (multiple of 32)
  int M, N;
  int r0;      // output row of acc[4j], acc[4j+1]; acc[4j+2], acc[4j+3] belong to row r0 + 8
  int q;       // lane % 4: this thread's columns are 8j + 2q + {0, 1}
};

// This consumer's ring of residual chunk buffers (Epi::kResBufs > 0).  Chunk k of a tile is columns
// [32k, 32k + 32) of the consumer's 64 rows; 16-byte unit u of row r sits at unit u ^ (r % 8) of that row
// (TMA 128B swizzle).  The chunks of successive tiles take the buffers in turn.
struct ResStream {
  float* buf;       // kResBufs x 64 x 32 fp32
  uint64_t* full;   // kResBufs mbarriers: the producer's TMA landed
  uint64_t* empty;  // kResBufs mbarriers: all 128 consumer threads are done with the buffer
};

// wgmma.m64nWk16 on the first W/2 registers of a consumer's accumulator (rpx_ptx.cuh).
template <int W>
RPX_DEVICE void wgmma_ws(float (&acc)[128], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  static_assert(W == 64 || W == 128 || W == 192 || W == 256, "MMA width: a multiple of 64 up to the tile width");
  if constexpr (W == 64) wgmma_m64n64k16_ss(acc, desc_a, desc_b, accumulate);
  else if constexpr (W == 128) wgmma_m64n128k16_ss(acc, desc_a, desc_b, accumulate);
  else if constexpr (W == 192) wgmma_m64n192k16_ss(acc, desc_a, desc_b, accumulate);
  else wgmma_m64n256k16_ss(acc, desc_a, desc_b, accumulate);
}

// Epi must provide:
//   struct Params;                                  (trivially copyable kernel argument)
//   static constexpr int kResBufs;                  (residual chunk buffers per consumer; 0: no residual stream)
//   __device__ Epi(const Params&, const ResStream&);
//   __device__ void prefetch(const FragCtx&);       (runs while the tile's first k-block is in flight: global
//                                                    reads that do not depend on the accumulator)
//   __device__ void tile(const FragCtx&, const float (&acc)[128]);
// With kResBufs > 0, tmR maps the residual matrix ([M, N] fp32, box 32 x 64, 128B swizzle): the producer loads,
// for every tile and consumer whose first row is < M, the chunks k with 32k < n_cols in order, and tile() must
// consume exactly those.
template <class Epi, int STAGES, int CLUSTER>
__global__ void __launch_bounds__(kWsThreads, 1)
gemm_ws_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmR, int M, int N, int K, int tiles_m, int tiles_n,
               typename Epi::Params ep) {
  static_assert(CLUSTER == 1 || CLUSTER == 2, "one CTA, or a pair sharing the B tile");
  using Cfg = WsCfg<STAGES, Epi::kResBufs>;
  constexpr int R = Epi::kResBufs;
  extern __shared__ uint8_t smem_raw[];
  // 128B swizzle needs 1024-byte aligned tile bases.
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024 - (raw_addr & 1023)) & 1023);
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * Cfg::kABytes;
  float* sR = reinterpret_cast<float*>(smem + Cfg::kRingBytes);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + Cfg::kRingBytes + Cfg::kResBytes);
  uint64_t* empty = full + STAGES;
  uint64_t* rfull = empty + STAGES;  // [2][R]
  uint64_t* rempty = rfull + 2 * R;  // [2][R]

  const int warp = threadIdx.x >> 5;
  const int wg = warp >> 2;
  const int num_kb = K / kBlockK;
  // Work units: tiles (CLUSTER = 1) or vertically adjacent tile pairs; this CTA takes units u0, u0 + u_step, ...
  const int rank = CLUSTER > 1 ? (int)cluster_ctarank() : 0;
  const int num_units = (tiles_m + CLUSTER - 1) / CLUSTER * tiles_n;
  const int u0 = (int)blockIdx.x / CLUSTER;
  const int u_step = (int)gridDim.x / CLUSTER;
  auto unit_m = [&](int u) { return CLUSTER * (u / tiles_n) + rank; };

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (R > 0) tma_prefetch_desc(&tmR);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], CLUSTER * 8);  // every consumer warp of every CTA of the cluster
    }
    for (int s = 0; s < 2 * R; ++s) {
      mbar_init(&rfull[s], 1);
      mbar_init(&rempty[s], 128);  // every thread of the consumer
    }
    fence_mbar_init();
  }
  __syncthreads();
  // the peer's barriers are initialised before anything multicasts into this CTA or arrives on them
  if (CLUSTER > 1) cluster_sync_all();
  // Under programmatic dependent launch (rpx_ptx.cuh) the preceding kernel may still be running: A, the row
  // scales and the residual stream are its outputs.
  pdl_launch_dependents();
  pdl_wait();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      // ---------------------------------------------------------------- TMA producer: operands
      int stage = 0;
      uint32_t phase = 0;
      for (int u = u0; u < num_units; u += u_step) {
        const int m_blk = unit_m(u), n_blk = u % tiles_n;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          // with CLUSTER = 2 the peer's half of B completes on this barrier too
          mbar_arrive_expect_tx(&full[stage], Cfg::kStageBytes);
          tma_load_2d(sA + stage * Cfg::kABytes, &tmA, &full[stage], kb * kBlockK, m_blk * kBlockM);
          if constexpr (CLUSTER == 1) {
            tma_load_2d(sB + stage * Cfg::kBBytes, &tmB, &full[stage], kb * kBlockK, n_blk * kWsBlockN);
          } else {
            constexpr int H = kWsBlockN / 2;
            tma_load_2d_multicast(sB + stage * Cfg::kBBytes + rank * H * kBlockK * 2, &tmB, &full[stage], kb * kBlockK,
                                  n_blk * kWsBlockN + rank * H, (uint16_t)0x3);
          }
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    } else if (R > 0 && (warp == 1 || warp == 2) && elect_one()) {
      // ---------------------------------------------------------------- TMA producer: residual chunks
      const int w = warp - 1;  // consumer served
      float* buf = sR + w * R * (kResChunkBytes / 4);
      uint64_t* rf = rfull + w * R;
      uint64_t* re = rempty + w * R;
      int b = 0;
      uint32_t phase = 0;
      for (int u = u0; u < num_units; u += u_step) {
        const int row0 = unit_m(u) * kBlockM + 64 * w;
        const int n0 = (u % tiles_n) * kWsBlockN;
        const int n_cols = N - n0 < kWsBlockN ? N - n0 : kWsBlockN;
        if (row0 >= M) continue;
        for (int col = 0; col < n_cols; col += kResChunkCols) {
          mbar_wait(&re[b], phase ^ 1);
          mbar_arrive_expect_tx(&rf[b], kResChunkBytes);  // rows past M arrive zero-filled and count in full
          tma_load_2d(buf + b * (kResChunkBytes / 4), &tmR, &rf[b], n0 + col, row0);
          if (++b == R) {
            b = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers
    setmaxnreg_inc<232>();
    const int cw = wg - 1;  // which 64-row half of the tile
    const int lane = threadIdx.x & 31;
    Epi epi(ep, ResStream{sR + cw * R * (kResChunkBytes / 4), rfull + cw * R, rempty + cw * R});
    float acc[128];
    int stage = 0;
    uint32_t phase = 0;
    // One arrival per warp (lane 0, once the warp's wgmma_wait has returned in every lane), on this CTA's
    // barrier and, with CLUSTER = 2, on the peer's.
    auto release = [&](int st) {
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&empty[st]);
        if (CLUSTER > 1) mbar_arrive_cluster(&empty[st], (uint32_t)(rank ^ 1));
      }
    };
    // One tile's k-loop on MMAs W columns wide (W a compile-time constant: no branch between wgmma forms
    // inside the loop).
    auto mainloop = [&](auto width, const FragCtx& c) {
      constexpr int W = decltype(width)::value;
      int prev = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full[stage], phase);
        // +8 KB (>>4 = 512) for the second 64-row half of A; +32 bytes (>>4 = 2) per K=16 step inside the atom
        const uint64_t a_desc = make_smem_desc_kmajor_sw128(smem_u32(sA + stage * Cfg::kABytes)) + 512 * cw;
        const uint64_t b_desc = make_smem_desc_kmajor_sw128(smem_u32(sB + stage * Cfg::kBBytes));
        wgmma_fence_operand(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / kMmaK; ++k) wgmma_ws<W>(acc, a_desc + 2 * k, b_desc + 2 * k, (kb | k) != 0);
        wgmma_commit();
        if (kb == 0) epi.prefetch(c);
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
      wgmma_fence_operand(acc);
      release(prev);
    };
    for (int u = u0; u < num_units; u += u_step) {
      FragCtx c;
      c.n_blk = u % tiles_n;
      c.m0 = unit_m(u) * kBlockM;
      c.n0 = c.n_blk * kWsBlockN;
      c.n_cols = N - c.n0 < kWsBlockN ? N - c.n0 : kWsBlockN;
      c.M = M;
      c.N = N;
      c.r0 = c.m0 + 64 * cw + 16 * (warp & 3) + (lane >> 2);
      c.q = lane & 3;
      // The last n-tile of an N that is not a multiple of 256 issues MMAs only as wide as its columns rounded up
      // to 64; the B rows between n_cols and that width are TMA zero-fill, as are those past it, which no MMA reads.
      switch ((c.n_cols + 63) / 64) {
        case 1: mainloop(std::integral_constant<int, 64>{}, c); break;
        case 2: mainloop(std::integral_constant<int, 128>{}, c); break;
        case 3: mainloop(std::integral_constant<int, 192>{}, c); break;
        default: mainloop(std::integral_constant<int, 256>{}, c); break;
      }
      epi.tile(c, acc);
    }
  }
  // The peer may still multicast into this CTA's ring or arrive on its barriers until it is done too.
  if (CLUSTER > 1) {
    __syncwarp();
    cluster_sync_all();
  }
}

// ============================================================================ register-fragment epilogues
// Same arithmetic as EpiStoreF32 / EpiStoreBF16 / EpiGeGLUT of rpx_gemm.cuh, element for element.

// bf16 stores of a quad's fragment as 16-byte vectors.  Lane q of a quad holds, for a row and a block of 32
// columns, the bf16 pairs x_t at columns 8t + 2q, 8t + 2q + 1 (t = 0..3, fragment blocks j = 4b + t); the four
// lanes exchange them (a 4 x 4 transpose, two xor shuffles per stage) so that lane q returns columns
// [8q, 8q + 8) of the block.  A warp then stores 64 contiguous bytes per row and instruction instead of 16.
// Every lane of the warp must call it.
RPX_DEVICE uint4 quad_columns(uint32_t x0, uint32_t x1, uint32_t x2, uint32_t x3, int q) {
  // stage 1 (lanes q, q ^ 2): the off-diagonal 2 x 2 blocks
  const bool hi = q & 2;
  uint32_t r0 = __shfl_xor_sync(0xffffffffu, hi ? x0 : x2, 2);
  uint32_t r1 = __shfl_xor_sync(0xffffffffu, hi ? x1 : x3, 2);
  if (hi) {
    x0 = r0;
    x1 = r1;
  } else {
    x2 = r0;
    x3 = r1;
  }
  // stage 2 (lanes q, q ^ 1): inside each 2 x 2 block
  const bool odd = q & 1;
  r0 = __shfl_xor_sync(0xffffffffu, odd ? x0 : x1, 1);
  r1 = __shfl_xor_sync(0xffffffffu, odd ? x2 : x3, 1);
  if (odd) {
    x0 = r0;
    x2 = r1;
  } else {
    x1 = r0;
    x3 = r1;
  }
  return make_uint4(x0, x1, x2, x3);
}

// C[m, n] = acc (fp32).  The bare core behind rpx_gemm_bf16_f32.
struct EpiWsStoreF32 {
  using Params = EpiStoreF32::Params;
  static constexpr int kResBufs = 0;
  Params p;
  __device__ EpiWsStoreF32(const Params& p_, const ResStream&) : p(p_) {}
  __device__ void prefetch(const FragCtx&) {}
  __device__ void tile(const FragCtx& c, const float (&acc)[128]) {
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      if (8 * j < c.n_cols) {
        float* dst = p.C + (size_t)c.r0 * p.ldc + c.n0 + 8 * j + 2 * c.q;
        if (c.r0 < c.M) *reinterpret_cast<float2*>(dst) = make_float2(acc[4 * j], acc[4 * j + 1]);
        if (c.r0 + 8 < c.M) *reinterpret_cast<float2*>(dst + 8 * (size_t)p.ldc) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
    }
  }
};

// C[m, n] = acc * rs[m] (fp32).  The generator's output head (rpx_decoder.cu): the decoder's final RMSNorm weight is
// folded into B, its row scale applied here.
struct EpiWsStoreF32Scaled {
  struct Params {
    float* C;
    int ldc;
    RowScale rs;
  };
  static constexpr int kResBufs = 0;
  Params p;
  float rs0 = 0.f, rs1 = 0.f;
  __device__ EpiWsStoreF32Scaled(const Params& p_, const ResStream&) : p(p_) {}
  __device__ void prefetch(const FragCtx& c) {
    rs0 = c.r0 < c.M ? p.rs.get(c.r0) : 0.f;
    rs1 = c.r0 + 8 < c.M ? p.rs.get(c.r0 + 8) : 0.f;
  }
  __device__ void tile(const FragCtx& c, const float (&acc)[128]) {
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      if (8 * j < c.n_cols) {
        float* dst = p.C + (size_t)c.r0 * p.ldc + c.n0 + 8 * j + 2 * c.q;
        if (c.r0 < c.M) *reinterpret_cast<float2*>(dst) = make_float2(acc[4 * j] * rs0, acc[4 * j + 1] * rs0);
        if (c.r0 + 8 < c.M)
          *reinterpret_cast<float2*>(dst + 8 * (size_t)p.ldc) = make_float2(acc[4 * j + 2] * rs1, acc[4 * j + 3] * rs1);
      }
    }
  }
};

// C[m, n] = bf16(acc * rs[m]).  The QKV projection (RMSNorm folded: the weight into B, the row scale here).
struct EpiWsStoreBF16 {
  using Params = EpiStoreBF16::Params;
  static constexpr int kResBufs = 0;
  Params p;
  float rs0 = 0.f, rs1 = 0.f;
  __device__ EpiWsStoreBF16(const Params& p_, const ResStream&) : p(p_) {}
  __device__ void prefetch(const FragCtx& c) {
    rs0 = c.r0 < c.M ? p.rs.get(c.r0) : 0.f;
    rs1 = c.r0 + 8 < c.M ? p.rs.get(c.r0 + 8) : 0.f;
  }
  __device__ void tile(const FragCtx& c, const float (&acc)[128]) {
    __nv_bfloat16* dst = p.C + (size_t)c.r0 * p.ldc + c.n0 + 8 * c.q;
#pragma unroll
    for (int b = 0; b < 8; ++b) {  // 32-column blocks (n_cols is a multiple of 32: a block is valid or not, warp-wide)
      if (32 * b < c.n_cols) {
        const float* a = acc + 16 * b;
        const uint4 v0 = quad_columns(pack_bf16x2(a[0] * rs0, a[1] * rs0), pack_bf16x2(a[4] * rs0, a[5] * rs0),
                                      pack_bf16x2(a[8] * rs0, a[9] * rs0), pack_bf16x2(a[12] * rs0, a[13] * rs0), c.q);
        const uint4 v1 = quad_columns(pack_bf16x2(a[2] * rs1, a[3] * rs1), pack_bf16x2(a[6] * rs1, a[7] * rs1),
                                      pack_bf16x2(a[10] * rs1, a[11] * rs1), pack_bf16x2(a[14] * rs1, a[15] * rs1), c.q);
        if (c.r0 < c.M) *reinterpret_cast<uint4*>(dst + 32 * b) = v0;
        if (c.r0 + 8 < c.M) *reinterpret_cast<uint4*>(dst + 8 * (size_t)p.ldc + 32 * b) = v1;
      }
    }
  }
};

// Gated-GELU FFN up projection: n-tile t is packed weight rows [256t, 256t + 256), i.e. the gate rows and then
// the linear-branch rows of hidden units [128t, 128t + 128) (rpx_encoder.cu interleaves wi_0 / wi_1 in 128-row
// blocks), so gate column j and linear column j + 128 sit in the same thread: acc block j and block j + 16.
//   out[m, 128t + j] = bf16( gelu_new(acc[j]*rs) * (acc[128+j]*rs) )
struct EpiWsGeGLU {
  struct Params {
    __nv_bfloat16* out;  // [M, N/2]
    int ldo;
    RowScale rs;
  };
  static constexpr int kResBufs = 0;
  Params p;
  float rs0 = 0.f, rs1 = 0.f;
  __device__ EpiWsGeGLU(const Params& p_, const ResStream&) : p(p_) {}
  __device__ void prefetch(const FragCtx& c) {
    rs0 = c.r0 < c.M ? p.rs.get(c.r0) : 0.f;
    rs1 = c.r0 + 8 < c.M ? p.rs.get(c.r0 + 8) : 0.f;
  }
  __device__ void tile(const FragCtx& c, const float (&acc)[128]) {
    __nv_bfloat16* dst = p.out + (size_t)c.r0 * p.ldo + c.n_blk * (kWsBlockN / 2) + 8 * c.q;
#pragma unroll
    for (int b = 0; b < 4; ++b) {  // 32-column blocks of the output
      uint32_t w0[4], w1[4];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float* g = acc + 4 * (4 * b + t);
        const float* u = acc + 4 * (4 * b + t + 16);
        w0[t] = pack_bf16x2(gelu_new(g[0] * rs0) * (u[0] * rs0), gelu_new(g[1] * rs0) * (u[1] * rs0));
        w1[t] = pack_bf16x2(gelu_new(g[2] * rs1) * (u[2] * rs1), gelu_new(g[3] * rs1) * (u[3] * rs1));
      }
      const uint4 v0 = quad_columns(w0[0], w0[1], w0[2], w0[3], c.q);
      const uint4 v1 = quad_columns(w1[0], w1[1], w1[2], w1[3], c.q);
      if (c.r0 < c.M) *reinterpret_cast<uint4*>(dst + 32 * b) = v0;
      if (c.r0 + 8 < c.M) *reinterpret_cast<uint4*>(dst + 8 * (size_t)p.ldo + 32 * b) = v1;
    }
  }
};

// Residual update of the throughput path (attention output projection K8, FFN down projection K9):
//   h32[m, n] += acc;  h16[m, n] = bf16(h32[m, n]);  ss_out[2 n_blk + n / 128 % 2][m] = sum over the 128-column
//   half-tile of h32[m, n]^2
// i.e. one RMSNorm partial sum per 128 columns, the layout ss_parts(D, false) describes.  The residual block
// arrives in shared memory through the ResStream (RES_BUFS chunk buffers per consumer), so the epilogue never
// waits on a global load.  Per 32-column chunk, warp v of the consumer (fragment rows [16v, 16v + 16)):
//   1. adds its accumulator fragment into the chunk in place (h32 + acc, as EpiResidualChunkSS);
//   2. reads its 16 rows back with lanes along the row — lane (s, j) takes float4 j of rows s, s + 4, s + 8,
//      s + 12 — and writes h32 and h16 with 16- and 8-byte stores, 4 rows x 128 contiguous bytes per instruction;
//   3. fences its shared-memory writes against the async proxy (the buffer's next TMA fill) and releases it.
// Each lane sums its float4's squares over the half-tile's chunks in column order and a xor-1/2/4 shuffle adds
// the 8 lanes of a row (within a chunk, the order of EpiResidualChunkSS): a fixed order that depends on neither
// T nor the row's tile, so h32, h16 and the partial sums of a row are the same bits in every call.
template <int RES_BUFS>
struct EpiWsResidual {
  using Params = EpiResidualParams;
  static constexpr int kResBufs = RES_BUFS;
  Params p;
  ResStream rs;
  int b = 0;           // buffer of the next chunk
  uint32_t phase = 0;  // its rfull parity
  __device__ EpiWsResidual(const Params& p_, const ResStream& rs_) : p(p_), rs(rs_) {}
  __device__ void prefetch(const FragCtx&) {}
  __device__ void tile(const FragCtx& c, const float (&acc)[128]) {
    const int lane = threadIdx.x & 31;
    const int v = (threadIdx.x >> 5) & 3;
    const int row0 = c.r0 - 16 * v - (lane >> 2);  // first row of this consumer's 64
    if (row0 >= c.M) return;                        // (the producer loads nothing for it either)
    const int sub = lane >> 3, j4 = lane & 7;
    float ss[4];
#pragma unroll
    for (int k = 0; k < kWsBlockN / kResChunkCols; ++k) {
      if (kResChunkCols * k >= c.n_cols) break;
      if (k % 4 == 0) {
#pragma unroll
        for (int i = 0; i < 4; ++i) ss[i] = 0.f;
      }
      float* s = rs.buf + b * (kResChunkBytes / 4);
      mbar_wait(&rs.full[b], phase);
      // 1. fragment columns 8jj + 2q + {0, 1} of rows 16v + lane/4 (+ 8)
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = 4 * k + jj;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = 16 * v + (lane >> 2) + 8 * h;
          float2* x = reinterpret_cast<float2*>(s + r * kResChunkCols + (((2 * jj + (c.q >> 1)) ^ (r & 7)) << 2) + 2 * (c.q & 1));
          float2 hv = *x;
          hv.x += acc[4 * j + 2 * h];
          hv.y += acc[4 * j + 2 * h + 1];
          *x = hv;
        }
      }
      __syncwarp();
      // 2. rows along the lanes
      const size_t col = (size_t)c.n0 + kResChunkCols * k + 4 * j4;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = 16 * v + sub + 4 * i;
        const int m = row0 + r;
        const float4 hv = *reinterpret_cast<const float4*>(s + r * kResChunkCols + ((j4 ^ (r & 7)) << 2));
        ss[i] += hv.x * hv.x + hv.y * hv.y + hv.z * hv.z + hv.w * hv.w;
        if (m < c.M) {
          *reinterpret_cast<float4*>(p.h32 + (size_t)m * p.ld + col) = hv;
          *reinterpret_cast<uint2*>(p.h16 + (size_t)m * p.ld + col) =
              make_uint2(pack_bf16x2(hv.x, hv.y), pack_bf16x2(hv.z, hv.w));
        }
      }
      // 3. the buffer goes back to the producer
      fence_proxy_async_smem();
      mbar_arrive(&rs.empty[b]);
      if (++b == RES_BUFS) {
        b = 0;
        phase ^= 1;
      }
      if (k % 4 == 3 || kResChunkCols * (k + 1) >= c.n_cols) {
        const int part = 2 * c.n_blk + k / 4;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float t = ss[i];
          t += __shfl_xor_sync(0xffffffffu, t, 1);
          t += __shfl_xor_sync(0xffffffffu, t, 2);
          t += __shfl_xor_sync(0xffffffffu, t, 4);
          const int m = row0 + 16 * v + sub + 4 * i;
          if (j4 == 0 && m < c.M) p.ss_out[(size_t)part * p.ss_stride + m] = t;
        }
      }
    }
  }
};

}  // namespace rpx
