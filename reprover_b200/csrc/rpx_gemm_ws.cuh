// rpx_gemm_ws.cuh — the throughput-path GEMM core: 128 x 256 tiles, two consumer warpgroups, epilogues run
// straight from the accumulator registers.
//
//   D[M, N] (fp32) = A[M, K] * B[N, K]^T        A, B bf16, K contiguous, K % 64 == 0
//
// Structure (one persistent CTA per SM, 384 threads, tiles visited n-fastest like gemm_tc_kernel):
//   warpgroup 0     : TMA producer — one elected thread streams 128 x 64 A and 256 x 64 B tiles into a 4-deep
//                     128B-swizzled ring (48 KB per stage), completion on `full[]`.  It keeps filling the ring
//                     across tile boundaries, so the next tile's first k-blocks land while the consumers run the
//                     epilogue.  The warpgroup gives its registers away (setmaxnreg.dec to 40).
//   warpgroups 1, 2 : consumers — consumer w owns rows [64w, 64w + 64) of the tile and issues wgmma.m64n256k16
//                     (128 fp32 accumulator registers per thread, setmaxnreg.inc to 232); a stage goes back to
//                     the producer (`empty[]`) once the wgmma group that read it has retired.  After the last
//                     k-block each consumer runs the epilogue functor on its own fragment.
//
// Against gemm_tc_kernel (128 x 128 tiles, accumulator handed to epilogue warps through a 66 KB shared-memory
// tile): a k-block brings 48 KB for 4.2 MFLOP instead of 32 KB for 2.1 MFLOP, every m64n256k16 reads its A
// slice once per 256 columns, and no shared memory is held for the hand-off.  The epilogue no longer overlaps
// the MMAs of the next tile inside the CTA; its global reads are started early instead (Epi::prefetch).
//
// Fragment layout (rpx_ptx.cuh): the thread with lane l of warp v (0..3) of consumer w holds rows
// r0 = 64w + 16v + l/4 and r0 + 8 of the tile; acc[4j], acc[4j+1] are row r0, columns 8j + 2(l%4) + {0, 1}, and
// acc[4j+2], acc[4j+3] the same columns of row r0 + 8, for j = 0..31.  A quad of lanes holds 8 contiguous
// columns of a row: fp32 accesses from the fragment fill whole 32-byte sectors.
#pragma once
#include "rpx_gemm.cuh"

namespace rpx {

constexpr int kWsBlockN = 256;
constexpr int kWsStages = 4;
constexpr int kWsThreads = 384;

struct WsCfg {
  static constexpr int kABytes = kBlockM * kBlockK * 2;    // 16 KB
  static constexpr int kBBytes = kWsBlockN * kBlockK * 2;  // 32 KB
  static constexpr int kStageBytes = kABytes + kBBytes;
  // ring + 1 KB alignment slack + barriers
  static constexpr size_t kSmemBytes = (size_t)kWsStages * kStageBytes + 1024 + 256;
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

// Epi must provide:
//   struct Params;                                  (trivially copyable kernel argument)
//   __device__ explicit Epi(const Params&);
//   __device__ void prefetch(const FragCtx&);       (runs while the tile's first k-block is in flight: global
//                                                    reads that do not depend on the accumulator)
//   __device__ void tile(const FragCtx&, const float (&acc)[128]);
template <class Epi>
__global__ void __launch_bounds__(kWsThreads, 1)
gemm_ws_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, int M, int N, int K,
               int tiles_m, int tiles_n, typename Epi::Params ep) {
  extern __shared__ uint8_t smem_raw[];
  // 128B swizzle needs 1024-byte aligned tile bases.
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024 - (raw_addr & 1023)) & 1023);
  uint8_t* sA = smem;
  uint8_t* sB = smem + kWsStages * WsCfg::kABytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kWsStages * WsCfg::kStageBytes);
  uint64_t* empty = full + kWsStages;

  const int warp = threadIdx.x >> 5;
  const int wg = warp >> 2;
  const int num_kb = K / kBlockK;
  const int num_tiles = tiles_m * tiles_n;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < kWsStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 2 * 128);  // every thread of both consumers
    }
    fence_mbar_init();
  }
  __syncthreads();
  // Under programmatic dependent launch (rpx_ptx.cuh) the preceding kernel may still be running: A, the row
  // scales and the residual stream are its outputs.
  pdl_launch_dependents();
  pdl_wait();

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const int m_blk = t / tiles_n, n_blk = t % tiles_n;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full[stage], WsCfg::kStageBytes);
          tma_load_2d(sA + stage * WsCfg::kABytes, &tmA, &full[stage], kb * kBlockK, m_blk * kBlockM);
          tma_load_2d(sB + stage * WsCfg::kBBytes, &tmB, &full[stage], kb * kBlockK, n_blk * kWsBlockN);
          if (++stage == kWsStages) {
            stage = 0;
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
    Epi epi(ep);
    float acc[128];
    int stage = 0;
    uint32_t phase = 0;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      FragCtx c;
      c.n_blk = t % tiles_n;
      c.m0 = (t / tiles_n) * kBlockM;
      c.n0 = c.n_blk * kWsBlockN;
      c.n_cols = N - c.n0 < kWsBlockN ? N - c.n0 : kWsBlockN;
      c.M = M;
      c.N = N;
      c.r0 = c.m0 + 64 * cw + 16 * (warp & 3) + (lane >> 2);
      c.q = lane & 3;
      int prev = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full[stage], phase);
        // +8 KB (>>4 = 512) for the second 64-row half of A; +32 bytes (>>4 = 2) per K=16 step inside the atom
        const uint64_t a_desc = make_smem_desc_kmajor_sw128(smem_u32(sA + stage * WsCfg::kABytes)) + 512 * cw;
        const uint64_t b_desc = make_smem_desc_kmajor_sw128(smem_u32(sB + stage * WsCfg::kBBytes));
        wgmma_fence_operand(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / kMmaK; ++k) wgmma_m64n256k16_ss(acc, a_desc + 2 * k, b_desc + 2 * k, (kb | k) != 0);
        wgmma_commit();
        if (kb == 0) epi.prefetch(c);
        // the group of the previous k-block has retired once at most this one is in flight: its stage is free
        if (kb > 0) {
          wgmma_wait<1>();
          mbar_arrive(&empty[prev]);
        }
        prev = stage;
        if (++stage == kWsStages) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_operand(acc);
      mbar_arrive(&empty[prev]);
      epi.tile(c, acc);
    }
  }
}

// ============================================================================ register-fragment epilogues
// Same arithmetic as EpiStoreF32 / EpiGeGLUT of rpx_gemm.cuh, element for element.

// C[m, n] = acc (fp32).  The bare core behind rpx_gemm_bf16_f32.
struct EpiWsStoreF32 {
  using Params = EpiStoreF32::Params;
  Params p;
  __device__ explicit EpiWsStoreF32(const Params& p_) : p(p_) {}
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
  Params p;
  float rs0 = 0.f, rs1 = 0.f;
  __device__ explicit EpiWsGeGLU(const Params& p_) : p(p_) {}
  __device__ void prefetch(const FragCtx& c) {
    rs0 = c.r0 < c.M ? p.rs.get(c.r0) : 0.f;
    rs1 = c.r0 + 8 < c.M ? p.rs.get(c.r0 + 8) : 0.f;
  }
  __device__ void tile(const FragCtx& c, const float (&acc)[128]) {
    __nv_bfloat16* dst = p.out + (size_t)c.r0 * p.ldo + c.n_blk * (kWsBlockN / 2) + 2 * c.q;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float* g = acc + 4 * j;
      const float* u = acc + 4 * (j + 16);
      if (c.r0 < c.M)
        *reinterpret_cast<uint32_t*>(dst + 8 * j) =
            pack_bf16x2(gelu_new(g[0] * rs0) * (u[0] * rs0), gelu_new(g[1] * rs0) * (u[1] * rs0));
      if (c.r0 + 8 < c.M)
        *reinterpret_cast<uint32_t*>(dst + 8 * (size_t)p.ldo + 8 * j) =
            pack_bf16x2(gelu_new(g[2] * rs1) * (u[2] * rs1), gelu_new(g[3] * rs1) * (u[3] * rs1));
    }
  }
};

}  // namespace rpx
