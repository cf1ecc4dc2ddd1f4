// rpx_gemm_launch.cuh — the host-side launchers of the two contraction cores: launch_gemm (gemm_tc_kernel, for the
// encoder's latency-path GEMMs and the similarity stages) and launch_gemm_ws (gemm_ws_kernel, for the encoder's
// throughput-path GEMMs).
#pragma once
#include "rpx_common.cuh"
#include "rpx_gemm.cuh"
#include "rpx_gemm_ws.cuh"

namespace rpx {

constexpr int kGemmStages = 4;

// Grid of the similarity stages (M_FASTEST launches, rpx_simtopk.cu).  The kernel sees M = tiles_m * 128 rows while
// the A map covers only the M real query rows: TMA zero-fills the rest and the epilogue switches them off.
struct SimGrid {
  int tiles_m;   // query blocks
  int tiles_n;   // corpus tiles visited: tiles 0, stride, 2 * stride, ... (the sampling pass) or every tile
  int stride;
  int max_ctas;  // persistent grid, a multiple of tiles_m (so every CTA keeps one query block); capped at the tiles
};

// The one launcher of gemm_tc_kernel.  A: [M, K] bf16 (row pitch lda), B: [N, K] bf16 (row pitch ldb).  K % 64 == 0.
// Encoder GEMMs (n-fastest): N % 32 == 0, a persistent grid of at most one CTA per SM, launched under PDL when the
// forward pass enables it, and one slot of the debug timeline each.  `prefetch_ptr`: the SMs the GEMM leaves idle
// fetch `prefetch_bytes` there into L2.
// Similarity stages (M_FASTEST): the grid comes from `sim`, any N (the epilogue masks the ragged tail), plain launch.
template <int BLOCK_N, class Epi, bool M_FASTEST = false, int STAGES = kGemmStages, bool SPLIT_B = false, int BM = kBlockM>
int launch_gemm(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K,
                const typename Epi::Params& ep, cudaStream_t stream, const void* prefetch_ptr = nullptr,
                size_t prefetch_bytes = 0, const SimGrid& sim = SimGrid{}) {
  using Cfg = GemmCfg<BLOCK_N, STAGES, BM>;
  static_assert(BM == kBlockM || !M_FASTEST, "64-row tiles: encoder GEMMs only");
  RPX_REQUIRE(M > 0 && N > 0 && K > 0, RPX_ERR_INVALID, "gemm: empty problem M=%d N=%d K=%d", M, N, K);
  RPX_REQUIRE(K % kBlockK == 0, RPX_ERR_UNSUPPORTED, "gemm: K=%d must be a multiple of %d", K, kBlockK);
  RPX_REQUIRE(M_FASTEST || N % 32 == 0, RPX_ERR_UNSUPPORTED, "gemm: N=%d must be a multiple of 32", N);
  DeviceInfo dev;
  RPX_TRY(get_device_info(&dev));
  CUtensorMap tmA, tmB;
  RPX_TRY(make_tmap_bf16_2d(&tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, BM));
  RPX_TRY(make_tmap_bf16_2d(&tmB, B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, SPLIT_B ? BLOCK_N / 2 : BLOCK_N));
  RPX_REQUIRE(!SPLIT_B || N % BLOCK_N == 0, RPX_ERR_UNSUPPORTED, "gemm: split-B tiles need N %% %d == 0", BLOCK_N);
  const size_t smem = Cfg::smem_bytes(Epi::kSmemBytes);
  RPX_REQUIRE(smem <= dev.smem_optin, RPX_ERR_UNSUPPORTED, "gemm: needs %zu B smem, device allows %zu",
              smem, dev.smem_optin);
  auto kern = gemm_tc_kernel<BLOCK_N, STAGES, Epi, M_FASTEST, SPLIT_B, BM>;
  static thread_local int configured_dev = -1;  // per-instantiation, per-thread
  if (configured_dev != dev.device) {
    RPX_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured_dev = dev.device;
  }
  if (M_FASTEST) {
    const int64_t tiles = (int64_t)sim.tiles_m * sim.tiles_n;
    const int grid = tiles < sim.max_ctas ? (int)tiles : sim.max_ctas;
    RPX_CUDA_OK(launch_pdl(kern, dim3(grid), dim3(kGemmThreads), smem, stream, false, tmA, tmB, sim.tiles_m * BM, N, K,
                           sim.tiles_m, sim.tiles_n, sim.stride, ep, L2Prefetch{nullptr, 0u, grid, nullptr}));
    return RPX_OK;
  }
  const int tiles_m = ceil_div(M, BM);
  const int tiles_n = ceil_div(N, BLOCK_N);
  int grid = tiles_m * tiles_n;
  if (grid > dev.num_sms) grid = dev.num_sms;
  L2Prefetch pf{prefetch_ptr, (uint32_t)prefetch_bytes, grid, next_timeline_slot()};
  if (prefetch_ptr != nullptr && prefetch_bytes > 0 && prefetch_bytes < ((size_t)1 << 32) && grid < dev.num_sms)
    grid = dev.num_sms;  // surplus SMs run prefetch helpers
  RPX_CUDA_OK(launch_pdl(kern, dim3(grid), dim3(kGemmThreads), smem, stream, pdl_enabled(), tmA, tmB, M, N, K, tiles_m,
                         tiles_n, 1, ep, pf));
  return RPX_OK;
}

// The form of the throughput core the FFN up-projection runs (rpx_encoder.cu, ffn_up_gemm), which the bare entry
// rpx_gemm_bf16_f32 runs as well.
constexpr int kFfnUpStages = 4;
constexpr int kFfnUpCluster = 2;

// Throughput core (gemm_ws_kernel): 128 x 256 tiles, persistent over one CTA per SM, a STAGES-deep operand ring;
// CLUSTER = 2 runs clusters of two CTAs on vertically adjacent tiles that share the B tile by TMA multicast.
// A: [M, K] bf16 (row pitch lda), B: [N, K] bf16 (row pitch ldb).  K % 64 == 0, N % 32 == 0.
// Residual epilogues (Epi::kResBufs > 0) stream ep.h32 ([M, N] fp32, row pitch ep.ld) through TMA.
template <class Epi, int STAGES, int CLUSTER>
int launch_gemm_ws(const void* A, int64_t lda, const void* B, int64_t ldb, int M, int N, int K,
                   const typename Epi::Params& ep, cudaStream_t stream) {
  RPX_REQUIRE(M > 0 && N > 0 && K > 0, RPX_ERR_INVALID, "gemm: empty problem M=%d N=%d K=%d", M, N, K);
  RPX_REQUIRE(K % kBlockK == 0, RPX_ERR_UNSUPPORTED, "gemm: K=%d must be a multiple of %d", K, kBlockK);
  RPX_REQUIRE(N % 32 == 0, RPX_ERR_UNSUPPORTED, "gemm: N=%d must be a multiple of 32", N);
  DeviceInfo dev;
  RPX_TRY(get_device_info(&dev));
  CUtensorMap tmA, tmB, tmR;
  RPX_TRY(make_tmap_bf16_2d(&tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, kBlockM));
  // (each CTA of a pair loads one half of the B tile)
  RPX_TRY(make_tmap_bf16_2d(&tmB, B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, kWsBlockN / CLUSTER));
  if constexpr (Epi::kResBufs > 0)
    RPX_TRY(make_tmap_2d(&tmR, 4, ep.h32, (uint64_t)M, (uint64_t)N, (uint64_t)ep.ld, kResChunkCols, 64, 128));
  else
    tmR = tmA;  // not read
  const int tiles_m = ceil_div(M, kBlockM);
  const int tiles_n = ceil_div(N, kWsBlockN);
  const size_t smem = WsCfg<STAGES, Epi::kResBufs>::kSmemBytes;
  RPX_REQUIRE(smem <= dev.smem_optin, RPX_ERR_UNSUPPORTED, "gemm: needs %zu B smem, device allows %zu", smem,
              dev.smem_optin);
  auto kern = gemm_ws_kernel<Epi, STAGES, CLUSTER>;
  static thread_local int configured_dev = -1;  // per-instantiation, per-thread
  static thread_local int max_clusters = 0;     // co-resident clusters of this instantiation on that device
  if (configured_dev != dev.device) {
    RPX_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(CLUSTER * dev.num_sms);
    cfg.blockDim = dim3(kWsThreads);
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = CLUSTER;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    RPX_CUDA_OK(cudaOccupancyMaxActiveClusters(&max_clusters, kern, &cfg));
    RPX_REQUIRE(max_clusters > 0, RPX_ERR_UNSUPPORTED, "gemm: no cluster of %d CTAs with %zu B smem fits the device",
                CLUSTER, smem);
    configured_dev = dev.device;
  }
  int clusters = ceil_div(tiles_m, CLUSTER) * tiles_n;  // work units
  if (clusters > max_clusters) clusters = max_clusters;
  RPX_CUDA_OK(launch_pdl<CLUSTER>(kern, dim3(CLUSTER * clusters), dim3(kWsThreads), smem, stream, pdl_enabled(), tmA,
                                  tmB, tmR, M, N, K, tiles_m, tiles_n, ep));
  return RPX_OK;
}

}  // namespace rpx
