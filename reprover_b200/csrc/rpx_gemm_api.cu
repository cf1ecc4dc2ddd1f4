// rpx_gemm_api.cu — test entry points for the bare contraction cores: rpx_gemm_bf16_f32 runs the throughput core
// (gemm_ws_kernel), rpx_gemm1_bf16_f32 the single-CTA form of gemm_tc_kernel, rpx_gemm2_bf16_f32 its paired form.
#include "rpx_gemm_launch.cuh"

extern "C" int rpx_gemm_bf16_f32(const void* d_A, const void* d_B, float* d_C, int32_t M, int32_t N,
                                 int32_t K, void* stream) {
  using namespace rpx;
  RPX_REQUIRE(d_A && d_B && d_C, RPX_ERR_INVALID, "rpx_gemm_bf16_f32: null pointer");
  EpiWsStoreF32::Params ep{d_C, N};
  return launch_gemm_ws<EpiWsStoreF32, kFfnUpStages, kFfnUpCluster>(d_A, K, d_B, K, M, N, K, ep,
                                                                   static_cast<cudaStream_t>(stream));
}

extern "C" int rpx_gemm1_bf16_f32(const void* d_A, const void* d_B, float* d_C, int32_t M, int32_t N, int32_t K,
                                  void* stream) {
  using namespace rpx;
  RPX_REQUIRE(d_A && d_B && d_C, RPX_ERR_INVALID, "rpx_gemm1_bf16_f32: null pointer");
  EpiStoreF32::Params ep{d_C, N};
  return launch_gemm<128, EpiStoreF32>(d_A, K, d_B, K, M, N, K, ep, static_cast<cudaStream_t>(stream));
}

extern "C" int rpx_gemm2_bf16_f32(const void* d_A, const void* d_B, float* d_C, int32_t M, int32_t N, int32_t K,
                                  void* stream) {
  using namespace rpx;
  RPX_REQUIRE(d_A && d_B && d_C, RPX_ERR_INVALID, "rpx_gemm2_bf16_f32: null pointer");
  EpiStoreF32::Params ep{d_C, N};
  return launch_gemm_pair<EpiStoreF32>(d_A, K, d_B, K, M, N, K, ep, static_cast<cudaStream_t>(stream));
}
