// rpx_attention.cu — T5 self-attention over packed variable-length sequences on wgmma.
//
// Replaces HF T5Attention.forward (modeling_t5.py:253-344; SURVEY.md §2.1 K4-K7):
//   scores = q k^T            (NO 1/sqrt(d) scaling in T5)
//          + position_bias    (bucketed relative bias, shared by all layers; K5)
//          + padding mask     (packed layout: keys simply stop at the sequence end)
//   out    = softmax_fp32(scores) v, heads merged to [T, heads*64]
// without ever materialising the [B, heads, L, L] score tensor.
//
// One CTA per (64-query tile, head, sequence), 160 threads:
//   warps 0-3  one warpgroup: per 64-key step S = Q K^T (wgmma m64n64k16 x4, Q and K from shared memory,
//              S in registers), bias + key mask + online softmax in fp32 on the registers (a query row is
//              spread over the four lanes of a quad), then O += P V (wgmma m64n64k16 x4 with P as the
//              register A operand and V as the MN-major B operand straight from the [keys, 64] tile TMA
//              delivered).  O stays in registers until the end.
//   warp 4     one elected thread: TMA loads of Q once and of K / V tile by tile into a double buffer
//              (tensor maps over the packed qkv activation matrix, box 64 columns x 64 rows).
// Small tiles keep many CTAs per state on the latency path and several CTAs per SM, which hide each
// other's softmax behind their tensor-core work.
#include "rpx_common.cuh"
#include "rpx_kernels.cuh"
#include "rpx_ptx.cuh"

namespace rpx {

namespace {

constexpr int kHD = 64;    // head dim (d_kv)
constexpr int kQT = 64;    // query rows per CTA (wgmma M)
constexpr int kKT = 64;    // keys per step (wgmma N for S, K extent for PV)
constexpr int kAttnThreads = 160;  // one warpgroup + one TMA warp
constexpr int kTileBytes = 64 * 128;  // [64 rows][64 bf16], 128B-swizzled

// smem map (bytes, 1024-aligned base): Q | K[2] | V[2] | bias | barriers
constexpr int kOffQ = 0;
constexpr int kOffK = kTileBytes;
constexpr int kOffV = 3 * kTileBytes;
constexpr int kOffBias = 5 * kTileBytes;

__host__ __device__ constexpr int bias_floats(int R) { return ((2 * R + 1) + 3) & ~3; }
size_t attention_smem_bytes(int R) { return 1024 + kOffBias + (size_t)bias_floats(R) * 4 + 64; }

// 2^x on the SFU (one MUFU.EX2; -inf -> 0, denormal results flushed).
RPX_DEVICE float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__global__ void __launch_bounds__(kAttnThreads, 2)
t5_attention_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_kv,
                    __nv_bfloat16* __restrict__ out, const int32_t* __restrict__ cu_seqlens,
                    const float* __restrict__ bias_lut, int n_heads, int R, int ld_out) {
  const int seq = blockIdx.z, head = blockIdx.y, qt = blockIdx.x;
  // Under programmatic dependent launch this CTA may start while the QKV projection is still running.
  // cu_seqlens and bias_lut were complete before the first kernel of the chain started, so the whole
  // prologue (bias table, barriers) runs ahead; only the TMA loads of q / k / v wait for the predecessor
  // (pdl_wait below).  The MMA warps touch global memory only to store `out`, after consuming those loads.
  pdl_launch_dependents();
  const int t0 = cu_seqlens[seq];
  const int len = cu_seqlens[seq + 1] - t0;
  const int q0 = qt * kQT;
  if (q0 >= len) return;  // whole CTA

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024 - (raw & 1023)) & 1023);
  float* sBias = reinterpret_cast<float*>(smem + kOffBias);
  const int lut_w = 2 * R + 1;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBias + bias_floats(R) * 4);
  uint64_t* bar_q = bars + 0;
  uint64_t* bar_k = bars + 1;     // [2]
  uint64_t* bar_v = bars + 3;     // [2]
  uint64_t* bar_free = bars + 5;  // [2]: K / V buffer consumed by the warpgroup

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int inner = n_heads * kHD;
  const int n_kt = (len + kKT - 1) / kKT;

  for (int i = threadIdx.x; i < lut_w; i += kAttnThreads) sBias[i] = bias_lut[head * lut_w + i];
  if (warp == 4) {
    if (elect_one()) {
      mbar_init(bar_q, 1);
      for (int b = 0; b < 2; ++b) {
        mbar_init(&bar_k[b], 1);
        mbar_init(&bar_v[b], 1);
        mbar_init(&bar_free[b], 128);
      }
      fence_mbar_init();
    }
    __syncwarp();
  }
  __syncthreads();

  if (warp == 4) {
    // ------------------------------------------------------------------ TMA producer (one thread)
    if (elect_one()) {
      const int kcol = inner + head * kHD, vcol = 2 * inner + head * kHD;
      pdl_wait();
      mbar_arrive_expect_tx(bar_q, kTileBytes);
      tma_load_2d(smem + kOffQ, &tm_q, bar_q, head * kHD, t0 + q0);
      for (int kt = 0; kt < n_kt; ++kt) {
        const int b = kt & 1;
        if (kt >= 2) mbar_wait<0>(&bar_free[b], ((kt >> 1) - 1) & 1);
        mbar_arrive_expect_tx(&bar_k[b], kTileBytes);
        tma_load_2d(smem + kOffK + b * kTileBytes, &tm_kv, &bar_k[b], kcol, t0 + kt * kKT);
        mbar_arrive_expect_tx(&bar_v[b], kTileBytes);
        tma_load_2d(smem + kOffV + b * kTileBytes, &tm_kv, &bar_v[b], vcol, t0 + kt * kKT);
      }
    }
  } else {
    // ------------------------------------------------------------------ softmax / MMA warpgroup
    // this thread's two query rows (wgmma accumulator layout, rpx_ptx.cuh) and its column pairs
    const int g = lane >> 2, cq = 2 * (lane & 3);
    const int qpos0 = q0 + warp * 16 + g, qpos1 = qpos0 + 8;
    const float kLog2e = 1.4426950408889634f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    const uint64_t q_desc = make_smem_desc_kmajor_sw128(smem_u32(smem + kOffQ));
    mbar_wait<0>(bar_q, 0);
    for (int kt = 0; kt < n_kt; ++kt) {
      const int b = kt & 1;
      const uint32_t ph = (kt >> 1) & 1;
      const int kb = kt * kKT;
      float sc[32];
      mbar_wait<0>(&bar_k[b], ph);
      {
        const uint64_t k_desc = make_smem_desc_kmajor_sw128(smem_u32(smem + kOffK + b * kTileBytes));
        wgmma_fence_operand(sc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kHD / 16; ++k) wgmma_m64n64k16_ss(sc, q_desc + 2 * k, k_desc + 2 * k, k != 0);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_operand(sc);
      }
      // bias + key mask, row maxima
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int key = kb + 8 * j + cq + e;
          const bool ok = key < len;
          const float b0 = sBias[min(max(key - qpos0 + R, 0), 2 * R)];
          const float b1 = sBias[min(max(key - qpos1 + R, 0), 2 * R)];
          sc[4 * j + e] = ok ? sc[4 * j + e] + b0 : -INFINITY;
          sc[4 * j + 2 + e] = ok ? sc[4 * j + 2 + e] + b1 : -INFINITY;
          mx0 = fmaxf(mx0, sc[4 * j + e]);
          mx1 = fmaxf(mx1, sc[4 * j + 2 + e]);
        }
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      // key 0 of the sequence lies in the first step, so the running maxima are finite from then on
      const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
      const float scale0 = fast_exp2((m0 - mn0) * kLog2e), scale1 = fast_exp2((m1 - mn1) * kLog2e);  // 0 on the first step
      m0 = mn0;
      m1 = mn1;
      const float mb0 = mn0 * kLog2e, mb1 = mn1 * kLog2e;
      // P = exp(s - m) as the bf16 A operand of P V: k16 chunk c = accumulator columns [16c, 16c + 16)
      uint32_t pa[4][4];
      float ls0 = 0.f, ls1 = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float p00 = fast_exp2(fmaf(sc[4 * j], kLog2e, -mb0));
        const float p01 = fast_exp2(fmaf(sc[4 * j + 1], kLog2e, -mb0));
        const float p10 = fast_exp2(fmaf(sc[4 * j + 2], kLog2e, -mb1));
        const float p11 = fast_exp2(fmaf(sc[4 * j + 3], kLog2e, -mb1));
        ls0 += p00 + p01;
        ls1 += p10 + p11;
        pa[j >> 1][(j & 1) * 2] = pack_bf16x2(p00, p01);
        pa[j >> 1][(j & 1) * 2 + 1] = pack_bf16x2(p10, p11);
      }
      l0 = l0 * scale0 + ls0;  // this lane's share of the row sum (the quad is summed at the end)
      l1 = l1 * scale1 + ls1;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[4 * j] *= scale0;
        o[4 * j + 1] *= scale0;
        o[4 * j + 2] *= scale1;
        o[4 * j + 3] *= scale1;
      }
      mbar_wait<0>(&bar_v[b], ph);
      {
        const uint32_t v_base = smem_u32(smem + kOffV + b * kTileBytes);
        wgmma_fence_operand(o);
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < kKT / 16; ++c)  // 16 keys = two 8-row groups = 2048 B of V per step
          wgmma_m64n64k16_rs_bmn(o, pa[c], make_smem_desc_mnmajor_sw128(v_base + c * 2048), 1);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_operand(o);
      }
      mbar_arrive(&bar_free[b]);
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float inv0 = 1.f / l0, inv1 = 1.f / l1;
    __nv_bfloat16* dst0 = out + (int64_t)(t0 + qpos0) * ld_out + head * kHD + cq;
    __nv_bfloat16* dst1 = out + (int64_t)(t0 + qpos1) * ld_out + head * kHD + cq;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (qpos0 < len) *reinterpret_cast<uint32_t*>(dst0 + 8 * j) = pack_bf16x2(o[4 * j] * inv0, o[4 * j + 1] * inv0);
      if (qpos1 < len) *reinterpret_cast<uint32_t*>(dst1 + 8 * j) = pack_bf16x2(o[4 * j + 2] * inv1, o[4 * j + 3] * inv1);
    }
  }
}

}  // namespace

int launch_t5_attention(const __nv_bfloat16* qkv, __nv_bfloat16* out, const int32_t* cu_seqlens,
                        const float* bias_lut, int n_tokens, int n_seqs, int max_len, int n_heads, int d_kv,
                        int max_distance, cudaStream_t stream) {
  RPX_REQUIRE(d_kv == kHD, RPX_ERR_UNSUPPORTED, "attention: d_kv=%d (only 64 is implemented)", d_kv);
  RPX_REQUIRE(n_seqs > 0 && max_len > 0 && n_tokens > 0, RPX_ERR_INVALID, "attention: empty batch");
  RPX_REQUIRE(n_seqs <= 65535 && n_heads <= 65535, RPX_ERR_UNSUPPORTED, "attention: grid limits exceeded");
  const int inner = n_heads * d_kv;
  DeviceInfo dev;
  RPX_TRY(get_device_info(&dev));
  CUtensorMap tm_q, tm_kv;
  RPX_TRY(make_tmap_bf16_2d(&tm_kv, qkv, (uint64_t)n_tokens, (uint64_t)3 * inner, (uint64_t)3 * inner, kKT));
  RPX_TRY(make_tmap_bf16_2d(&tm_q, qkv, (uint64_t)n_tokens, (uint64_t)3 * inner, (uint64_t)3 * inner, kQT));
  const size_t smem = attention_smem_bytes(max_distance);
  RPX_REQUIRE(smem <= 100 * 1024, RPX_ERR_UNSUPPORTED, "attention: bias table too large (%zu B of shared memory)", smem);
  static thread_local int configured = -1;
  if (configured != dev.device) {
    RPX_CUDA_OK(cudaFuncSetAttribute(t5_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    configured = dev.device;
  }
  const dim3 grid((max_len + kQT - 1) / kQT, n_heads, n_seqs);
  RPX_CUDA_OK(launch_pdl(t5_attention_kernel, grid, dim3(kAttnThreads), smem, stream, pdl_enabled(), tm_q, tm_kv, out,
                         cu_seqlens, bias_lut, n_heads, max_distance, inner));
  return RPX_OK;
}

}  // namespace rpx
