// rpx_elementwise.cu — the HBM-bound byte / row kernels around the GEMMs:
// ByT5 tokenisation (K1 prologue), embedding gather (K1), final RMSNorm + masked
// mean-pool + L2 normalise (K2 + K10) or final RMSNorm per token (the hidden-state output),
// attention-mask validation, weight packing.
// All are coalesced, vectorised (16-byte) row streams; none is reshaped into a GEMM.
#include "rpx_common.cuh"
#include "rpx_kernels.cuh"
#include "rpx_ptx.cuh"

namespace rpx {

namespace {

// Largest s with cu[s] <= t  (cu is non-decreasing, cu[0] = 0, cu[n] > t).
__device__ __forceinline__ int find_seq(const int32_t* __restrict__ cu, int n, int t) {
  int lo = 0, hi = n;  // invariant: cu[lo] <= t < cu[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (cu[mid] <= t) lo = mid; else hi = mid;
  }
  return lo;
}

// HF ByT5Tokenizer (tokenization_byt5.py:195-208): id = byte + 3; EOS (1) appended;
// truncation keeps max_len - 1 bytes + EOS.  cu_tokens already encodes the truncation.
__global__ void tokenize_bytes_kernel(const uint8_t* __restrict__ bytes, const int64_t* __restrict__ cu_bytes,
                                      const int32_t* __restrict__ cu_tokens, int32_t* __restrict__ ids,
                                      int n_seqs, int n_tokens) {
  pdl_wait();
  pdl_launch_dependents();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_tokens) return;
  const int s = find_seq(cu_tokens, n_seqs, t);
  const int p = t - cu_tokens[s];
  const int last = cu_tokens[s + 1] - cu_tokens[s] - 1;
  ids[t] = (p == last) ? 1 : (int32_t)bytes[cu_bytes[s] + p] + 3;
}

__global__ void pack_ids_kernel(const int64_t* __restrict__ ids, const int32_t* __restrict__ cu_tokens,
                                int32_t* __restrict__ packed, int batch, int seq_len, int n_tokens,
                                int vocab, int32_t* __restrict__ bad_flag) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_tokens) return;
  const int s = find_seq(cu_tokens, batch, t);
  const int p = t - cu_tokens[s];
  const int64_t id = ids[(int64_t)s * seq_len + p];
  if (id < 0 || id >= vocab) {
    atomicOr(bad_flag, 2);
    packed[t] = 0;
  } else {
    packed[t] = (int32_t)id;
  }
}

__global__ void mask_lengths_kernel(const int64_t* __restrict__ mask, int32_t* __restrict__ lens,
                                    int32_t* __restrict__ bad_flag, int batch, int seq_len) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= batch) return;
  int cnt = 0, last = -1, bad = 0;
  for (int j = lane; j < seq_len; j += 32) {
    const int64_t m = mask[(int64_t)row * seq_len + j];
    if (m != 0 && m != 1) bad = 1;
    if (m != 0) {
      ++cnt;
      last = j;
    }
  }
  for (int off = 16; off; off >>= 1) {
    cnt += __shfl_xor_sync(0xffffffffu, cnt, off);
    last = max(last, __shfl_xor_sync(0xffffffffu, last, off));
    bad |= __shfl_xor_sync(0xffffffffu, bad, off);
  }
  if (lane == 0) {
    lens[row] = cnt;
    if (bad || cnt == 0 || cnt != last + 1) atomicOr(bad_flag, 1);
  }
}

// One warp per token.
__global__ void embed_kernel(const int32_t* __restrict__ ids, const float* __restrict__ table,
                             float* __restrict__ h32, __nv_bfloat16* __restrict__ h16, float* __restrict__ ss,
                             int ss_stride, int n_parts, int n_tokens, int d_model) {
  pdl_wait();
  pdl_launch_dependents();
  const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= n_tokens) return;
  const float4* src = reinterpret_cast<const float4*>(table + (int64_t)ids[t] * d_model);
  float4* d32 = reinterpret_cast<float4*>(h32 + (int64_t)t * d_model);
  uint2* d16 = reinterpret_cast<uint2*>(h16 + (int64_t)t * d_model);
  float acc = 0.f;
  for (int i = lane; i < d_model / 4; i += 32) {
    const float4 v = src[i];
    d32[i] = v;
    d16[i] = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
    acc += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  for (int off = 16; off; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if (lane == 0) {
    ss[t] = acc;
    for (int p = 1; p < n_parts; ++p) ss[(int64_t)p * ss_stride + t] = 0.f;
  }
}

// One CTA per sequence; thread i owns dims [4i, 4i+4).
__global__ void pool_normalize_kernel(const float* __restrict__ h32, const float* __restrict__ ss, int ss_stride,
                                      int n_parts, const float* __restrict__ ln_w,
                                      const int32_t* __restrict__ cu_tokens, void* __restrict__ out,
                                      int out_dtype, int d_model, float eps) {
  pdl_wait();
  pdl_launch_dependents();
  const int s = blockIdx.x;
  const int t0 = cu_tokens[s], t1 = cu_tokens[s + 1];
  const int i = threadIdx.x;
  const bool active = i < d_model / 4;
  const float inv_d = 1.0f / (float)d_model;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  // four tokens per trip: all loads of the trip go out before the first dependent FMA (one CTA per
  // sequence keeps only ~1.5 KB in flight per token row otherwise); accumulation order is still t0..t1
  constexpr int kU = 4;
  int t = t0;
  for (; t + kU <= t1; t += kU) {
    float4 v[kU];
    float sum[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      v[u] = active ? reinterpret_cast<const float4*>(h32 + (int64_t)(t + u) * d_model)[i]
                    : make_float4(0.f, 0.f, 0.f, 0.f);
      sum[u] = 0.f;
    }
    for (int p = 0; p < n_parts; ++p) {
#pragma unroll
      for (int u = 0; u < kU; ++u) sum[u] += ss[(int64_t)p * ss_stride + t + u];
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const float rs = rsqrtf(sum[u] * inv_d + eps);
      acc.x += v[u].x * rs;
      acc.y += v[u].y * rs;
      acc.z += v[u].z * rs;
      acc.w += v[u].w * rs;
    }
  }
  for (; t < t1; ++t) {
    float sum = 0.f;
    for (int p = 0; p < n_parts; ++p) sum += ss[(int64_t)p * ss_stride + t];
    const float rs = rsqrtf(sum * inv_d + eps);
    if (active) {
      const float4 v = reinterpret_cast<const float4*>(h32 + (int64_t)t * d_model)[i];
      acc.x += v.x * rs;
      acc.y += v.y * rs;
      acc.z += v.z * rs;
      acc.w += v.w * rs;
    }
  }
  const float inv_len = 1.0f / (float)(t1 - t0);
  float sq = 0.f;
  if (active) {
    const float4 w = reinterpret_cast<const float4*>(ln_w)[i];
    acc.x *= w.x * inv_len;
    acc.y *= w.y * inv_len;
    acc.z *= w.z * inv_len;
    acc.w *= w.w * inv_len;
    sq = acc.x * acc.x + acc.y * acc.y + acc.z * acc.z + acc.w * acc.w;
  }
  __shared__ float red[32];
  for (int off = 16; off; off >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sq;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if (threadIdx.x == 0) red[0] = v;
  }
  __syncthreads();
  // F.normalize: x / max(||x||_2, 1e-12)
  const float inv_norm = 1.0f / fmaxf(sqrtf(red[0]), 1e-12f);
  if (active) {
    acc.x *= inv_norm;
    acc.y *= inv_norm;
    acc.z *= inv_norm;
    acc.w *= inv_norm;
    if (out_dtype == RPX_DTYPE_F32) {
      reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + (int64_t)s * d_model)[i] = acc;
    } else {
      reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + (int64_t)s * d_model)[i] =
          make_uint2(pack_bf16x2(acc.x, acc.y), pack_bf16x2(acc.z, acc.w));
    }
  }
}

// Latency-path variant (one or a few sequences per call).  The kernel above walks a sequence's tokens one
// after the other in a single CTA: 56 dependent trips for a 225-token proof state, and one SM pulling the
// whole 1.3 MB of final hidden states — a tenth of the single-state encode.  Here the pooling is two short
// kernels:
//   pool_partial_kernel   one CTA per GROUP of 16 consecutive tokens of a sequence, one warp per token (lanes
//                         across the row, every 16-byte load of the row in flight at once; the row's RMSNorm
//                         partial sums fetched lane-parallel); the 16 scaled rows are added in token order and
//                         the group's row goes to `scratch[first token of the sequence + group]`;
//   pool_final_kernel     one CTA per sequence adds its group rows in group order, applies the final RMSNorm
//                         weight and the mean, L2-normalises.
// The grouping depends on the sequence alone, so a state's embedding does not depend on what it is batched
// with.  (Not bit-identical to the sequential order above, like the rest of the latency path.)
constexpr int kPoolGroup = 16;
__global__ void __launch_bounds__(kPoolGroup * 32)
pool_partial_kernel(const float* __restrict__ h32, const float* __restrict__ ss, int ss_stride, int n_parts,
                    const int32_t* __restrict__ cu_tokens, float* __restrict__ scratch, int d_model, float eps) {
  pdl_launch_dependents();
  extern __shared__ __align__(16) float part[];  // [kPoolGroup][d_model]
  const int s = blockIdx.y, g = blockIdx.x;
  const int t0 = cu_tokens[s], t1 = cu_tokens[s + 1];   // (written before the first kernel of the chain)
  if (t0 + g * kPoolGroup >= t1) return;
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n4 = d_model >> 2;
  const int t = t0 + g * kPoolGroup + warp;
  constexpr int kMaxIt = 16;  // d_model <= 16 * 32 * 4 = 2048 (checked by the launcher)
  if (t < t1) {
    const float4* row = reinterpret_cast<const float4*>(h32 + (int64_t)t * d_model);
    float4 v[kMaxIt];
#pragma unroll
    for (int i = 0; i < kMaxIt; ++i) {
      const int c = lane + 32 * i;
      v[i] = c < n4 ? row[c] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float sum = 0.f;
    for (int p = lane; p < n_parts; p += 32) sum += ss[(int64_t)p * ss_stride + t];
#pragma unroll
    for (int off = 16; off; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
    const float rs = rsqrtf(sum * (1.0f / (float)d_model) + eps);
#pragma unroll
    for (int i = 0; i < kMaxIt; ++i) {
      const int c = lane + 32 * i;
      if (c < n4)
        reinterpret_cast<float4*>(part + (size_t)warp * d_model)[c] = make_float4(v[i].x * rs, v[i].y * rs, v[i].z * rs, v[i].w * rs);
    }
  }
  __syncthreads();
  const int n_rows = min(kPoolGroup, t1 - (t0 + g * kPoolGroup));
  for (int i = threadIdx.x; i < n4; i += kPoolGroup * 32) {
    float4 tot = reinterpret_cast<const float4*>(part)[i];
    for (int w = 1; w < n_rows; ++w) {
      const float4 a = reinterpret_cast<const float4*>(part + (size_t)w * d_model)[i];
      tot.x += a.x;
      tot.y += a.y;
      tot.z += a.z;
      tot.w += a.w;
    }
    reinterpret_cast<float4*>(scratch + (int64_t)(t0 + g) * d_model)[i] = tot;
  }
}

__global__ void __launch_bounds__(512)
pool_final_kernel(const float* __restrict__ scratch, const float* __restrict__ ln_w, const int32_t* __restrict__ cu_tokens,
                  void* __restrict__ out, int out_dtype, int d_model) {
  pdl_launch_dependents();
  __shared__ float red[32];
  const int s = blockIdx.x;
  const int t0 = cu_tokens[s], t1 = cu_tokens[s + 1];
  const int n_groups = (t1 - t0 + kPoolGroup - 1) / kPoolGroup;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = threadIdx.x, n4 = d_model >> 2;
  const bool active = i < n4;
  pdl_wait();
  float4 tot = make_float4(0.f, 0.f, 0.f, 0.f);
  float sq = 0.f;
  if (active) {
    const float4* src = reinterpret_cast<const float4*>(scratch + (int64_t)t0 * d_model) + i;
    int g = 0;
    for (; g + 8 <= n_groups; g += 8) {   // eight independent loads in flight, additions in group order
      float4 a[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] = src[(size_t)(g + j) * n4];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        tot.x += a[j].x;
        tot.y += a[j].y;
        tot.z += a[j].z;
        tot.w += a[j].w;
      }
    }
    for (; g < n_groups; ++g) {
      const float4 a = src[(size_t)g * n4];
      tot.x += a.x;
      tot.y += a.y;
      tot.z += a.z;
      tot.w += a.w;
    }
    const float inv_len = 1.0f / (float)(t1 - t0);
    const float4 w4 = reinterpret_cast<const float4*>(ln_w)[i];
    tot.x *= w4.x * inv_len;
    tot.y *= w4.y * inv_len;
    tot.z *= w4.z * inv_len;
    tot.w *= w4.w * inv_len;
    sq = tot.x * tot.x + tot.y * tot.y + tot.z * tot.z + tot.w * tot.w;
  }
  for (int off = 16; off; off >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, off);
  if (lane == 0) red[warp] = sq;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if (threadIdx.x == 0) red[0] = v;
  }
  __syncthreads();
  const float inv_norm = 1.0f / fmaxf(sqrtf(red[0]), 1e-12f);  // F.normalize: x / max(||x||_2, 1e-12)
  if (active) {
    tot.x *= inv_norm;
    tot.y *= inv_norm;
    tot.z *= inv_norm;
    tot.w *= inv_norm;
    if (out_dtype == RPX_DTYPE_F32) {
      reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + (int64_t)s * d_model)[i] = tot;
    } else {
      reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(out) + (int64_t)s * d_model)[i] =
          make_uint2(pack_bf16x2(tot.x, tot.y), pack_bf16x2(tot.z, tot.w));
    }
  }
}

// Final RMSNorm of every token into a padded [batch, seq_len, d_model] output (HF T5Stack's
// `final_layer_norm`, modeling_t5.py:782, i.e. `last_hidden_state`).  One warp per output row (b, p), lanes
// across the columns, 8 columns per lane and trip (two 16-byte loads of h32 and of the weight, one 16-byte store
// of bf16 or two of fp32).  Row (b, p) holds token cu[b] + p while p < len_b and zeros past it.  The row scale
// sums the ss parts in the order of the pool kernel the forward pass would run: part after part as in
// pool_normalize_kernel, or (`lane_ss`, the latency path) lane-strided and reduced by shuffles as in
// pool_partial_kernel; then the same rsqrtf.
__global__ void hidden_store_kernel(const float* __restrict__ h32, const float* __restrict__ ss, int ss_stride,
                                    int n_parts, bool lane_ss, const float* __restrict__ ln_w,
                                    const int32_t* __restrict__ cu_tokens, void* __restrict__ out, int out_dtype,
                                    int64_t n_rows, int seq_len, int d_model, float eps) {
  pdl_wait();
  pdl_launch_dependents();
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= n_rows) return;
  const int b = (int)(row / seq_len), p = (int)(row % seq_len);
  const int t0 = cu_tokens[b], len = cu_tokens[b + 1] - t0;
  const int n8 = d_model >> 3;
  float4* o32 = reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + row * d_model);
  uint4* o16 = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(out) + row * d_model);
  if (p >= len) {
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int c = lane; c < n8; c += 32) {
      if (out_dtype == RPX_DTYPE_F32) {
        o32[2 * c] = z;
        o32[2 * c + 1] = z;
      } else {
        o16[c] = make_uint4(0u, 0u, 0u, 0u);
      }
    }
    return;
  }
  const int t = t0 + p;
  float sum = 0.f;
  if (lane_ss) {
    for (int q = lane; q < n_parts; q += 32) sum += ss[(int64_t)q * ss_stride + t];
#pragma unroll
    for (int off = 16; off; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
  } else {
    for (int q = 0; q < n_parts; ++q) sum += ss[(int64_t)q * ss_stride + t];
  }
  const float rs = rsqrtf(sum * (1.0f / (float)d_model) + eps);
  const float4* src = reinterpret_cast<const float4*>(h32 + (int64_t)t * d_model);
  const float4* w4 = reinterpret_cast<const float4*>(ln_w);
  for (int c = lane; c < n8; c += 32) {
    const float4 a = src[2 * c], bb = src[2 * c + 1];
    const float4 wa = w4[2 * c], wb = w4[2 * c + 1];
    const float4 ya = make_float4(a.x * rs * wa.x, a.y * rs * wa.y, a.z * rs * wa.z, a.w * rs * wa.w);
    const float4 yb = make_float4(bb.x * rs * wb.x, bb.y * rs * wb.y, bb.z * rs * wb.z, bb.w * rs * wb.w);
    if (out_dtype == RPX_DTYPE_F32) {
      o32[2 * c] = ya;
      o32[2 * c + 1] = yb;
    } else {
      o16[c] = make_uint4(pack_bf16x2(ya.x, ya.y), pack_bf16x2(ya.z, ya.w), pack_bf16x2(yb.x, yb.y),
                          pack_bf16x2(yb.z, yb.w));
    }
  }
}

__global__ void pack_weight_kernel(const float* __restrict__ src, const float* __restrict__ scale,
                                   __nv_bfloat16* __restrict__ dst, int n_rows, int n_cols, int dst_row0,
                                   int blk, int blk_stride) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)n_rows * n_cols) return;
  const int n = (int)(idx / n_cols), k = (int)(idx % n_cols);
  const float v = src[idx] * (scale ? scale[k] : 1.0f);
  const int64_t drow = dst_row0 + (int64_t)(n / blk) * blk_stride + (n % blk);
  dst[drow * n_cols + k] = __float2bfloat16_rn(v);
}

}  // namespace

int launch_tokenize_bytes(const uint8_t* bytes, const int64_t* cu_bytes, const int32_t* cu_tokens,
                          int32_t* ids, int n_seqs, int n_tokens, cudaStream_t stream) {
  RPX_CUDA_OK(launch_pdl(tokenize_bytes_kernel, dim3(ceil_div(n_tokens, 256)), dim3(256), 0, stream, pdl_enabled(), bytes,
                         cu_bytes, cu_tokens, ids, n_seqs, n_tokens));
  return RPX_OK;
}

int launch_pack_ids(const int64_t* ids, const int32_t* cu_tokens, int32_t* packed, int batch, int seq_len,
                    int n_tokens, int vocab, int32_t* bad_flag, cudaStream_t stream) {
  pack_ids_kernel<<<ceil_div(n_tokens, 256), 256, 0, stream>>>(ids, cu_tokens, packed, batch, seq_len, n_tokens,
                                                               vocab, bad_flag);
  RPX_CUDA_OK(cudaGetLastError());
  return RPX_OK;
}

int launch_mask_lengths(const int64_t* mask, int32_t* lens, int32_t* bad_flag, int batch, int seq_len,
                        cudaStream_t stream) {
  mask_lengths_kernel<<<ceil_div(batch, 8), 256, 0, stream>>>(mask, lens, bad_flag, batch, seq_len);
  RPX_CUDA_OK(cudaGetLastError());
  return RPX_OK;
}

int launch_embed(const int32_t* ids, const float* table, float* h32, __nv_bfloat16* h16, float* ss,
                 int ss_stride, int n_parts, int n_tokens, int d_model, cudaStream_t stream) {
  RPX_REQUIRE(d_model % 4 == 0, RPX_ERR_UNSUPPORTED, "embed: d_model must be a multiple of 4");
  RPX_CUDA_OK(launch_pdl(embed_kernel, dim3(ceil_div(n_tokens, 8)), dim3(256), 0, stream, pdl_enabled(), ids, table, h32, h16,
                         ss, ss_stride, n_parts, n_tokens, d_model));
  return RPX_OK;
}

int launch_pool_normalize(const float* h32, const float* ss, int ss_stride, int n_parts, const float* ln_w,
                          const int32_t* cu_tokens, void* out, int out_dtype, int n_seqs, int d_model,
                          float eps, cudaStream_t stream, float* group_scratch, int max_len) {
  const int threads = (int)align_up((size_t)d_model / 4, 32);
  RPX_REQUIRE(d_model % 4 == 0 && threads <= 1024, RPX_ERR_UNSUPPORTED, "pool: unsupported d_model=%d", d_model);
  RPX_REQUIRE(out_dtype == RPX_DTYPE_BF16 || out_dtype == RPX_DTYPE_F32, RPX_ERR_INVALID, "pool: bad out dtype");
  // latency path: `group_scratch` holds one fp32 row per token index (a sequence uses the first
  // ceil(len / 16) rows of its own token range)
  if (group_scratch != nullptr && d_model <= 2048 && threads <= 512 && n_seqs <= 65535) {
    const size_t smem = (size_t)kPoolGroup * d_model * sizeof(float);
    static thread_local bool configured = false;
    if (!configured) {
      RPX_CUDA_OK(cudaFuncSetAttribute(pool_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
      configured = true;
    }
    RPX_CUDA_OK(launch_pdl(pool_partial_kernel, dim3(ceil_div(max_len, kPoolGroup), n_seqs), dim3(kPoolGroup * 32), smem, stream,
                           pdl_enabled(), h32, ss, ss_stride, n_parts, cu_tokens, group_scratch, d_model, eps));
    RPX_CUDA_OK(launch_pdl(pool_final_kernel, dim3(n_seqs), dim3(threads), 0, stream, pdl_enabled(),
                           (const float*)group_scratch, ln_w, cu_tokens, out, out_dtype, d_model));
    return RPX_OK;
  }
  RPX_CUDA_OK(launch_pdl(pool_normalize_kernel, dim3(n_seqs), dim3(threads), 0, stream, pdl_enabled(), h32, ss, ss_stride,
                         n_parts, ln_w, cu_tokens, out, out_dtype, d_model, eps));
  return RPX_OK;
}

int launch_hidden_store(const float* h32, const float* ss, int ss_stride, int n_parts, bool lane_ss, const float* ln_w,
                        const int32_t* cu_tokens, void* out, int out_dtype, int batch, int seq_len, int d_model,
                        float eps, cudaStream_t stream) {
  RPX_REQUIRE(d_model % 8 == 0, RPX_ERR_UNSUPPORTED, "hidden store: d_model=%d must be a multiple of 8", d_model);
  RPX_REQUIRE(out_dtype == RPX_DTYPE_BF16 || out_dtype == RPX_DTYPE_F32, RPX_ERR_INVALID, "hidden store: bad out dtype");
  const int64_t n_rows = (int64_t)batch * seq_len;
  RPX_CUDA_OK(launch_pdl(hidden_store_kernel, dim3((unsigned)ceil_div64(n_rows, 8)), dim3(256), 0, stream, pdl_enabled(), h32,
                         ss, ss_stride, n_parts, lane_ss, ln_w, cu_tokens, out, out_dtype, n_rows, seq_len, d_model, eps));
  return RPX_OK;
}

int launch_pack_weight(const float* src, const float* scale, __nv_bfloat16* dst, int n_rows, int n_cols,
                       int dst_row0, int blk, int blk_stride, cudaStream_t stream) {
  const int64_t n = (int64_t)n_rows * n_cols;
  pack_weight_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, stream>>>(src, scale, dst, n_rows, n_cols, dst_row0,
                                                                        blk, blk_stride);
  RPX_CUDA_OK(cudaGetLastError());
  return RPX_OK;
}

}  // namespace rpx
