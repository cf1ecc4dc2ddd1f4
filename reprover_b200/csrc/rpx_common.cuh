// rpx_common.cuh — host-side plumbing shared by every translation unit:
// error codes + thread-local last-error string, CUDA call checking, the TMA
// tensor-map encoder (resolved from the driver at run time so the library loads
// on a machine without libcuda.so.1), device property cache.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/rpx.h"

namespace rpx {

// Thread-local message behind rpx_last_error().
void set_error(const char* fmt, ...);
const char* get_error();

#define RPX_CUDA_OK(expr)                                                                  \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) {                                                               \
      ::rpx::set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr,                  \
                       cudaGetErrorString(_e));                                            \
      return RPX_ERR_CUDA;                                                                 \
    }                                                                                      \
  } while (0)

#define RPX_REQUIRE(cond, code, ...)   \
  do {                                 \
    if (!(cond)) {                     \
      ::rpx::set_error(__VA_ARGS__);   \
      return (code);                   \
    }                                  \
  } while (0)

#define RPX_TRY(expr)            \
  do {                           \
    int _s = (expr);             \
    if (_s != RPX_OK) return _s; \
  } while (0)

// Encodes a 2-D row-major bf16 tensor [rows, cols] (cols contiguous, row pitch
// `ld_elems`) as a TMA map with a {box_cols=64, box_rows} box and 128-byte swizzle.
// Out-of-bounds box elements are zero-filled.
int make_tmap_bf16_2d(CUtensorMap* out, const void* gptr, uint64_t rows, uint64_t cols,
                      uint64_t ld_elems, uint32_t box_rows);
// (both map builders keep a small per-thread cache of encoded maps; the _uncached forms always call the driver)
int make_tmap_bf16_2d_uncached(CUtensorMap* out, const void* gptr, uint64_t rows, uint64_t cols,
                               uint64_t ld_elems, uint32_t box_rows);

// General 2-D row-major map: `elem_bytes` 2 (bf16) or 4 (fp32), box {box_cols, box_rows}, swizzle span
// `swizzle_bytes` in {0, 32, 64, 128} (box_cols * elem_bytes must not exceed it when non-zero).
int make_tmap_2d(CUtensorMap* out, int elem_bytes, const void* gptr, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                 uint32_t box_cols, uint32_t box_rows, int swizzle_bytes);
int make_tmap_2d_uncached(CUtensorMap* out, int elem_bytes, const void* gptr, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                          uint32_t box_cols, uint32_t box_rows, int swizzle_bytes);
int make_tmap_2d_uncached(CUtensorMap* out, int elem_bytes, const void* gptr, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                          uint32_t box_cols, uint32_t box_rows, int swizzle_bytes);

struct DeviceInfo {
  int device = -1;
  int num_sms = 0;
  int cc_major = 0, cc_minor = 0;
  size_t smem_optin = 0;
};
// Properties of the current device (cached per device ordinal).  Fails unless sm_90.
int get_device_info(DeviceInfo* out);

// Debug timeline (rpx_debug_set_timeline): each 1-CTA GEMM launch gets the next 8-stamp slot of the buffer.
unsigned long long* next_timeline_slot();

// Programmatic dependent launch is used along the kernel chain of encode calls of up to 16 k tokens (the
// kernels are short and their prologues are worth overlapping); full re-indexing chunks are launched
// plainly (their kernels are long enough that the overlap does not pay).  RPX_PDL=0 never, RPX_PDL=2 every encoder launch.
bool pdl_enabled();
void set_pdl_scope(bool on);  // per thread: true while such a forward enqueues its kernels

// Kernel launch with (optionally) the programmatic-stream-serialization attribute; see rpx_ptx.cuh.  CLUSTER > 1
// launches clusters of that many CTAs along x (grid.x must be a multiple of it).
template <int CLUSTER = 1, typename Kern, typename... Args>
inline cudaError_t launch_pdl(Kern kern, dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[2];
  int n = 0;
  if (CLUSTER > 1) {
    at[n].id = cudaLaunchAttributeClusterDimension;
    at[n].val.clusterDim.x = CLUSTER;
    at[n].val.clusterDim.y = 1;
    at[n].val.clusterDim.z = 1;
    ++n;
  }
  if (pdl) {
    at[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = at;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kern, args...);
}

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }
inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

}  // namespace rpx
