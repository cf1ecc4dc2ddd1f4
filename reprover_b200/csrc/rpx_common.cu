// rpx_common.cu — error plumbing, device info, TMA tensor-map encoding.
#include "rpx_common.cuh"

#include <cudaTypedefs.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>

namespace rpx {

static unsigned long long* g_timeline = nullptr;
static int g_timeline_slots = 0, g_timeline_next = 0;
unsigned long long* next_timeline_slot() {
  if (g_timeline == nullptr || g_timeline_next >= g_timeline_slots) return nullptr;
  return g_timeline + 8 * (size_t)(g_timeline_next++);
}

static thread_local bool g_pdl_scope = false;
void set_pdl_scope(bool on) { g_pdl_scope = on; }
bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("RPX_PDL");  // 0: never; 2: every encoder launch; default: latency path only
    v = e ? atoi(e) : 1;
  }
  return v == 2 || (v == 1 && g_pdl_scope);
}

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }

// cuTensorMapEncodeTiled is a driver entry point.  Resolving it through the
// runtime keeps libcuda.so.1 out of the link line, so the library still loads
// (and exports its symbols) on a build box with no driver installed.
static PFN_cuTensorMapEncodeTiled_v12000 resolve_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &p, 12000, cudaEnableDefault,
                                         &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  });
  return fn;
}

// cuTensorMapEncodeTiled costs a driver call per map; a single-state encode issues ~100 of them for the
// same few dozen (pointer, shape) combinations call after call.  Small per-thread 4-way set-associative cache.
namespace {
struct TmapKey {
  const void* ptr;
  uint64_t rows, cols, ld;
  uint32_t box_cols, box_rows;
  int elem, swizzle;
  bool operator==(const TmapKey& o) const {
    return ptr == o.ptr && rows == o.rows && cols == o.cols && ld == o.ld && box_cols == o.box_cols &&
           box_rows == o.box_rows && elem == o.elem && swizzle == o.swizzle;
  }
};
struct TmapSlot {
  TmapKey key{};
  bool valid = false;
  alignas(64) CUtensorMap map;
};
constexpr int kTmapSlots = 512, kTmapWays = 4;   // 128 sets x 4 ways
thread_local TmapSlot g_tmaps[kTmapSlots];
thread_local uint8_t g_tmap_next[kTmapSlots / kTmapWays];  // round-robin victim of each set
inline TmapSlot* tmap_set(const TmapKey& k) {
  uint64_t h = reinterpret_cast<uintptr_t>(k.ptr) * 0x9E3779B97F4A7C15ull;
  h ^= (k.rows * 0xC2B2AE3D27D4EB4Full) ^ (k.cols << 17) ^ (k.ld << 29) ^ ((uint64_t)k.box_rows << 41) ^
       ((uint64_t)k.box_cols << 49) ^ ((uint64_t)k.elem << 55) ^ ((uint64_t)k.swizzle << 58);
  h ^= h >> 29;
  return g_tmaps + (h % (kTmapSlots / kTmapWays)) * kTmapWays;
}
// The slot holding `k` (hit = true), or the slot to fill (an empty way, else the set's round-robin victim).
inline TmapSlot& tmap_slot(const TmapKey& k, bool* hit) {
  TmapSlot* set = tmap_set(k);
  *hit = true;
  for (int w = 0; w < kTmapWays; ++w)
    if (set[w].valid && set[w].key == k) return set[w];
  *hit = false;
  for (int w = 0; w < kTmapWays; ++w)
    if (!set[w].valid) return set[w];
  uint8_t& nxt = g_tmap_next[(set - g_tmaps) / kTmapWays];
  TmapSlot& v = set[nxt];
  nxt = (uint8_t)((nxt + 1) % kTmapWays);
  return v;
}
}  // namespace

int make_tmap_bf16_2d(CUtensorMap* out, const void* gptr, uint64_t rows, uint64_t cols,
                      uint64_t ld_elems, uint32_t box_rows) {
  const TmapKey key{gptr, rows, cols, ld_elems, 64u, box_rows, 2, 128};
  bool hit;
  TmapSlot& slot = tmap_slot(key, &hit);
  if (hit) {
    *out = slot.map;
    return RPX_OK;
  }
  RPX_TRY(make_tmap_bf16_2d_uncached(out, gptr, rows, cols, ld_elems, box_rows));
  slot.key = key;
  slot.map = *out;
  slot.valid = true;
  return RPX_OK;
}

int make_tmap_bf16_2d_uncached(CUtensorMap* out, const void* gptr, uint64_t rows, uint64_t cols,
                               uint64_t ld_elems, uint32_t box_rows) {
  auto encode = resolve_encode();
  RPX_REQUIRE(encode != nullptr, RPX_ERR_CUDA, "cuTensorMapEncodeTiled not available from driver");
  RPX_REQUIRE((reinterpret_cast<uintptr_t>(gptr) & 15) == 0, RPX_ERR_INVALID,
              "TMA operand base must be 16-byte aligned");
  RPX_REQUIRE((ld_elems * 2) % 16 == 0, RPX_ERR_INVALID, "TMA row pitch must be a multiple of 16 bytes");
  RPX_REQUIRE(box_rows >= 1 && box_rows <= 256, RPX_ERR_INVALID, "TMA box rows out of range");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld_elems * 2};
  cuuint32_t box[2] = {64, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = encode(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(gptr), dims,
                      strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                      CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  RPX_REQUIRE(r == CUDA_SUCCESS, RPX_ERR_CUDA,
              "cuTensorMapEncodeTiled failed (CUresult %d) rows=%llu cols=%llu ld=%llu", (int)r,
              (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld_elems);
  return RPX_OK;
}

int make_tmap_2d(CUtensorMap* out, int elem_bytes, const void* gptr, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                 uint32_t box_cols, uint32_t box_rows, int swizzle_bytes) {
  const TmapKey key{gptr, rows, cols, ld_elems, box_cols, box_rows, elem_bytes + 16, swizzle_bytes};
  bool hit;
  TmapSlot& slot = tmap_slot(key, &hit);
  if (hit) {
    *out = slot.map;
    return RPX_OK;
  }
  RPX_TRY(make_tmap_2d_uncached(out, elem_bytes, gptr, rows, cols, ld_elems, box_cols, box_rows, swizzle_bytes));
  slot.key = key;
  slot.map = *out;
  slot.valid = true;
  return RPX_OK;
}

int make_tmap_2d_uncached(CUtensorMap* out, int elem_bytes, const void* gptr, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                          uint32_t box_cols, uint32_t box_rows, int swizzle_bytes) {
  auto encode = resolve_encode();
  RPX_REQUIRE(encode != nullptr, RPX_ERR_CUDA, "cuTensorMapEncodeTiled not available from driver");
  RPX_REQUIRE(elem_bytes == 2 || elem_bytes == 4, RPX_ERR_INVALID, "TMA map: element size %d", elem_bytes);
  RPX_REQUIRE((reinterpret_cast<uintptr_t>(gptr) & 15) == 0, RPX_ERR_INVALID,
              "TMA operand base must be 16-byte aligned");
  RPX_REQUIRE((ld_elems * elem_bytes) % 16 == 0, RPX_ERR_INVALID, "TMA row pitch must be a multiple of 16 bytes");
  RPX_REQUIRE(box_rows >= 1 && box_rows <= 256 && box_cols >= 1 && box_cols <= 256, RPX_ERR_INVALID,
              "TMA box out of range");
  CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_NONE;
  if (swizzle_bytes == 32) sw = CU_TENSOR_MAP_SWIZZLE_32B;
  else if (swizzle_bytes == 64) sw = CU_TENSOR_MAP_SWIZZLE_64B;
  else if (swizzle_bytes == 128) sw = CU_TENSOR_MAP_SWIZZLE_128B;
  else RPX_REQUIRE(swizzle_bytes == 0, RPX_ERR_INVALID, "TMA map: swizzle span %d", swizzle_bytes);
  RPX_REQUIRE(swizzle_bytes == 0 || (int)(box_cols * elem_bytes) <= swizzle_bytes, RPX_ERR_INVALID,
              "TMA map: inner box extent exceeds the swizzle span");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld_elems * (uint64_t)elem_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = encode(out, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                      const_cast<void*>(gptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                      CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  RPX_REQUIRE(r == CUDA_SUCCESS, RPX_ERR_CUDA,
              "cuTensorMapEncodeTiled failed (CUresult %d) rows=%llu cols=%llu ld=%llu box=%ux%u", (int)r,
              (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld_elems, box_cols, box_rows);
  return RPX_OK;
}

int get_device_info(DeviceInfo* out) {
  static std::mutex mu;
  static DeviceInfo cache[64];
  int dev = -1;
  RPX_CUDA_OK(cudaGetDevice(&dev));
  RPX_REQUIRE(dev >= 0 && dev < 64, RPX_ERR_CUDA, "unexpected device ordinal %d", dev);
  std::lock_guard<std::mutex> lk(mu);
  if (cache[dev].device != dev) {
    DeviceInfo d;
    d.device = dev;
    RPX_CUDA_OK(cudaDeviceGetAttribute(&d.num_sms, cudaDevAttrMultiProcessorCount, dev));
    RPX_CUDA_OK(cudaDeviceGetAttribute(&d.cc_major, cudaDevAttrComputeCapabilityMajor, dev));
    RPX_CUDA_OK(cudaDeviceGetAttribute(&d.cc_minor, cudaDevAttrComputeCapabilityMinor, dev));
    int optin = 0;
    RPX_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    d.smem_optin = (size_t)optin;
    cache[dev] = d;
  }
  *out = cache[dev];
  RPX_REQUIRE(out->cc_major == 9 && out->cc_minor == 0, RPX_ERR_UNSUPPORTED,
              "device %d is sm_%d%d; this engine is sm_90a (H100) only", dev, out->cc_major,
              out->cc_minor);
  return RPX_OK;
}

}  // namespace rpx

extern "C" {

const char* rpx_last_error(void) { return rpx::get_error(); }
int rpx_version(void) { return RPX_VERSION; }

int rpx_debug_set_timeline(unsigned long long* d_stamps, int32_t n_slots) {
  rpx::g_timeline = d_stamps;
  rpx::g_timeline_slots = d_stamps ? n_slots : 0;
  rpx::g_timeline_next = 0;
  return RPX_OK;
}
int rpx_device_check(void) {
  rpx::DeviceInfo d;
  return rpx::get_device_info(&d);
}

}  // extern "C"
