// rpx_index.cu — the index handle and the similarity + top-k entry points of the C ABI.
//
// `rpx_index` stands where the reference keeps `self.corpus_embeddings` (retrieval/model.py:190,
// 363-366): a [n, d] bf16 matrix that is written once by reindex_corpus and then queried by every
// retrieve().  Creating the handle runs the one pass that depends only on the matrix (the row-norm
// bound of the exactness guard); `rpx_index_topk` is `Corpus.get_nearest_premises`' device half
// (common.py:307-322) and picks one of three paths:
//     nq <= 2            rpx_smallq.cu   one HBM-bound streaming kernel (the reference's real call: nq = 1)
//     otherwise          rpx_simtopk.cu  wgmma with the top-k fused into the epilogue
//     k > 200 or flagged rpx_exact.cu    exact fp64 pass (always launched; returns at once if idle)
#include <stdlib.h>

#include <new>

#include "rpx_common.cuh"
#include "rpx_kernels.cuh"
#include "rpx_topk_common.cuh"

struct rpx_index {
  const __nv_bfloat16* E;
  int64_t n;
  int d;
  rpx::IndexState* state;
};

namespace rpx {
namespace {

constexpr size_t kStateBytes = 256;
constexpr int kMaxSmsForSizing = 160;  // workspace queries work without a device

int small_q_max() {
  static int v = -1;
  if (v < 0) {
    // Largest nq routed to the streaming kernel (0..4; RPX_SMALLQ_MAX overrides, tools/topk_bench.py times every
    // path by query count).  One or two queries leave the streaming kernel HBM-bound; from three on it needs a
    // second pass, and the FMA work of several queries per index byte is what a tensor core is for.
    const char* e = getenv("RPX_SMALLQ_MAX");
    v = e ? atoi(e) : 2;
    if (v < 0) v = 0;
    if (v > 4) v = 4;
  }
  return v;
}

struct WsLayout {
  size_t flagged, bounds, cand, path, total;
};

WsLayout ws_layout(int64_t n, int nq, int k, int d, int num_sms) {
  WsLayout L{};
  size_t off = 0;
  auto take = [&](size_t bytes) {
    size_t o = off;
    off = align_up(off + bytes, 256);
    return o;
  };
  L.flagged = take((size_t)nq * sizeof(uint32_t));
  L.bounds = take((size_t)nq * sizeof(ExactBound));
  L.cand = take(exact_cand_bytes(n));
  size_t path = smallq_workspace_bytes(num_sms);
  if (k <= kFastPathMaxK) {
    // the plan shrinks with d (shared-memory limits); size for the narrowest legal d as well
    const size_t m1 = mma_topk_workspace_bytes(nq, k, d, num_sms), m2 = mma_topk_workspace_bytes(nq, k, 64, num_sms);
    if (m1 > path) path = m1;
    if (m2 > path) path = m2;
  }
  L.path = take(path);
  L.total = off;
  return L;
}

int topk_dispatch(const rpx_index* ix, const void* d_Q, int32_t nq, int32_t k, const uint32_t* d_access_mask,
                  int64_t mask_stride_words, float* d_out_scores, double* d_out_scores64, int64_t* d_out_idx,
                  int32_t* d_out_count, int64_t* d_out_packed, int64_t idx_offset, int32_t flags, void* d_workspace,
                  size_t workspace_bytes, void* stream) {
  RPX_REQUIRE(ix && d_Q && d_out_scores && d_out_idx && d_workspace, RPX_ERR_INVALID, "top-k: null argument");
  RPX_REQUIRE(nq >= 1, RPX_ERR_INVALID, "top-k: nq=%d", nq);
  RPX_REQUIRE(k >= 1 && k <= 1024, RPX_ERR_UNSUPPORTED, "top-k: k=%d outside [1, 1024]", k);
  RPX_REQUIRE(ix->d > 0 && ix->d % 64 == 0 && ix->d <= 8192, RPX_ERR_UNSUPPORTED,
              "top-k: d=%d must be a multiple of 64 (<= 8192)", ix->d);
  RPX_REQUIRE(ix->n >= 0 && ix->n < (int64_t)INT32_MAX - 512, RPX_ERR_UNSUPPORTED, "top-k: n=%lld out of range",
              (long long)ix->n);
  RPX_REQUIRE(d_access_mask == nullptr || mask_stride_words * 32 >= ix->n, RPX_ERR_INVALID, "top-k: mask stride too small");
  RPX_REQUIRE((reinterpret_cast<uintptr_t>(d_workspace) & 255) == 0, RPX_ERR_INVALID, "workspace must be 256-byte aligned");
  DeviceInfo dev;
  RPX_TRY(get_device_info(&dev));
  const WsLayout L = ws_layout(ix->n, nq, k, ix->d, dev.num_sms);
  RPX_REQUIRE(L.total <= workspace_bytes, RPX_ERR_WORKSPACE, "top-k: workspace %zu < %zu", workspace_bytes, L.total);
  uint8_t* base = static_cast<uint8_t*>(d_workspace);
  TopkCall c;
  c.Q = static_cast<const __nv_bfloat16*>(d_Q);
  c.nq = nq;
  c.E = ix->E;
  c.n = ix->n;
  c.d = ix->d;
  c.k = k;
  c.mask = d_access_mask;
  c.mask_stride = mask_stride_words;
  c.out_scores = d_out_scores;
  c.out_scores64 = d_out_scores64;
  c.out_idx = d_out_idx;
  c.out_count = d_out_count;
  c.out_packed = d_out_packed;
  c.idx_offset = idx_offset;
  c.state = ix->state;
  c.flagged = reinterpret_cast<uint32_t*>(base + L.flagged);
  c.bounds = reinterpret_cast<ExactBound*>(base + L.bounds);
  c.st = static_cast<cudaStream_t>(stream);
  void* cand_ws = base + L.cand;
  void* path_ws = base + L.path;

  int path = 0;  // 1 tensor core, 2 streaming, 4 exact
  if (flags & RPX_TOPK_FORCE_EXACT) path = 4;
  else if (flags & RPX_TOPK_FORCE_STREAM) path = 2;
  else if (flags & RPX_TOPK_FORCE_MMA) path = 1;
  else if (k > kFastPathMaxK) path = 4;
  else if (ix->n > 0 && nq <= small_q_max() && smallq_supported(nq, k, ix->d)) path = 2;
  else path = 1;
  if (path == 2) {
    RPX_REQUIRE(ix->n > 0 && smallq_supported(nq, k, ix->d), RPX_ERR_UNSUPPORTED,
                "top-k: the streaming path takes 1..4 queries, k <= %d, d <= 2048, n > 0", kFastPathMaxK);
    RPX_TRY(launch_smallq_topk(c, path_ws, topk_n_res(k)));
  } else if (path == 1) {
    RPX_REQUIRE(k <= kFastPathMaxK, RPX_ERR_UNSUPPORTED, "top-k: the tensor-core path takes k <= %d", kFastPathMaxK);
    RPX_TRY(run_mma_topk(c, path_ws, workspace_bytes - L.path));
  }
  // exact pass: every query when it is the chosen path, otherwise only what the guard flagged
  return launch_exact_topk(c, cand_ws, path == 4);
}

}  // namespace
}  // namespace rpx

using namespace rpx;

extern "C" {

size_t rpx_index_state_bytes(void) { return kStateBytes; }

int rpx_index_create(const void* d_E, int64_t n, int32_t d, void* d_state, void* stream, rpx_index** out) {
  RPX_REQUIRE(out && d_state, RPX_ERR_INVALID, "rpx_index_create: null argument");
  RPX_REQUIRE(d_E != nullptr || n == 0, RPX_ERR_INVALID, "rpx_index_create: null matrix");
  RPX_REQUIRE(n >= 0 && d > 0 && d % 8 == 0, RPX_ERR_INVALID, "rpx_index_create: n=%lld d=%d", (long long)n, d);
  RPX_REQUIRE((reinterpret_cast<uintptr_t>(d_E) & 15) == 0 && (reinterpret_cast<uintptr_t>(d_state) & 15) == 0,
              RPX_ERR_INVALID, "rpx_index_create: pointers must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RPX_CUDA_OK(cudaMemsetAsync(d_state, 0, kStateBytes, st));
  RPX_TRY(launch_row_norm_max(static_cast<const __nv_bfloat16*>(d_E), n, d, static_cast<IndexState*>(d_state), st));
  rpx_index* ix = new (std::nothrow) rpx_index();
  RPX_REQUIRE(ix != nullptr, RPX_ERR_INVALID, "out of host memory");
  ix->E = static_cast<const __nv_bfloat16*>(d_E);
  ix->n = n;
  ix->d = d;
  ix->state = static_cast<IndexState*>(d_state);
  *out = ix;
  return RPX_OK;
}

int rpx_index_destroy(rpx_index* ix) {
  delete ix;
  return RPX_OK;
}

int rpx_index_stats(rpx_index* ix, void* stream, float* h_norm_max, float* h_max_err, float* h_max_eps,
                    int64_t* h_n_exact) {
  RPX_REQUIRE(ix, RPX_ERR_INVALID, "rpx_index_stats: null handle");
  IndexState s;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RPX_CUDA_OK(cudaMemcpyAsync(&s, ix->state, sizeof(s), cudaMemcpyDeviceToHost, st));
  RPX_CUDA_OK(cudaStreamSynchronize(st));
  if (h_norm_max) *h_norm_max = sqrtf(s.norm2_max);
  if (h_max_err) memcpy(h_max_err, &s.max_err_bits, 4);
  if (h_max_eps) memcpy(h_max_eps, &s.max_eps_bits, 4);
  if (h_n_exact) *h_n_exact = (int64_t)s.n_exact_total;
  return RPX_OK;
}

size_t rpx_index_topk_workspace_bytes(int64_t n, int32_t d, int32_t nq, int32_t k) {
  if (nq < 1 || k < 1 || k > 1024 || n < 0 || d <= 0) return 0;
  const size_t a = ws_layout(n, nq, k, d, kMaxSmsForSizing).total, b = ws_layout(n, nq, k, d, 132).total;
  return (a > b ? a : b) + 256;
}

int rpx_index_topk(rpx_index* ix, const void* d_Q, int32_t nq, int32_t k, const uint32_t* d_access_mask,
                   int64_t mask_stride_words, float* d_out_scores, double* d_out_scores64, int64_t* d_out_idx,
                   int32_t* d_out_count, int64_t* d_out_packed, int64_t idx_offset, int32_t flags, void* d_workspace,
                   size_t workspace_bytes, void* stream) {
  return topk_dispatch(ix, d_Q, nq, k, d_access_mask, mask_stride_words, d_out_scores, d_out_scores64, d_out_idx,
                       d_out_count, d_out_packed, idx_offset, flags, d_workspace, workspace_bytes, stream);
}

size_t rpx_sim_topk_workspace_bytes(int64_t n, int32_t d, int32_t nq, int32_t k) {
  const size_t inner = rpx_index_topk_workspace_bytes(n, d, nq, k);
  return inner ? inner + kStateBytes : 0;
}

int rpx_sim_topk(const void* d_Q, int32_t nq, const void* d_E, int64_t n, int32_t d, int32_t k,
                 const uint32_t* d_access_mask, int64_t mask_stride_words, float* d_out_scores,
                 double* d_out_scores64, int64_t* d_out_idx, int32_t* d_out_count, int64_t idx_offset,
                 void* d_workspace, size_t workspace_bytes, void* stream) {
  RPX_REQUIRE(d_Q && d_out_scores && d_out_idx && d_workspace, RPX_ERR_INVALID, "rpx_sim_topk: null argument");
  RPX_REQUIRE(d_E != nullptr || n == 0, RPX_ERR_INVALID, "rpx_sim_topk: null index");
  RPX_REQUIRE(workspace_bytes > kStateBytes, RPX_ERR_WORKSPACE, "rpx_sim_topk: workspace too small");
  RPX_REQUIRE((reinterpret_cast<uintptr_t>(d_workspace) & 255) == 0, RPX_ERR_INVALID, "workspace must be 256-byte aligned");
  RPX_REQUIRE(d > 0 && d % 64 == 0 && d <= 8192, RPX_ERR_UNSUPPORTED, "rpx_sim_topk: d=%d must be a multiple of 64 (<= 8192)", d);
  // one-shot form: the handle state lives at the front of the workspace and the row-norm pass runs per call
  rpx_index ix;
  ix.E = static_cast<const __nv_bfloat16*>(d_E);
  ix.n = n;
  ix.d = d;
  ix.state = static_cast<IndexState*>(d_workspace);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RPX_CUDA_OK(cudaMemsetAsync(d_workspace, 0, kStateBytes, st));
  RPX_TRY(launch_row_norm_max(ix.E, n, d, ix.state, st));
  return topk_dispatch(&ix, d_Q, nq, k, d_access_mask, mask_stride_words, d_out_scores, d_out_scores64, d_out_idx,
                       d_out_count, nullptr, idx_offset, 0, static_cast<uint8_t*>(d_workspace) + kStateBytes,
                       workspace_bytes - kStateBytes, stream);
}

int rpx_topk_merge(const double* d_scores64, const int64_t* d_idx, int32_t n_parts, int32_t nq, int32_t k,
                   float* d_out_scores, double* d_out_scores64, int64_t* d_out_idx, int32_t* d_out_count,
                   void* stream) {
  RPX_REQUIRE(d_scores64 && d_idx && d_out_scores && d_out_idx, RPX_ERR_INVALID, "rpx_topk_merge: null argument");
  return launch_topk_merge(d_scores64, d_idx, false, n_parts, nq, k, d_out_scores, d_out_scores64, d_out_idx, d_out_count,
                           static_cast<cudaStream_t>(stream));
}

int rpx_topk_merge_packed(const int64_t* d_packed, int32_t n_parts, int32_t nq, int32_t k, float* d_out_scores,
                          double* d_out_scores64, int64_t* d_out_idx, int32_t* d_out_count, void* stream) {
  RPX_REQUIRE(d_packed && d_out_scores && d_out_idx, RPX_ERR_INVALID, "rpx_topk_merge_packed: null argument");
  RPX_REQUIRE((reinterpret_cast<uintptr_t>(d_packed) & 15) == 0, RPX_ERR_INVALID, "rpx_topk_merge_packed: 16-byte alignment");
  return launch_topk_merge(nullptr, d_packed, true, n_parts, nq, k, d_out_scores, d_out_scores64, d_out_idx, d_out_count,
                           static_cast<cudaStream_t>(stream));
}

}  // extern "C"
