// rpx_bm25.cu — exact BM25Okapi scoring and top-k over an inverted index (the reference's BM25 baseline,
// retrieval/bm25/main.py:48-52: `bm25.get_batch_scores(query, accessible)` then `np.argsort(scores)[::-1][:k]`).
//
// The index is CSR over terms: the postings of term t are [term_ptr[t], term_ptr[t+1]), each a document and the
// term's fp64 contribution c(t, d) to that document's score, computed on the host exactly as rank_bm25 computes it.
// A document's score is the plain fp64 sum ((0 + c(q1, d)) + c(q2, d)) + ... over the query tokens present in d, in
// query order (a token absent from d adds +-0.0, which changes no sum).  The kernel keeps that order: each CTA owns
// a tile of documents whose scores live in shared memory, walks the query's tokens in order and adds each token's
// postings that fall in the tile, one token at a time.  Postings of one token name distinct documents, so the adds of
// one step never collide, and a barrier separates consecutive tokens.  No atomics, no reassociation: the scores equal
// get_batch_scores bit for bit, whatever the tiling and the batch.
//
//   bm25_tile_kernel  grid (tiles, queries).  Scores one (query, tile); then either writes the tile's scores
//                     (dense row) or selects the tile's k best accessible documents under (score desc, index asc) —
//                     MSB-first radix select on the monotone fp64 keys, ties cut by index — and writes them sorted.
//   merge             the tiles' sorted lists go through the k-way merge of the multi-GPU path
//                     (launch_topk_merge, rpx_simtopk.cu), in rounds when tiles * k exceeds what one merge CTA holds.
#include <new>

#include "rpx_common.cuh"
#include "rpx_kernels.cuh"
#include "rpx_topk_common.cuh"

struct rpx_bm25 {
  const int64_t* term_ptr;
  const int32_t* post_doc;
  const double* post_c;
  int32_t vocab;
  int64_t n_docs;
};

namespace rpx {
namespace {

constexpr int kTile = 4096;                    // documents per CTA (32 KB of fp64 scores)
constexpr int kThreads = 256;
constexpr int kPerThread = kTile / kThreads;   // selection: thread t owns documents [16 t, 16 t + 16) of the tile
constexpr int kMaxK = 1024;
constexpr int kMergeEntries = 96 * 1024 / 16;  // (score, index) entries one launch_topk_merge CTA holds
constexpr int kMaxQueries = 65535;             // grid.y
static_assert(kPerThread == 16, "selection masks assume 16 documents per thread");

struct Bm25Params {
  const int64_t* term_ptr;
  const int32_t* post_doc;
  const double* post_c;
  int32_t vocab;
  int64_t n_docs;
  const int32_t* tokens;
  const int64_t* offsets;   // [nq + 1] device; nullptr: one query, tokens [0, n_tokens)
  int64_t n_tokens;
  const uint32_t* mask;     // optional [n_rows][mask_stride]
  int64_t mask_stride;
  const int32_t* mask_rows; // [nq] device: the mask row of each query
  int k, nq;
  double* dense_out;        // dense mode: [n_docs] scores of the one query
  double* part_s;           // top-k mode: [tiles, nq, k] sorted lists
  int64_t* part_i;
};

__device__ __forceinline__ int64_t lower_bound_doc(const int32_t* __restrict__ a, int64_t lo, int64_t hi, int32_t v) {
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (__ldg(a + mid) < v) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// Exclusive block-wide prefix sum of one int per thread (kThreads threads); `scratch` holds >= 9 ints.
__device__ __forceinline__ int block_exclusive_scan(int v, int* scratch, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int y = __shfl_up_sync(kFullMask, x, off);
    if (lane >= off) x += y;
  }
  __syncthreads();
  if (lane == 31) scratch[warp] = x;
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int w = 0; w < kThreads / 32; ++w) {
      const int t = scratch[w];
      scratch[w] = run;
      run += t;
    }
    scratch[kThreads / 32] = run;
  }
  __syncthreads();
  *total = scratch[kThreads / 32];
  return scratch[warp] + x - v;
}

__global__ void __launch_bounds__(kThreads) bm25_tile_kernel(const Bm25Params p) {
  __shared__ double s[kTile];
  // scoring: the token ranges of one chunk of the query; selection: the selected keys and tile-local indexes
  __shared__ __align__(16) uint8_t aux[kMaxK * (sizeof(uint64_t) + sizeof(uint32_t))];
  __shared__ int hist[256];
  __shared__ uint64_t bcast[2];
  __shared__ int n_sel;

  const int tid = threadIdx.x;
  const int q = blockIdx.y;
  const int64_t lo = (int64_t)blockIdx.x * kTile;
  const int64_t hi = lo + kTile < p.n_docs ? lo + kTile : p.n_docs;
  for (int j = tid; j < kTile; j += kThreads) s[j] = 0.0;

  // ---- scoring: the query's tokens in order, kThreads at a time (their posting ranges are found in parallel)
  int64_t* rng_a = reinterpret_cast<int64_t*>(aux);
  int64_t* rng_b = rng_a + kThreads;
  const int64_t t0 = p.offsets ? p.offsets[q] : 0;
  const int64_t t1 = p.offsets ? p.offsets[q + 1] : p.n_tokens;
  for (int64_t c0 = t0; c0 < t1; c0 += kThreads) {
    const int nc = t1 - c0 < kThreads ? (int)(t1 - c0) : kThreads;
    __syncthreads();  // the previous chunk's ranges are consumed
    if (tid < nc) {
      const int32_t t = __ldg(p.tokens + c0 + tid);
      int64_t a = 0, b = 0;
      if (t >= 0 && t < p.vocab) {  // an id outside the vocabulary adds nothing, like an unknown token
        const int64_t pa = __ldg(p.term_ptr + t), pb = __ldg(p.term_ptr + t + 1);
        a = lower_bound_doc(p.post_doc, pa, pb, (int32_t)lo);
        b = lower_bound_doc(p.post_doc, a, pb, (int32_t)hi);
      }
      rng_a[tid] = a;
      rng_b[tid] = b;
    }
    __syncthreads();
    for (int i = 0; i < nc; ++i) {
      const int64_t a = rng_a[i], b = rng_b[i];
      if (a == b) continue;  // same decision in every thread: the token has no posting in this tile
#pragma unroll 4
      for (int64_t j = a + tid; j < b; j += kThreads) s[__ldg(p.post_doc + j) - lo] += __ldg(p.post_c + j);
      __syncthreads();  // the next token may add to the same documents
    }
  }
  __syncthreads();

  if (p.dense_out) {
    for (int64_t j = tid; j < hi - lo; j += kThreads) p.dense_out[lo + j] = s[j];
    return;
  }

  // ---- selection: the tile's k best accessible documents under (score desc, index asc)
  const uint32_t* mrow = p.mask ? p.mask + (size_t)__ldg(p.mask_rows + q) * p.mask_stride : nullptr;
  const int base = tid * kPerThread;
  uint32_t valid = 0;  // bit e: document lo + base + e exists and is accessible
  if (lo + base < hi) {
    valid = hi - (lo + base) >= kPerThread ? 0xFFFFu : (1u << (hi - (lo + base))) - 1u;
    if (mrow) valid &= (__ldg(mrow + ((lo + base) >> 5)) >> ((lo + base) & 31)) & 0xFFFFu;  // base % 16 == 0
  }
  uint64_t key[kPerThread];
#pragma unroll
  for (int e = 0; e < kPerThread; ++e) key[e] = dkey(s[base + e]);
  int* redi = hist;
  const int n_valid = block_reduce<int>(__popc(valid), redi, [](int a, int b) { return a + b; }, 0);
  const int k = p.k;
  uint32_t take = valid;
  if (n_valid > k) {
    // k-th largest key T among the valid entries, 8 bits at a time; `need` = how many entries equal to T belong
    uint64_t prefix = 0ull, pmask = 0ull;
    int need = k;
    for (int pass = 0; pass < 8; ++pass) {
      const int shift = 56 - 8 * pass;
      hist[tid] = 0;  // kThreads == 256 bins
      __syncthreads();
#pragma unroll
      for (int e = 0; e < kPerThread; ++e)
        if (((valid >> e) & 1u) && (key[e] & pmask) == prefix) atomicAdd(&hist[(int)((key[e] >> shift) & 255ull)], 1);
      __syncthreads();
      if (tid < 32) {
        // lane l holds bins 255 - 8 l ... 248 - 8 l (descending); find the bin where the running count reaches `need`
        int c[8], sum = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          c[i] = hist[255 - 8 * tid - i];
          sum += c[i];
        }
        int incl = sum;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
          const int y = __shfl_up_sync(kFullMask, incl, off);
          if (tid >= off) incl += y;
        }
        int run = incl - sum;
        if (run < need && incl >= need) {
          int i = 0;
          while (run + c[i] < need) run += c[i++];
          bcast[0] = (uint64_t)(255 - 8 * tid - i);
          bcast[1] = (uint64_t)run;
        }
      }
      __syncthreads();
      prefix |= bcast[0] << shift;
      pmask |= 255ull << shift;
      need -= (int)bcast[1];
      __syncthreads();
    }
    // take every key above T and the first `need` keys equal to T in index order
    uint32_t eq = 0;
    take = 0;
#pragma unroll
    for (int e = 0; e < kPerThread; ++e) {
      if (!((valid >> e) & 1u)) continue;
      if (key[e] > prefix) take |= 1u << e;
      else if (key[e] == prefix) eq |= 1u << e;
    }
    int n_eq_total;
    int before = block_exclusive_scan(__popc(eq), hist, &n_eq_total);
#pragma unroll
    for (int e = 0; e < kPerThread; ++e)
      if (((eq >> e) & 1u) && before < need) {
        take |= 1u << e;
        ++before;
      }
  }
  uint64_t* sel_key = reinterpret_cast<uint64_t*>(aux);
  uint32_t* sel_idx = reinterpret_cast<uint32_t*>(sel_key + kMaxK);
  int n_taken;
  int pos = block_exclusive_scan(__popc(take), hist, &n_taken);  // also orders the ranges' last use before reuse
#pragma unroll
  for (int e = 0; e < kPerThread; ++e)
    if ((take >> e) & 1u) {
      sel_key[pos] = key[e];
      sel_idx[pos] = (uint32_t)(base + e);
      ++pos;
    }
  if (tid == 0) n_sel = n_taken;
  __syncthreads();
  // selected entries arrive in index order, so the rank of an entry is the number of larger keys plus the number of
  // equal keys before it
  const int ns = n_sel;
  const size_t row = ((size_t)blockIdx.x * p.nq + q) * k;
  for (int c = tid; c < ns; c += kThreads) {
    const uint64_t kc = sel_key[c];
    int rank = 0;
    for (int j = 0; j < ns; ++j) {
      const uint64_t kj = sel_key[j];
      rank += (kj > kc || (kj == kc && j < c)) ? 1 : 0;
    }
    p.part_s[row + rank] = undkey(kc);
    p.part_i[row + rank] = lo + sel_idx[c];
  }
  for (int r = ns + tid; r < k; r += kThreads) {
    p.part_s[row + r] = -INFINITY;
    p.part_i[row + r] = -1;
  }
}

struct Bm25Ws {
  size_t offsets, rows, a_s, a_i, b_s, b_i, f32, total;
};

int64_t n_tiles(int64_t n_docs) { return ceil_div64(n_docs, kTile); }

Bm25Ws bm25_ws_layout(int64_t n_docs, int nq, int k) {
  Bm25Ws L{};
  size_t off = 0;
  auto take = [&](size_t bytes) {
    const size_t o = off;
    off = align_up(off + bytes, 256);
    return o;
  };
  const size_t tiles = (size_t)n_tiles(n_docs);
  const size_t group = (size_t)(kMergeEntries / k);
  const size_t round2 = (tiles + group - 1) / group;  // parts after the first merge round (when there is one)
  const size_t list = (size_t)nq * k;
  L.offsets = take((size_t)(nq + 1) * sizeof(int64_t));
  L.rows = take((size_t)nq * sizeof(int32_t));
  L.a_s = take(tiles * list * sizeof(double));
  L.a_i = take(tiles * list * sizeof(int64_t));
  L.b_s = take(round2 * list * sizeof(double));
  L.b_i = take(round2 * list * sizeof(int64_t));
  L.f32 = take(round2 * list * sizeof(float));
  L.total = off;
  return L;
}

int launch_tiles(const rpx_bm25* ix, const Bm25Params& p, int nq, cudaStream_t st) {
  DeviceInfo dev;
  RPX_TRY(get_device_info(&dev));
  bm25_tile_kernel<<<dim3((unsigned)n_tiles(ix->n_docs), (unsigned)nq), kThreads, 0, st>>>(p);
  RPX_CUDA_OK(cudaGetLastError());
  return RPX_OK;
}

Bm25Params base_params(const rpx_bm25* ix, const int32_t* d_tokens) {
  Bm25Params p{};
  p.term_ptr = ix->term_ptr;
  p.post_doc = ix->post_doc;
  p.post_c = ix->post_c;
  p.vocab = ix->vocab;
  p.n_docs = ix->n_docs;
  p.tokens = d_tokens;
  return p;
}

}  // namespace
}  // namespace rpx

using namespace rpx;

extern "C" {

int rpx_bm25_create(const int64_t* d_term_ptr, const int32_t* d_post_doc, const double* d_post_c, int32_t vocab,
                    int64_t n_docs, int64_t nnz, rpx_bm25** out) {
  RPX_REQUIRE(out, RPX_ERR_INVALID, "rpx_bm25_create: null argument");
  *out = nullptr;
  RPX_REQUIRE(d_term_ptr && (nnz == 0 || (d_post_doc && d_post_c)), RPX_ERR_INVALID, "rpx_bm25_create: null index array");
  RPX_REQUIRE(vocab >= 1 && nnz >= 0, RPX_ERR_INVALID, "rpx_bm25_create: vocab=%d nnz=%lld", vocab, (long long)nnz);
  RPX_REQUIRE(n_docs >= 1 && n_docs <= (int64_t)INT32_MAX - kTile, RPX_ERR_UNSUPPORTED,
              "rpx_bm25_create: n_docs=%lld outside [1, %d]", (long long)n_docs, INT32_MAX - kTile);
  rpx_bm25* ix = new (std::nothrow) rpx_bm25();
  RPX_REQUIRE(ix != nullptr, RPX_ERR_INVALID, "out of host memory");
  ix->term_ptr = d_term_ptr;
  ix->post_doc = d_post_doc;
  ix->post_c = d_post_c;
  ix->vocab = vocab;
  ix->n_docs = n_docs;
  *out = ix;
  return RPX_OK;
}

int rpx_bm25_destroy(rpx_bm25* ix) {
  delete ix;
  return RPX_OK;
}

size_t rpx_bm25_topk_workspace_bytes(int64_t n_docs, int32_t nq, int32_t k) {
  if (n_docs < 1 || nq < 1 || nq > kMaxQueries || k < 1 || k > kMaxK) return 0;
  return bm25_ws_layout(n_docs, nq, k).total + 256;
}

int rpx_bm25_topk(const rpx_bm25* ix, const int32_t* d_tokens, const int64_t* h_offsets, int32_t nq,
                  const uint32_t* d_access_mask, int64_t mask_stride_words, const int32_t* h_mask_rows,
                  int32_t n_mask_rows, int32_t k, double* d_out_scores64, int64_t* d_out_idx, int32_t* d_out_count,
                  void* d_workspace, size_t workspace_bytes, void* stream) {
  RPX_REQUIRE(ix && h_offsets && d_out_scores64 && d_out_idx && d_workspace, RPX_ERR_INVALID,
              "rpx_bm25_topk: null argument");
  RPX_REQUIRE(nq >= 1 && nq <= kMaxQueries, RPX_ERR_UNSUPPORTED, "rpx_bm25_topk: nq=%d outside [1, %d]", nq, kMaxQueries);
  RPX_REQUIRE(k >= 1 && k <= kMaxK, RPX_ERR_UNSUPPORTED, "rpx_bm25_topk: k=%d outside [1, %d]", k, kMaxK);
  RPX_REQUIRE(h_offsets[0] >= 0, RPX_ERR_INVALID, "rpx_bm25_topk: negative offset");
  for (int32_t q = 0; q < nq; ++q)
    RPX_REQUIRE(h_offsets[q + 1] >= h_offsets[q], RPX_ERR_INVALID, "rpx_bm25_topk: offsets decrease at query %d", q);
  RPX_REQUIRE(d_tokens || h_offsets[nq] == h_offsets[0], RPX_ERR_INVALID, "rpx_bm25_topk: null token array");
  if (d_access_mask) {
    RPX_REQUIRE(h_mask_rows && n_mask_rows >= 1, RPX_ERR_INVALID, "rpx_bm25_topk: a mask needs its per-query rows");
    RPX_REQUIRE(mask_stride_words * 32 >= ix->n_docs, RPX_ERR_INVALID, "rpx_bm25_topk: mask stride too small");
    for (int32_t q = 0; q < nq; ++q)
      RPX_REQUIRE(h_mask_rows[q] >= 0 && h_mask_rows[q] < n_mask_rows, RPX_ERR_INVALID,
                  "rpx_bm25_topk: query %d names mask row %d of %d", q, h_mask_rows[q], n_mask_rows);
  }
  RPX_REQUIRE((reinterpret_cast<uintptr_t>(d_workspace) & 255) == 0, RPX_ERR_INVALID, "workspace must be 256-byte aligned");
  const Bm25Ws L = bm25_ws_layout(ix->n_docs, nq, k);
  RPX_REQUIRE(L.total <= workspace_bytes, RPX_ERR_WORKSPACE, "rpx_bm25_topk: workspace %zu < %zu", workspace_bytes, L.total);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* ws = static_cast<uint8_t*>(d_workspace);
  // pageable host -> device copies: the host arrays are staged before these calls return
  RPX_CUDA_OK(cudaMemcpyAsync(ws + L.offsets, h_offsets, (size_t)(nq + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  if (d_access_mask)
    RPX_CUDA_OK(cudaMemcpyAsync(ws + L.rows, h_mask_rows, (size_t)nq * sizeof(int32_t), cudaMemcpyHostToDevice, st));

  Bm25Params p = base_params(ix, d_tokens);
  p.offsets = reinterpret_cast<const int64_t*>(ws + L.offsets);
  p.mask = d_access_mask;
  p.mask_stride = mask_stride_words;
  p.mask_rows = reinterpret_cast<const int32_t*>(ws + L.rows);
  p.k = k;
  p.nq = nq;
  p.part_s = reinterpret_cast<double*>(ws + L.a_s);
  p.part_i = reinterpret_cast<int64_t*>(ws + L.a_i);
  RPX_TRY(launch_tiles(ix, p, nq, st));

  // merge the tiles' lists; groups of `group` lists per merge CTA, in rounds until one group is left
  double* cur_s = p.part_s;
  int64_t* cur_i = p.part_i;
  double* nxt_s = reinterpret_cast<double*>(ws + L.b_s);
  int64_t* nxt_i = reinterpret_cast<int64_t*>(ws + L.b_i);
  float* f32 = reinterpret_cast<float*>(ws + L.f32);
  const int group = kMergeEntries / k;
  const size_t list = (size_t)nq * k;
  int parts = (int)n_tiles(ix->n_docs);
  while (parts > group) {
    const int groups = ceil_div(parts, group);
    for (int g = 0; g < groups; ++g) {
      const int n = parts - g * group < group ? parts - g * group : group;
      RPX_TRY(launch_topk_merge(cur_s + (size_t)g * group * list, cur_i + (size_t)g * group * list, false, n, nq, k,
                                f32 + (size_t)g * list, nxt_s + (size_t)g * list, nxt_i + (size_t)g * list, nullptr, st));
    }
    double* ts = cur_s;
    int64_t* ti = cur_i;
    cur_s = nxt_s;
    cur_i = nxt_i;
    nxt_s = ts;
    nxt_i = ti;
    parts = groups;
  }
  return launch_topk_merge(cur_s, cur_i, false, parts, nq, k, f32, d_out_scores64, d_out_idx, d_out_count, st);
}

int rpx_bm25_scores(const rpx_bm25* ix, const int32_t* d_tokens, int64_t n_tokens, double* d_out, void* stream) {
  RPX_REQUIRE(ix && d_out && (d_tokens || n_tokens == 0) && n_tokens >= 0, RPX_ERR_INVALID, "rpx_bm25_scores: bad argument");
  Bm25Params p = base_params(ix, d_tokens);
  p.n_tokens = n_tokens;
  p.dense_out = d_out;
  return launch_tiles(ix, p, 1, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
