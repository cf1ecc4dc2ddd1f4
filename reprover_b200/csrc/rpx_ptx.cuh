// rpx_ptx.cuh — thin inline-PTX wrappers for the sm_90a features the engine uses:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA), fences.
//
// Everything here is sm_90a-only by design (no multi-arch dispatch).  Waits are
// bounded: a barrier that does not flip within ~2 s of SM clock traps instead of
// hanging the GPU.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace rpx {

#define RPX_DEVICE __device__ __forceinline__

RPX_DEVICE uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

RPX_DEVICE uint32_t lane_id() { return threadIdx.x & 31; }

// Returns 1 in exactly one (converged) lane of the warp.
RPX_DEVICE uint32_t elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .b32 rx;\n"
      ".reg .pred px;\n"
      "elect.sync rx|px, 0xFFFFFFFF;\n"
      "@px mov.s32 %0, 1;\n"
      "}\n"
      : "+r"(pred));
  return pred;
}

// ----------------------------------------------------------------------------- mbarrier
RPX_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
RPX_DEVICE void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
RPX_DEVICE void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
RPX_DEVICE void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
RPX_DEVICE void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
#ifndef RPX_WAIT_HINT_NS
#define RPX_WAIT_HINT_NS 2000
#endif
// One mbarrier.try_wait probe.  HINT_NS > 0 adds a suspend-time hint: a failed probe may park the
// thread for up to that long (ptxas emits NANOSLEEP.SYNCS), which frees issue slots for the other
// warps of the sub-partition — good for the long waits of the GEMM pipelines, bad for short
// latency-critical handshakes (attention), which use HINT_NS = 0.
template <uint32_t HINT_NS>
RPX_DEVICE uint32_t mbar_try_wait_t(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  if constexpr (HINT_NS > 0) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(HINT_NS)
        : "memory");
  } else {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  }
  return ok;
}
// Bounded wait: a barrier that has not flipped after ~2 s of SM clock is a pipeline bug, not a slow kernel,
// and traps.  There is deliberately no printf on that path: printf is a function call, and ptxas serialises
// every wgmma of a kernel in which one may run while wgmma groups are in flight.  The loop body is kept to
// the bare minimum: these spin loops share their SM sub-partition's issue slots with other warps.
template <uint32_t HINT_NS = RPX_WAIT_HINT_NS>
RPX_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait_t<HINT_NS>(bar, parity)) return;
  uint32_t spins = 0;
  long long t0 = 0;
  while (!mbar_try_wait_t<HINT_NS>(bar, parity)) {
    if ((++spins & 0x3FFu) == 0) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      if (now - t0 > 4000000000LL) __trap();
    }
  }
}

// ----------------------------------------------------------------------------- TMA
// 2-D tiled load: coordinates are (c0 = innermost/contiguous dim, c1 = row).
RPX_DEVICE void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int32_t c0,
                            int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)),
        "r"(c0), "r"(c1)
      : "memory");
}
// Same, with an L2 eviction-priority hint (createpolicy-encoded constants below).
RPX_DEVICE void tma_load_2d_hint(void* smem_dst, const void* tmap, uint64_t* bar, int32_t c0,
                                 int32_t c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)),
        "r"(c0), "r"(c1), "l"(policy)
      : "memory");
}
// Same, multicast: the box lands at the same shared-memory offset in every CTA of the cluster named in
// `cta_mask`, and each of them gets the complete_tx on its own barrier at `bar`'s offset.
RPX_DEVICE void tma_load_2d_multicast(void* smem_dst, const void* tmap, uint64_t* bar, int32_t c0, int32_t c1,
                                      uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "h"(cta_mask)
      : "memory");
}
// 2-D tiled store shared -> global, tracked by the issuing thread's bulk async-group.
RPX_DEVICE void tma_store_2d(const void* tmap, const void* smem_src, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(tmap)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
RPX_DEVICE void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// Until at most N of this thread's bulk groups still have shared-memory reads outstanding.
template <int N>
RPX_DEVICE void bulk_wait_group_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;

RPX_DEVICE void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}

// ----------------------------------------------------------------------------- thread-block clusters
RPX_DEVICE uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// All threads of all CTAs of the cluster; release/acquire at cluster scope.
RPX_DEVICE void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// Arrive on the barrier at `bar`'s offset in the shared memory of cluster CTA `cta`.  The arrive has the default
// CTA-scope release semantics: the pipelines use it to hand a stage back once their wgmma reads of it have
// completed (wgmma.wait_group), which needs no ordering of other memory operations.  `.release.cluster` would
// compile to a GPU-scope MEMBAR before every arrival, which waits for the thread's outstanding global stores.
RPX_DEVICE void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n"
      ".reg .b32 ra;\n"
      "mapa.shared::cluster.u32 ra, %0, %1;\n"
      "mbarrier.arrive.shared::cluster.b64 _, [ra];\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(cta)
      : "memory");
}

// ----------------------------------------------------------------------------- wgmma
// Warpgroup MMA: the four warps of an aligned warpgroup (warps 4i .. 4i+3) issue each wgmma together.
// The fp32 accumulator of an m64nN instruction is spread over the warpgroup's registers: warp w holds rows
// [16w, 16w + 16); lane l holds, for every 8-column block j, d[4j], d[4j+1] = row 16w + l/4, columns
// 8j + 2(l%4) + {0, 1}, and d[4j+2], d[4j+3] = the same columns of row 16w + l/4 + 8.
RPX_DEVICE void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
RPX_DEVICE void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// Until at most N of this warpgroup's committed wgmma groups are still in flight.
template <int N>
RPX_DEVICE void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Tells the compiler that the accumulator registers change here: keeps their reads after a wgmma_wait and
// their writes before a wgmma_fence in program order.
template <int R>
RPX_DEVICE void wgmma_fence_operand(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 64] (+)= A[64 x 16] (smem, K-major) * B[64 x 16]^T (smem, K-major); fp32 accumulator in registers.
// The m64nN forms below write d[0, N/2): the fragment of an m64nN instruction is the first N/2 registers of a
// wider one's, so a narrower MMA can run on a prefix of a wider accumulator.
template <int R>
RPX_DEVICE void wgmma_m64n64k16_ss(float (&d)[R], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  static_assert(R >= 32, "m64n64 writes 32 accumulator registers");
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

// D[64 x 128] (+)= A[64 x 16] (smem, K-major) * B[128 x 16]^T (smem, K-major); fp32 accumulator in registers.
template <int R>
RPX_DEVICE void wgmma_m64n128k16_ss(float (&d)[R], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  static_assert(R >= 64, "m64n128 writes 64 accumulator registers");
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

// D[64 x 192] (+)= A[64 x 16] (smem, K-major) * B[192 x 16]^T (smem, K-major); fp32 accumulator in registers.
template <int R>
RPX_DEVICE void wgmma_m64n192k16_ss(float (&d)[R], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  static_assert(R >= 96, "m64n192 writes 96 accumulator registers");
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %98, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n192k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, %96, %97, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

// D[64 x 256] (+)= A[64 x 16] (smem, K-major) * B[256 x 16]^T (smem, K-major); fp32 accumulator in registers.
RPX_DEVICE void wgmma_m64n256k16_ss(float (&d)[128], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate));
}

// D[64 x 64] (+)= A[64 x 16] (registers, bf16x2) * B[16 x 64] (smem, MN-major); fp32 accumulator in registers.
RPX_DEVICE void wgmma_m64n64k16_rs_bmn(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %37, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate));
}

// ----------------------------------------------------------------------------- descriptors
// Shared-memory matrix descriptor (sm_90 wgmma) for a bf16 tile stored as rows of 128 B (64 elements) with
// the 128-byte swizzle TMA writes (CU_TENSOR_MAP_SWIZZLE_128B):
//   start address >> 4            bits [0,14)
//   leading byte offset >> 4      bits [16,30)
//   stride byte offset >> 4       bits [32,46)   (8 rows * 128 B = 1024 B between row groups)
//   layout type = 1 (SWIZZLE_128B) bits [62,64)
// K-major (rows = M or N, 64 K-elements per row): the leading offset is unused.  Advancing along K inside
// the 128-B swizzle atom is done by adding (k_bytes >> 4) to the low word.  MN-major (rows = K, 64
// N-elements per row, one swizzle atom wide): groups of 8 K-rows sit 1024 B apart; both offset fields
// carry that stride, since with a single atom along N the other one is never used.
// The tile base must be 1024-byte aligned.
RPX_DEVICE uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(lbo_bytes >> 4) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
RPX_DEVICE uint64_t make_smem_desc_kmajor_sw128(uint32_t smem_addr) { return make_smem_desc_sw128(smem_addr, 16); }
RPX_DEVICE uint64_t make_smem_desc_mnmajor_sw128(uint32_t smem_addr) { return make_smem_desc_sw128(smem_addr, 1024); }

// ----------------------------------------------------------------------------- programmatic dependent launch
// Kernels of one encoder call are launched with programmatic stream serialization (rpx_common.cuh
// launch_pdl): a kernel may start while its predecessor in the stream is still running, so that its
// prologue (barrier init, descriptor prefetch) overlaps the predecessor's tail.
// pdl_wait() returns once the predecessor grid has completed and its writes are visible: every kernel
// calls it before the first access to global memory another kernel wrote.  pdl_launch_dependents() lets
// the successor be scheduled once every CTA of this grid has issued it.  Both are no-ops for a kernel
// launched without the attribute.
RPX_DEVICE void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
RPX_DEVICE void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ----------------------------------------------------------------------------- register budget
// Re-balances the register file between warpgroups of a warp-specialised kernel: every warp of the
// warpgroup executes it, and the new per-thread budget N is a multiple of 8 in [24, 256].
template <uint32_t N>
RPX_DEVICE void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <uint32_t N>
RPX_DEVICE void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// ----------------------------------------------------------------------------- misc
RPX_DEVICE uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

}  // namespace rpx
