// PTX wrappers shared by the tensor-core kernels of libtecogan_b200 (sm_90a): mbarriers, TMA
// (tensor + bulk), wgmma with shared-memory descriptors.
#pragma once
#include <cuda.h>
#include "tg_common.cuh"

namespace {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.b32 %0, 1, 0, p;\n}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok;
}
// Bounded wait: a protocol bug must fault with a message instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int tag) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 3000000000LL) {
      if ((threadIdx.x & 31) == 0 && blockIdx.x < 2)
        printf("tecogan: mbarrier timeout tag=%d block=%d thread=%d parity=%u\n", tag, blockIdx.x,
               threadIdx.x, parity);
      __trap();
    }
  }
}
// Same bound without the message, for the threads that issue wgmma: a call (printf) inside their loop
// would make ptxas serialise the wgmma pipeline.
__device__ __forceinline__ void mbar_wait_mma(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > 3000000000LL) __trap();
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const void* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const void* map, uint32_t bar, int c0,
                                            int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes,
                                          uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar)
      : "memory");
}
// smem -> global tensor store; out-of-bounds box elements are not written.  Completion is tracked by
// the issuing thread's bulk async-groups.
__device__ __forceinline__ void tma_store_4d(const void* map, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
      ::"l"(reinterpret_cast<uint64_t>(map)), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_5d(const void* map, uint32_t src, int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
      ::"l"(reinterpret_cast<uint64_t>(map)), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the issuing thread's bulk stores have finished READING shared memory (the source may be reused)
__device__ __forceinline__ void bulk_wait_group_read0() {
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
// all but the most recent of the issuing thread's bulk store groups have finished reading shared memory
__device__ __forceinline__ void bulk_wait_group_read1() {
  asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
}
// the issuing thread's bulk stores are complete (their writes are done)
__device__ __forceinline__ void bulk_wait_group0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// generic-proxy smem writes -> visible to a following TMA / wgmma (async proxy) read
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// four 8x8 b16 matrices; lane l addresses row l%8 of matrix l/8.  .trans: the thread's fragment
// (row l/4, cols 2*(l%4)+{0,1}) is element (memory row 2*(l%4)+{0,1}, column l/4).
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}
__device__ __forceinline__ void stmatrix_x4_trans(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]),
               "r"(r[1]), "r"(r[2]), "r"(r[3])
               : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ float4 ld_shared_v4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr)
               : "memory");
  return v;
}

// ---- thread-block clusters (distributed shared memory)
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_id_x() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_count_x() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%nclusterid.x;" : "=r"(r));
  return r;
}
// the shared::cluster address of the same shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa_shared(uint32_t saddr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(saddr), "r"(rank));
  return r;
}
// 16 bytes into a peer CTA's shared memory; completes 16 bytes of transaction count on the peer's mbarrier
__device__ __forceinline__ void st_async_v4(uint32_t cluster_addr, float4 v, uint32_t cluster_bar) {
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v4.f32 [%0], {%1, %2, %3, %4}, [%5];"
               ::"r"(cluster_addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "r"(cluster_bar)
               : "memory");
}
// arrive on an mbarrier of any CTA of the cluster (release: this thread's prior accesses happen before)
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_bar) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_bar) : "memory");
}
// bounded wait with cluster-scope acquire: arrivals / st.async data from peer CTAs are visible after it
__device__ __forceinline__ void mbar_wait_cluster(uint32_t bar, uint32_t parity) {
  auto try_wait = [&]() {
    uint32_t ok;
    asm volatile(
        "{\n.reg .pred p;\nmbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n"
        "selp.b32 %0, 1, 0, p;\n}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok;
  };
  if (try_wait()) return;
  long long t0 = clock64();
  while (!try_wait())
    if (clock64() - t0 > 3000000000LL) __trap();
}
// every thread of every CTA of the cluster (not .aligned: callers may sit behind divergent role branches)
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;\nbarrier.cluster.wait.acquire;" ::: "memory");
}

// wgmma shared-memory descriptor, K-major operand, 128B swizzle (cute::GMMA::GmmaDescriptor):
// [0,14) start>>4 | [16,30) LBO>>4 (unused for swizzled K-major, 1) | [32,46) SBO>>4 = byte stride
// between 8-row groups | [62,64) layout = 1 (SWIZZLE_128B).  This returns the constant high part;
// the start address is OR-ed into the low 14 bits per MMA.  The swizzle is a function of the
// absolute shared-memory address (1024-byte aligned atoms), so a start address advanced by whole
// 128-byte rows or 32-byte K steps addresses the shifted view of a TMA-written tile.
__host__ __device__ __forceinline__ uint64_t gmma_desc_hi(uint32_t sbo_bytes) {
  return (static_cast<uint64_t>(1) << 16) | (static_cast<uint64_t>(sbo_bytes >> 4) << 32) |
         (static_cast<uint64_t>(1) << 62);
}
__device__ __forceinline__ uint32_t gmma_addr16(uint32_t saddr) { return (saddr & 0x3FFFFu) >> 4; }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, fp16 in, fp32 accumulate, both operands K-major in smem.
// Accumulator fragment of thread t of the warpgroup, register i (N/2 of them):
//   row = 16*(t/32) + (t%32)/4 + 8*((i/2)%2),  col = 8*(i/4) + 2*(t%4) + i%2.
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_n48(float (&d)[24], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %26, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23}, "
      "%24, %25, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
      : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <int NF>
__device__ __forceinline__ void wgmma_k16(float (&d)[NF], uint64_t da, uint64_t db, uint32_t scale_d) {
  static_assert(NF == 32 || NF == 24, "N = 64 or 48");
  if constexpr (NF == 32) wgmma_n64(d, da, db, scale_d);
  else wgmma_n48(d, da, db, scale_d);
}

// transposed-conv taps of parity accumulator `a` (1/2/2/4 groups) of one 16x8 tile, pixels on N:
//   acc[64 cout][128 px] (+)= W[group] (A: the packed [cout][64] tile, K-major, SBO 1024, 8 KB per group)
//                             x the group's shifted view of the 17x9 halo box (B: K-major, 16 core groups of
//                             8 pixels, SBO = one box row of 9 x 128 B, origin 0, start += (dy*9+dx)*128 B)
// one m64n128k16 per (group, k-step).  The first MMA of the parity overwrites acc (scale-d = 0).
template <int A>
__device__ __forceinline__ void convT_pxn_parity(float (&acc)[64], uint32_t x16, uint32_t w16) {
  constexpr uint32_t kBoxW = 9;
  const uint64_t w_hi = gmma_desc_hi(1024u), x_hi = gmma_desc_hi(kBoxW * 128u);
#pragma unroll
  for (int g = 0; g < 9; ++g) {
    const TgGroup gr = tg_group(TG_CONVT_3X3_S2, g);
    if (gr.acc != A) continue;
    const bool first = g == 0 || tg_group(TG_CONVT_3X3_S2, g > 0 ? g - 1 : 0).acc != gr.acc;
    const uint32_t a16 = w16 + (uint32_t)g * (64u * 128u / 16u);
    const uint32_t b16 = x16 + (uint32_t)(gr.dy * (int)kBoxW + gr.dx) * 8u;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      wgmma_n128(acc, w_hi | (uint64_t)(a16 + 2u * k), x_hi | (uint64_t)(b16 + 2u * k), (first && k == 0) ? 0u : 1u);
  }
}
__device__ __forceinline__ void convT_pxn_mmas(float (&acc)[64], uint32_t x16, uint32_t w16, int a) {
  switch (a) {
    case 0: convT_pxn_parity<0>(acc, x16, w16); break;
    case 1: convT_pxn_parity<1>(acc, x16, w16); break;
    case 2: convT_pxn_parity<2>(acc, x16, w16); break;
    default: convT_pxn_parity<3>(acc, x16, w16); break;
  }
}

}  // namespace
