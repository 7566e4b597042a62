// Pieces shared by the tensor-core kernels of libtecogan_b200 (sm_90a): PTX wrappers (mbarriers, TMA tensor +
// bulk, wgmma with shared-memory descriptors), the pixels-on-N mainloops and register epilogues, and the host-side
// tensor-map encoder.
#pragma once
#include <cuda.h>

#include <mutex>

#include "tg_common.cuh"
#include "tg_epilogue.cuh"

namespace {

constexpr int TH = 16, TW = 8;            // output tile of every tensor-core kernel: 16x8 pixels
constexpr uint32_t kSmemLimit = 232448;   // 227 KB opt-in limit per CTA

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
// The n64 fragment is therefore registers 0-31 of the n128 one; wgmma_n64 writes d[0..31] of a longer array.
template <int L>
__device__ __forceinline__ void wgmma_n64(float (&d)[L], uint64_t da, uint64_t db, uint32_t scale_d) {
  static_assert(L >= 32, "m64n64 needs 32 accumulator registers");
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
__device__ __forceinline__ void wgmma_n40(float (&d)[20], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %22, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n40k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19}, "
      "%20, %21, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19])
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

// 3x3 conv taps of 64-channel chunk c (of `chunks`) of one 16x8 tile, pixels on N:
//   acc[64 cout][128 px] (+)= W[tap][c] (A: the packed [cout][64] tile, K-major, SBO 1024; the resident tiles at w16
//                             are ordered [tap][chunk], tile16 = one tile's size / 16)
//                             x the tap's shifted view of the 18x10 halo box (B: K-major, 16 core groups of 8
//                             pixels, SBO = one box row of 10 x 128 B, origin -1, start += ((dy+1)*10+dx+1)*128 B)
// one m64n128k16 per (tap, k-step < ksteps), taps outer and k-steps inner: that order is the accumulation order,
// hence the output bits.  The first MMA of chunk 0 overwrites acc (scale-d = 0).
// N = 64 (a bottom tile row with at most 8 rows inside the image: rows 8-15 are clipped by the TMA store): each MMA is
// an m64n64k16 over the first 8 core groups (tile rows 0-7), with the same descriptors.  Registers 0-31 of the n128
// fragment are the n64 fragment, so rows 0-7 get the same products in the same order; acc[32..63] are not written and
// keep what the caller left there.  A caller that picks N at run time must wait for the MMAs (wgmma_wait) inside each
// branch: if the two paths join inside the wgmma pipeline stage, the register moves at the join make ptxas serialise
// every wgmma of the kernel (C7515).
// KS > 0 fixes the k-steps at compile time (ksteps_rt is then ignored).  With a run-time count each wgmma sits behind its
// own `k < ksteps` branch, and ptxas fences every one of them (WARPGROUP.ARRIVE, info C7519).
template <int N = 128, int KS = 0>
__device__ __forceinline__ void halo_pxn_mmas(float (&acc)[64], uint32_t x16, uint32_t w16, uint32_t tile16, int chunks,
                                              int c, int ksteps_rt) {
  static_assert(N == 128 || N == 64, "all 16 tile rows, or rows 0-7");
  const int ksteps = KS > 0 ? KS : ksteps_rt;
  constexpr uint32_t kBoxW = TW + 2;
  const uint64_t w_hi = gmma_desc_hi(1024u), x_hi = gmma_desc_hi(kBoxW * 128u);
#pragma unroll
  for (int g = 0; g < 9; ++g) {
    const TgGroup gr = tg_group(TG_CONV_3X3, g);
    const uint32_t a16 = w16 + (uint32_t)(g * chunks + c) * tile16;
    const uint32_t b16 = x16 + (uint32_t)((gr.dy + 1) * (int)kBoxW + (gr.dx + 1)) * 8u;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (k < ksteps) {
        const uint64_t da = w_hi | (uint64_t)(a16 + 2u * k), db = x_hi | (uint64_t)(b16 + 2u * k);
        const uint32_t sc = (g == 0 && c == 0 && k == 0) ? 0u : 1u;
        if constexpr (N == 128) wgmma_n128(acc, da, db, sc);
        else wgmma_n64(acc, da, db, sc);
      }
  }
}

// ---- register epilogue of the pixels-on-N accumulators: acc[64 cout][128 px] -> fp16 -> stmatrix into an output
// tile [pixel][channel], `pitch` bytes per pixel (128 B rows with the 128B swizzle = the TMA box image of a 64-channel
// tile, or a dense unswizzled slice of fewer channels).  Thread t of the warpgroup holds couts 16*(t/32) + (t%32)/4
// + {0, 8} and pixel columns 8*j + 2*(t%4) + {0, 1}, j = 0..15 (tile row j); one stmatrix.x4.trans writes two tile
// rows x 16 couts of its warp.
// Lane l addresses pixel row l%8 of 8x8 matrix m = l/8 = (tile row 2*jp + m/2, 8-channel chunk 2*q + m%2), q = the
// warp's pair of chunks within the tile; the swizzled offset of (pixel px, chunk) is px*128 + ((chunk ^ px%8) << 4).
// pool: matrix m = (pooled row pair 2*ip + m/2, chunk 2*q + m%2), its column 2*c + e = pooled pixel (row
// 2*(2*ip + m/2) + e, column c), i.e. lane l addresses pooled-tile pixel 8*(m/2) + kk, kk = 4*(l%2) + (l%8)/2.
__device__ __forceinline__ uint32_t pxn_mat_off(int lane, int q, uint32_t pitch, bool swizzled, bool pool) {
  const uint32_t kk = pool ? 4u * (lane & 1) + ((lane & 7) >> 1) : (uint32_t)(lane & 7);
  const uint32_t chunk = (uint32_t)(2 * q + ((lane >> 3) & 1));
  return (uint32_t)(8 * ((lane >> 3) >> 1) + kk) * pitch + ((swizzled ? chunk ^ kk : chunk) << 4);
}
// act(acc + bias) [+ the residual already in the tile, overwritten in place] -> the 16x8 px tile at `tile`; b0 / b1 =
// the bias of the thread's couts (t%32)/4 and + 8.
__device__ __forceinline__ void pxn_store_tile(const float (&acc)[64], uint32_t tile, uint32_t pitch, uint32_t mat_off,
                                               float b0, float b1, int act, bool residual) {
#pragma unroll
  for (int jp = 0; jp < 8; ++jp) {
    const uint32_t addr = tile + (uint32_t)jp * 16u * pitch + mat_off;
    uint32_t rv[4], ov[4];
    if (residual) ldmatrix_x4_trans(addr, rv);
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int i = 4 * (2 * jp + (m >> 1)) + 2 * (m & 1);
      const float bb = (m & 1) ? b1 : b0;
      float a0 = tg_epi_val(acc[i], bb, act), a1 = tg_epi_val(acc[i + 1], bb, act);
      if (residual) {
        const float2 rf = __half22float2(*reinterpret_cast<const __half2*>(&rv[m]));
        a0 += rf.x; a1 += rf.y;
      }
      const __half2 o = __floats2half2_rn(a0, a1);
      ov[m] = *reinterpret_cast<const uint32_t*>(&o);
    }
    stmatrix_x4_trans(addr, ov);
  }
}
// MaxPool2d(2, 2) folded in: the 2x2 block (tile rows 2*pr, 2*pr + 1; columns 2*(t%4), + 1) of a cout lies in four
// registers of one thread, so the pooled 8x4 px tile is formed without shuffles, from the same fp16 values the
// unpooled epilogue stores.  mat_off from pxn_mat_off(pool = true).
__device__ __forceinline__ void pxn_store_tile_pool2(const float (&acc)[64], uint32_t tile, uint32_t pitch,
                                                     uint32_t mat_off, float b0, float b1, int act) {
#pragma unroll
  for (int ip = 0; ip < 2; ++ip) {
    uint32_t ov[4];
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const float bb = (m & 1) ? b1 : b0;
      __half v[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int pr = 2 * (2 * ip + (m >> 1)) + e;
        const int i0 = 4 * (2 * pr) + 2 * (m & 1), i1 = i0 + 4;
        const __half2 r0 = __floats2half2_rn(tg_epi_val(acc[i0], bb, act), tg_epi_val(acc[i0 + 1], bb, act));
        const __half2 r1 = __floats2half2_rn(tg_epi_val(acc[i1], bb, act), tg_epi_val(acc[i1 + 1], bb, act));
        const __half2 mx = __hmax2(r0, r1);
        v[e] = __hmax(__low2half(mx), __high2half(mx));
      }
      const __half2 o = __halves2half2(v[0], v[1]);
      ov[m] = *reinterpret_cast<const uint32_t*>(&o);
    }
    stmatrix_x4_trans(tile + (uint32_t)ip * 16u * pitch + mat_off, ov);
  }
}

// ---- host side: tensor maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// fp16 tensor of `rank` dims (dims[0] contiguous), element strides of dims 1.., 128B swizzle (or none)
inline int encode_f16(CUtensorMap* m, const void* ptr, int rank, const cuuint64_t* dims, const size_t* elem_strides,
                      const cuuint32_t* box, bool swizzle = true) {
  EncodeTiledFn fn = get_encode_fn();
  TG_REQUIRE(fn != nullptr, TG_E_DRIVER, "cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t strides[4];
  for (int i = 0; i + 1 < rank; ++i) strides[i] = (cuuint64_t)elem_strides[i] * 2;
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides, box,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  TG_REQUIRE(r == CUDA_SUCCESS, TG_E_DRIVER,
             "cuTensorMapEncodeTiled failed (%d) rank=%d dims=%llux%llux%llux%llu box=%ux%ux%u", (int)r, rank,
             (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2],
             (unsigned long long)dims[3], box[0], box[1], box[2]);
  return TG_OK;
}

// NHWC fp16 tensor [n][h][w][c] with explicit element strides for w/h/n (parity views)
inline int encode_nhwc(CUtensorMap* m, const void* ptr, int c, int w, int h, int n, size_t sw, size_t sh, size_t sn,
                       int box_c, int box_w, int box_h, bool swizzle = true) {
  const cuuint64_t dims[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
  const size_t strides[3] = {sw, sh, sn};
  const cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
  return encode_f16(m, ptr, 4, dims, strides, box, swizzle);
}

}  // namespace
