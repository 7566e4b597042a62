// The fused SRNet tail on sm_90a (H100), built from the same TMA / mbarrier / wgmma pieces as tg_conv_wgmma.cu.
//
// convT_convout_kernel: last ConvTranspose2d(64,64,3,2,1,op=1) + ReLU -> conv_out 3x3
//   (64 -> out_nc <= 3) -> + upsample_func(lr_curr) or + the pre-written frame -> fp32 NCHW (+ uint8 NHWC).
//   Per 16x8 tile of the transposed conv's input (17x9 halo box), parity by parity: the transposed conv
//   runs pixels-on-N (M = 64 couts, N = the 128 input pixels, one m64n128k16 per (tap group, k-step));
//   its accumulators are written, +bias, ReLU, fp16, by stmatrix into one 128-pixel K-major 128B-swizzled
//   operand block (pixels outside the image are zero = conv_out's zero padding); conv_out runs as
//   m64n40 wgmmas on that block, N packed so that one thread holds all nine tap products of one cout
//   for its pixels; the tap products are summed into the output pixels they land on in registers
//   (x-neighbours by shuffle, y-neighbours in the thread's other row or, across warps, through a small
//   edge buffer).  The tile's 30x14 interior HR pixels are outputs (tiles advance by 15x7 input pixels,
//   the transposed conv is recomputed on a one-pixel ring).
//   Warpgroup 0 runs the transposed conv with two accumulator sets, so parity a + 1's MMAs are in flight
//   under parity a's epilogue; warpgroups 1 and 2 run conv_out, the summation and the global I/O of
//   alternate tiles, each fed through its own two operand blocks.  The 64-channel HR map never reaches HBM.
#include <cuda.h>

#include "tg_common.cuh"
#include "tg_wgmma.cuh"

namespace {

constexpr uint32_t kWtBytes = 9 * 64 * 128;          // nine [64 cout][64 cin] fp16 weight tiles

// warpgroup 0 (WG-T) runs the transposed conv and its epilogue; warpgroups 1 and 2 (WG-O 0 / 1) run conv_out and
// the output of alternate tiles.  No producer warp: WG-T's thread 0 issues the halo TMAs.  WG-T holds two
// 64-register accumulator sets, each WG-O the conv_out products and the 16 output sums.
constexpr int kTailThreads = 384;
constexpr int kStepY = 15, kStepX = 7;               // input pixels a tile advances by
constexpr uint32_t kTailHalo = (TW + 1) * (TH + 1) * 128;            // 19584
constexpr uint32_t kTailStage = (kTailHalo + 1023u) & ~1023u;        // 20480
constexpr int kTailStages = 2;                       // halo ring: the tile in use + the next one loading
constexpr uint32_t kWoBytes = TG_TAIL_OUT_ROWS * 128;                // [40 rows][64], see pack_tail_out_kernel
constexpr uint32_t kHrBlock = 128 * 128;                             // one parity block: 128 px x 128 B
// a WG-O's edge buffer: per parity (a & 1), per row pair w = 4 * m-block + warp (slots 1..8; slots 0 and 9 pad the
// reads of the tile's first and last block rows, whose sums are never stored), per lane one tap row (3 of 4 floats)
constexpr uint32_t kEdgeBytes = 2 * 10 * 32 * 16;                    // 10240
// a WG-O's finished sums of one tile, [32 HR rows][16 HR columns][4] fp32 (3 couts + pad): they pass from the
// threads that summed them (one cout, 16 pixels) to the threads that store them (one pixel, 3 couts)
constexpr uint32_t kSumBytes = 32 * 16 * 16;                         // 8192
// layout: header | w_up | w_out | edge buffers and sums of WG-O 0 and 1 | 2 halo stages | 2 operand blocks per WG-O
constexpr uint32_t kTailOffWt = 2048;
constexpr uint32_t kTailOffWo = kTailOffWt + kWtBytes;               // 75776
constexpr uint32_t kTailOffEdge = kTailOffWo + kWoBytes;             // 80896
constexpr uint32_t kTailOffSum = kTailOffEdge + 2 * kEdgeBytes;      // 101376
constexpr uint32_t kTailOffHalo = kTailOffSum + 2 * kSumBytes;       // 117760
constexpr uint32_t kTailOffBlk = kTailOffHalo + kTailStages * kTailStage;   // 158720
constexpr uint32_t kTailSmem = 1024 + kTailOffBlk + 4 * kHrBlock;    // 225280
static_assert(kTailSmem <= kSmemLimit, "tail smem");
static_assert(kTailOffWo % 1024 == 0 && kTailOffHalo % 1024 == 0 && kTailOffBlk % 1024 == 0, "swizzle atoms");

struct TailParams {
  CUtensorMap map_x;
  const unsigned char* w_up;
  const unsigned char* w_out;
  const float* b_up;
  const float* b_out;
  const float* lr;
  float* y;
  uint8_t* y_u8;
  int n, h, w, cout_real, lr_scale, up_mode, accumulate;
  int tiles_x, tiles_y, num_tiles;
};

// conv_out's weights as the tail reads them: one 128B-swizzled [40 rows][64 k] tile, tap t of cout co in row
// 8 * (t >> 1) + 2 * co + (t & 1).  In an m64n40 accumulator fragment lane l holds columns 8j + 2 (l & 3) + e, so
// lane quad position co holds all nine tap products of cout co (rows of co = 3 and of tap 9 are zero).
__global__ void pack_tail_out_kernel(const float* __restrict__ w, __half* __restrict__ packed, int cout, int cin) {
  tg_pdl_wait();
  // no early trigger: the weights this kernel writes are loaded by the next tail BEFORE its PDL wait
  for (int i = threadIdx.x; i < TG_TAIL_OUT_ROWS * 64; i += blockDim.x) {
    const int k = i % 64, row = i / 64;
    const int tap = 2 * (row >> 3) + (row & 1), co = (row >> 1) & 3;
    float v = 0.f;
    if (tap < 9 && co < cout && k < cin) v = w[(((size_t)co * cin + k) * 3 + tap / 3) * 3 + tap % 3];
    *reinterpret_cast<__half*>(reinterpret_cast<unsigned char*>(packed) + tg_wtile_off(row, k)) = __float2half(v);
  }
}

// fp16 pair of tg_act(v, TG_ACT_RELU) = fmaxf(v, v * 0).  For finite v that is v when v >= +0 and -0 when v < 0 or
// v = -0; rounding to fp16 keeps the sign, so the pair is the rounded v with every half whose sign bit is set replaced
// by -0 (0x8000): prmt replicates each half's sign bit over the half, lop3 selects.  Same bits, three integer
// instructions per pair instead of two multiplies and two max.
__device__ __forceinline__ uint32_t relu_f16x2(float v0, float v1) {
  const __half2 hv = __floats2half2_rn(v0, v1);
  const uint32_t h = *reinterpret_cast<const uint32_t*>(&hv);
  uint32_t neg;
  asm("prmt.b32 %0, %1, 0, 0xBB99;" : "=r"(neg) : "r"(h));
  return (h & ~neg) | (neg & 0x80008000u);
}

// WG-T's epilogue of one parity: pxn_store_tile with ReLU, except that input pixels outside the image become zero
// (conv_out's zero padding) -- a per-element predicate the conv kernels have no use for, so it is its own loop.  The
// predicate is a mask per fp16 pair (the thread's two columns are fixed per tile, the row test is one compare); the
// tiles whose 16x8 input pixels all lie in the image skip it.
template <bool kEdge>
__device__ __forceinline__ void tail_convT_store(const float (&acc)[64], uint32_t blk, uint32_t mat_off, float b0,
                                                 float b1, int y0, int x0, int lane, int h, int w) {
  const int ix = x0 + 2 * (lane & 3);
  const uint32_t xmask = ((unsigned)ix < (unsigned)w ? 0x0000FFFFu : 0u) |
                         ((unsigned)(ix + 1) < (unsigned)w ? 0xFFFF0000u : 0u);
#pragma unroll
  for (int jp = 0; jp < 8; ++jp) {
    uint32_t ov[4];
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int i = 4 * (2 * jp + (m >> 1)) + 2 * (m & 1);
      const float bb = (m & 1) ? b1 : b0;
      ov[m] = relu_f16x2(acc[i] + bb, acc[i + 1] + bb);
      if (kEdge) ov[m] &= (unsigned)(y0 + 2 * jp + (m >> 1)) < (unsigned)h ? xmask : 0u;
    }
    stmatrix_x4_trans(blk + (uint32_t)jp * 2048u + mat_off, ov);
  }
}
__device__ __forceinline__ void tail_convT_epilogue(const float (&acc)[64], uint32_t blk, uint32_t mat_off, float b0,
                                                    float b1, int y0, int x0, int lane, int h, int w) {
  if (y0 >= 0 && y0 + 16 <= h && x0 >= 0 && x0 + 8 <= w)
    tail_convT_store<false>(acc, blk, mat_off, b0, b1, y0, x0, lane, h, w);
  else
    tail_convT_store<true>(acc, blk, mat_off, b0, b1, y0, x0, lane, h, w);
}

__global__ void __launch_bounds__(kTailThreads, 1) convT_convout_kernel(const __grid_constant__ TailParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (base - raw);
  const int warp = __shfl_sync(0xFFFFFFFFu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  // bar_halo[s]: halo stage s has landed (TMA bytes).  bar_full[2c + b] / bar_empty[2c + b]: WG-O c's operand
  // block b has been written by WG-T (one arrival per WG-T warp) / read by WG-O c's conv_out MMAs (one arrival per
  // WG-O warp).
  const uint32_t bar_halo = base, bar_w = base + 32, bar_full = base + 40, bar_empty = base + 72;
  float* bup_s = reinterpret_cast<float*>(sm + 1024);
  float* bout_s = reinterpret_cast<float*>(sm + 1024 + 256);

  if (threadIdx.x == 0) {
    for (int s = 0; s < kTailStages; ++s) mbar_init(bar_halo + 8 * s, 1);
    mbar_init(bar_w, 1);
    for (int b = 0; b < 4; ++b) {
      mbar_init(bar_full + 8 * b, 4);
      mbar_init(bar_empty + 8 * b, 4);
    }
    fence_barrier_init();
  }
  __syncthreads();
  // weights are static: load them before the programmatic-dependent-launch wait
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.map_x);
    mbar_expect_tx(bar_w, kWtBytes + kWoBytes);
    for (int t = 0; t < 9; ++t) bulk_load(base + kTailOffWt + t * 8192u, p.w_up + (size_t)t * 8192u, 8192u, bar_w);
    bulk_load(base + kTailOffWo, p.w_out, kWoBytes, bar_w);
  }
  tg_pdl_wait();
  tg_pdl_trigger();
  if (threadIdx.x < 64) bup_s[threadIdx.x] = __ldg(p.b_up + threadIdx.x);
  if (threadIdx.x < 4) bout_s[threadIdx.x] = threadIdx.x < p.cout_real ? __ldg(p.b_out + threadIdx.x) : 0.f;
  __syncthreads();
  const int per_img = p.tiles_x * p.tiles_y;
  const int grid = (int)gridDim.x;
  const int r = threadIdx.x & 127, q = r >> 5;
  const uint32_t blk0 = base + kTailOffBlk;

  // WG-T walks the CTA's tiles blockIdx.x + i * gridDim.x, parity a = 0..3 of each; WG-O c takes the tiles with
  // i % 2 == c.  Parity a of a tile goes through its WG-O's operand block a & 1, so each block is used twice per
  // tile of that WG-O and its k-th use has mbarrier phase k & 1 = a >> 1.  Deadlock-free: WG-T waits only on halo
  // stages (its own TMAs) and on bar_empty of a block whose previous use it has already published; WG-O waits only
  // on bar_full, which WG-T arrives on without waiting for anything later than that block's previous release.
  // Waits and arrivals on each block barrier alternate, so a parity wait is never more than one phase behind.
  if (warp < 4) {
    // ============================================================ WG-T: halo TMAs, transposed conv, epilogue
    const uint32_t wt16 = gmma_addr16(base + kTailOffWt);
    const uint32_t mat_off = pxn_mat_off(lane, q, 128u, /*swizzled=*/true, /*pool=*/false);
    const float b0 = bup_s[16 * q + (lane >> 2)], b1 = bup_s[16 * q + (lane >> 2) + 8];
    // the CTA's i-th tile goes to halo stage i % 2
    auto load_halo = [&](int tile, int st) {
      const int img = tile / per_img, rr = tile - img * per_img;
      mbar_expect_tx(bar_halo + 8 * st, kTailHalo);
      tma_load_4d(base + kTailOffHalo + (uint32_t)st * kTailStage, &p.map_x, bar_halo + 8 * st, 0,
                  (rr % p.tiles_x) * kStepX - 1, (rr / p.tiles_x) * kStepY - 1, img);
    };
    if (r == 0)
      for (int k = 0; k < 2; ++k)
        if ((int)blockIdx.x + k * grid < p.num_tiles) load_halo((int)blockIdx.x + k * grid, k);
    int stage = 0;
    uint32_t phase = 0;
    int py0 = 0, px0 = 0;     // origin of the previous tile: its parity 3 is written under this tile's parity 0
    uint32_t cur = 0;         // 2 * (WG-O of the current tile): index of its first operand block
    float acc[2][64];         // parity a accumulates into acc[a & 1]
    mbar_wait_mma(bar_w, 0);
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += grid, cur ^= 2u) {
      const int img = tile / per_img, rr = tile - img * per_img;
      const int y0 = (rr / p.tiles_x) * kStepY - 1, x0 = (rr % p.tiles_x) * kStepX - 1;
      const int s = stage;
      mbar_wait_mma(bar_halo + 8 * s, phase);
      if (++stage == kTailStages) { stage = 0; phase ^= 1u; }
      const uint32_t x16 = gmma_addr16(base + kTailOffHalo + (uint32_t)s * kTailStage);
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        wgmma_fence();
        convT_pxn_mmas(acc[a & 1], x16, wt16, a);
        wgmma_commit();
        // parity a - 1 (for a = 0: the previous tile's parity 3) has landed; parity a stays in flight under its
        // epilogue
        wgmma_wait<1>();
        if (a == 0) {
          // every warp is past the previous tile's last MMAs: its halo stage takes the next tile
          named_bar_sync(1, 128);
          if (r == 0 && tile != (int)blockIdx.x && tile + grid < p.num_tiles) load_halo(tile + grid, s ^ 1);
        }
        if (a > 0 || tile != (int)blockIdx.x) {
          const int e = (a + 3) & 3;       // the parity written now
          const uint32_t b = (a > 0 ? cur : cur ^ 2u) + ((uint32_t)e & 1u);
          // the WG-O's MMAs have read this block's previous use (parity e - 2 of its tile, or of its previous tile)
          mbar_wait_mma(bar_empty + 8 * b, (uint32_t)((e >> 1) & 1) ^ 1u);
          tail_convT_epilogue(acc[e & 1], blk0 + b * kHrBlock, mat_off, b0, b1, a > 0 ? y0 : py0, a > 0 ? x0 : px0,
                              lane, p.h, p.w);
          fence_proxy_async_smem();        // generic-proxy writes -> read by wgmma (async proxy)
          __syncwarp();
          if (lane == 0) mbar_arrive(bar_full + 8 * b);
        }
      }
      py0 = y0;
      px0 = x0;
    }
    // the last tile's parity 3
    wgmma_wait<0>();
    if ((int)blockIdx.x < p.num_tiles) {
      const uint32_t b = (cur ^ 2u) + 1u;
      mbar_wait_mma(bar_empty + 8 * b, 0u);
      tail_convT_epilogue(acc[1], blk0 + b * kHrBlock, mat_off, b0, b1, py0, px0, lane, p.h, p.w);
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_full + 8 * b);
    }
  } else {
    // ============================================================ WG-O c: conv_out, register shift-add, output
    const int c = (warp >> 2) - 1;
    const uint32_t wo16 = gmma_addr16(base + kTailOffWo);
    const uint64_t k_hi = gmma_desc_hi(1024u);
    // The thread's conv_out fragment: block pixels (row 8h + 2q + rb, column bx) for h, rb = 0, 1 (pixel row
    // j = 2h + rb), all nine taps of cout cq (lane quad position 3 is padding).  The thread owns the HR outputs of
    // those block pixels, (2 * row + ey, 2 * bx + ex) as o[j][e = 2ey + ex], of cout cq; the interior 30x14 of the
    // tile's 32x16 are stored.
    const int bx = lane >> 2, cq = lane & 3;
    float4* edge = reinterpret_cast<float4*>(sm + kTailOffEdge + (uint32_t)c * kEdgeBytes);
    float* sums = reinterpret_cast<float*>(sm + kTailOffSum + (uint32_t)c * kSumBytes);
    // the pad slots feed only sums that are never stored; zero them once.  Every thread passes the first parity's
    // named barrier after this store, before any read.
    edge[(r >> 6) * 320 + ((r >> 5) & 1) * 288 + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
    const int H = 2 * p.h, W = 2 * p.w;
    const int lh = H / p.lr_scale, lw = W / p.lr_scale;
    mbar_wait_mma(bar_w, 0);
    for (int tile = blockIdx.x + c * grid; tile < p.num_tiles; tile += 2 * grid) {
      const int img = tile / per_img, rr = tile - img * per_img;
      const int y0 = (rr / p.tiles_x) * kStepY - 1, x0 = (rr % p.tiles_x) * kStepX - 1;
      // the frame this tile adds onto is loaded into the output registers now; the loads complete under the MMAs
      float o[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int Y = 2 * (8 * (j >> 1) + 2 * q + (j & 1)) + (e >> 1), X = 2 * bx + (e & 1);
          const int gy = 2 * y0 + Y, gx = 2 * x0 + X;
          const bool ok = Y >= 1 && Y <= 30 && X >= 1 && X <= 14 && gy >= 0 && gy < H && gx >= 0 && gx < W;
          o[j][e] = 0.f;
          if (p.accumulate && ok && cq < p.cout_real)
            o[j][e] = p.y[(((size_t)img * p.cout_real + cq) * H + gy) * W + gx];
        }
      // parity a = (py, px) of the HR pixels: operand block -> conv_out tap products -> summed into the output
      // pixels they land on
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        const int py = a >> 1, px = a & 1;
        const uint32_t b = 2u * (uint32_t)c + ((uint32_t)a & 1u);
        const uint32_t blk16 = gmma_addr16(blk0 + b * kHrBlock);
        mbar_wait_mma(bar_full + 8 * b, (uint32_t)py);
        float d2[2][20];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_n40(d2[0], k_hi | (uint64_t)(blk16 + 2u * k), k_hi | (uint64_t)(wo16 + 2u * k), k > 0 ? 1u : 0u);
          wgmma_n40(d2[1], k_hi | (uint64_t)(blk16 + 512u + 2u * k), k_hi | (uint64_t)(wo16 + 2u * k), k > 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * b);   // WG-T may write the block's next use
        // tap t of pixel row j
        auto P = [&](int j, int t) { return d2[j >> 1][4 * (t >> 1) + 2 * (j & 1) + (t & 1)]; };
        // HR pixel (Y, X) takes tap (ty, tx) from HR pixel (Y + ty - 1, X + tx - 1), which is in this parity block
        // for ty = 1 if Y % 2 == py, else for ty = 0 and 2 (the same in x).  One of those two taps comes from the
        // neighbouring block pixel: tap column txn from column bx + 1 (lane + 4) for px = 0, bx - 1 (lane - 4) for
        // px = 1; tap row tyn from block row + dy.
        const int dy = py ? -1 : 1, tyn = py ? 0 : 2, txn = px ? 0 : 2;
        float xs[4][3];   // tap (ty, txn) of the x-neighbour
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int ty = 0; ty < 3; ++ty)
            xs[j][ty] = px ? __shfl_up_sync(0xFFFFFFFFu, P(j, 3 * ty), 4)
                           : __shfl_down_sync(0xFFFFFFFFu, P(j, 3 * ty + 2), 4);
        // tap row tyn of pixel row j as the pixel row above / below it takes it (column txn from the x-neighbour)
        auto nrow = [&](int j, int tx) { return tx == txn ? xs[j][tyn] : P(j, 3 * tyn + tx); };
        // pixel row 2h + py is the y-neighbour of a row of another warp (or of the other m-block): it goes through
        // the edge buffer of this parity, slot 1 + 4h + q; double-buffering by a & 1 lets one barrier per parity
        // order both the writes after the last reads of the previous use and the reads after the writes
        float4* eb = edge + (a & 1) * 320 + (1 + q) * 32 + lane;
#pragma unroll
        for (int h = 0; h < 2; ++h)
          eb[h * 128] = make_float4(nrow(2 * h + py, 0), nrow(2 * h + py, 1), nrow(2 * h + py, 2), 0.f);
        named_bar_sync(2 + c, 128);
        float ny[4][3];   // tap row tyn of pixel row j's y-neighbour
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float4 v = eb[h * 128 + dy * 32];
          ny[2 * h + 1 - py][0] = v.x;
          ny[2 * h + 1 - py][1] = v.y;
          ny[2 * h + 1 - py][2] = v.z;
#pragma unroll
          for (int tx = 0; tx < 3; ++tx) ny[2 * h + py][tx] = nrow(2 * h + 1 - py, tx);
        }
        // each output adds its taps of this parity in slot order (ty, then tx), as the nine taps of a pixel are
        // split over the four parities
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int ey = e >> 1, ex = e & 1;
#pragma unroll
            for (int sl = 0; sl < 4; ++sl) {
              const int ty = (ey == py ? 1 : 0) + 2 * (sl >> 1), tx = (ex == px ? 1 : 0) + 2 * (sl & 1);
              if (ty > 2 || tx > 2) continue;
              const bool ynb = ey != py && ty == tyn, xnb = ex != px && tx == txn;
              o[j][e] += ynb ? ny[j][tx] : xnb ? xs[j][ty] : P(j, 3 * ty + tx);
            }
            // the sums are done before the next parity's MMAs are issued: sinking them past those would keep
            // this parity's tap products live next to the next one's accumulators
            asm volatile("" : "+f"(o[j][e]));
          }
      }
      // the sums pass to one thread per HR pixel (Y0 + 8j, X) with all couts, as values, for the output stage.  The
      // next tile writes them only after its parity barriers, which every thread passes after its reads here.
      const int Y0 = r >> 4, X = r & 15;
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (cq < 3) sums[((2 * (8 * (j >> 1) + 2 * q + (j & 1)) + (e >> 1)) * 16 + 2 * bx + (e & 1)) * 4 + cq] = o[j][e];
      named_bar_sync(2 + c, 128);
      // + bias (+ upsample_func(lr)) -> fp32 NCHW (+ uint8 NHWC), one pixel per iteration: the in-kernel upsample is
      // inlined three times rather than twelve.
#pragma unroll 1
      for (int j = 0; j < 4; ++j) {
        const float4 s = reinterpret_cast<const float4*>(sums)[(Y0 + 8 * j) * 16 + X];
        const float oj[3] = {s.x, s.y, s.z};
        const int Y = Y0 + 8 * j, gy = 2 * y0 + Y, gx = 2 * x0 + X;
        if (Y < 1 || Y > 30 || X < 1 || X > 14 || gy < 0 || gy >= H || gx < 0 || gx >= W) continue;
        uint32_t q8[3] = {0u, 0u, 0u};
#pragma unroll
        for (int co = 0; co < 3; ++co) {
          if (co >= p.cout_real) continue;
          float v = oj[co] + bout_s[co];
          if (p.lr) v = v + tg_upsample_at(p.lr + ((size_t)img * p.cout_real + co) * lh * lw, lh, lw, lh, lw,
                                           p.lr_scale, p.up_mode, gy, gx);
          p.y[(((size_t)img * p.cout_real + co) * H + gy) * W + gx] = v;
          q8[co] = (uint32_t)fminf(fmaxf(rintf(v * 255.f), 0.f), 255.f);
        }
        if (p.y_u8) {
          uint8_t* up = p.y_u8 + (((size_t)img * H + gy) * W + gx) * p.cout_real;
#pragma unroll
          for (int co = 0; co < 3; ++co)
            if (co < p.cout_real) up[co] = (uint8_t)q8[co];
        }
      }
    }
  }
}

}  // namespace

extern "C" {

int tg_pack_tail_out_weights(const float* w_oihw, int cout, int cin, void* packed, void* stream) {
  TG_REQUIRE(w_oihw && packed, TG_E_INVALID, "pack_tail_out: null pointer");
  TG_REQUIRE(cout >= 1 && cout <= 3 && cin >= 1 && cin <= 64, TG_E_UNSUPPORTED,
             "pack_tail_out: cout=%d (1..3) cin=%d (<= 64)", cout, cin);
  tg_launch(pack_tail_out_kernel, dim3(1), dim3(256), 0, (cudaStream_t)stream, w_oihw, (__half*)packed, cout, cin);
  TG_CUDA_LAUNCH_CHECK("pack_tail_out");
  return TG_OK;
}

int tg_convT_convout_tcgen05(const tg_tail_desc* d, void* stream) {
  TG_REQUIRE(d != nullptr, TG_E_INVALID, "convT_convout: null descriptor");
  TG_REQUIRE(d->x && d->w_up && d->b_up && d->w_out && d->b_out && d->y, TG_E_INVALID, "convT_convout: null pointer");
  TG_REQUIRE(d->n > 0 && d->h > 0 && d->w > 0, TG_E_INVALID, "convT_convout: bad size");
  TG_REQUIRE(d->cout_real >= 1 && d->cout_real <= 3, TG_E_UNSUPPORTED, "convT_convout: out_nc=%d (1..3)", d->cout_real);
  TG_REQUIRE(d->reserved == 0, TG_E_INVALID, "convT_convout: reserved must be 0");
  TG_REQUIRE(!(d->accumulate && d->lr), TG_E_INVALID, "convT_convout: accumulate and lr are exclusive");
  TG_REQUIRE(((uintptr_t)d->x & 15) == 0 && ((uintptr_t)d->w_up & 15) == 0 && ((uintptr_t)d->w_out & 15) == 0 &&
                 ((uintptr_t)d->y & 7) == 0, TG_E_INVALID, "convT_convout: pointer alignment");
  if (d->lr != nullptr) {
    TG_REQUIRE(d->lr_scale == 2 || d->lr_scale == 4, TG_E_UNSUPPORTED, "convT_convout: lr_scale %d (2 or 4)", d->lr_scale);
    TG_REQUIRE((2 * d->h) % d->lr_scale == 0 && (2 * d->w) % d->lr_scale == 0, TG_E_INVALID,
               "convT_convout: output size is not lr_scale x the LR size");
    TG_REQUIRE(d->up_mode == TG_UP_BICUBIC || d->up_mode == TG_UP_BILINEAR, TG_E_INVALID, "convT_convout: up_mode");
  }
  TailParams p;
  // NHWC fp16 [n][h][w][64], one 17x9 px halo box of all 64 channels per tile
  int rc = encode_nhwc(&p.map_x, d->x, 64, d->w, d->h, d->n, 64, (size_t)d->w * 64, (size_t)d->h * d->w * 64, 64,
                       TW + 1, TH + 1);
  if (rc != TG_OK) return rc;
  p.w_up = reinterpret_cast<const unsigned char*>(d->w_up);
  p.w_out = reinterpret_cast<const unsigned char*>(d->w_out);
  p.b_up = d->b_up; p.b_out = d->b_out; p.lr = d->lr; p.y = d->y; p.y_u8 = d->y_u8;
  p.n = d->n; p.h = d->h; p.w = d->w; p.cout_real = d->cout_real;
  p.lr_scale = d->lr ? d->lr_scale : 2; p.up_mode = d->up_mode; p.accumulate = d->accumulate;
  // HR rows -1 .. 2h-1 are covered in strips of 30 (the first strip starts at the even row -2)
  p.tiles_y = tg_ceil_div(2 * d->h + 1, 2 * kStepY);
  p.tiles_x = tg_ceil_div(2 * d->w + 1, 2 * kStepX);
  p.num_tiles = p.tiles_x * p.tiles_y * d->n;
  static TgPerDeviceOnce attr_once;
  const cudaError_t attr_err = attr_once.run([] {
    return cudaFuncSetAttribute(convT_convout_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTailSmem);
  });
  TG_REQUIRE(attr_err == cudaSuccess, (int)attr_err, "convT_convout: cudaFuncSetAttribute: %s",
             cudaGetErrorString(attr_err));
  int sms = 0;
  rc = tg_device_sm_count(&sms);
  if (rc != TG_OK) return rc;
  int grid = d->max_ctas > 0 && d->max_ctas < sms ? d->max_ctas : sms;
  if (grid > p.num_tiles) grid = p.num_tiles;
  const cudaError_t lerr =
      tg_launch(convT_convout_kernel, dim3(grid), dim3(kTailThreads), kTailSmem, (cudaStream_t)stream, p);
  TG_REQUIRE(lerr == cudaSuccess, (int)lerr, "convT_convout: launch failed: %s", cudaGetErrorString(lerr));
  TG_CUDA_LAUNCH_CHECK("convT_convout");
  return TG_OK;
}

}  // extern "C"
