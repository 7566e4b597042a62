// 3x3 convolution / stride-2 transposed convolution / stride-2 convolution as a persistent,
// warp-specialised wgmma implicit GEMM for sm_90a (H100).
//
//   M tile  = 128 output pixels = a 16x8 patch of one image (row m <-> pixel (m>>3, m&7)), issued as
//             two m64 wgmmas (tile rows 0-7 and 8-15)
//   N       = 64 output channels per CTA (layers with 128 ... 384 are split over 2 ... 6 CTAs); 48 for
//             the thin heads (MODE_TAPN: 9 taps x 4 couts in N, 3x3 shift-add in the epilogue)
//   K       = 64-channel chunks x 9 taps; wgmma K = 16 -> 4 k-steps per (tap, chunk)
//   A       : NHWC fp16 activations, fetched by TMA (4-D tiled map, 128B swizzle, OOB zero fill =
//             the conv's zero padding) either as ONE halo box (18x10 px) per (tile, chunk) whose
//             nine shifted views are addressed through the wgmma descriptor (start address +=
//             (dy*10+dx)*128 B, 8-row-group stride = 10*128 B), or as one 16x8 box per tap.
//   B       : weights pre-packed on the device in the exact swizzled smem image
//             (tg_pack_*_weights), either resident in smem for the whole kernel (SRNet, thin
//             FNet layers, one K chunk per CTA of a cluster for the 128 / 256-channel FNet layers: see
//             consumer_splitk) or streamed per (tap, chunk) with cp.async.bulk (tap mode).
//   D       : fp32 accumulators in the registers of the consumer warpgroup (64 per thread).
//   roles   : warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = consumers that take the
//             CTA's tiles alternately, each with its own ring of smem stages (the forward pixels-on-N
//             conv3x3 has three consumers on one shared ring, see below).  Data gradients, the
//             stride-2 conv, the tap-mode kernels and the thin heads keep the pixels on M: wgmma ->
//             accumulators staged to a per-consumer fp32 smem tile -> one thread per pixel applies bias /
//             act / residual (or the derivative, pool, pixel-shuffle and thin-head epilogues) and writes
//             the pixel's 128-byte NHWC row.
//             The tap-mode transposed conv keeps 4 parity accumulators (1/2/2/4 taps), computed and
//             stored one after the other; each stores its pixel's output of that parity (pixel shuffle).
//
// The forward halo conv and transposed conv with NHWC output (the SRNet body, the first SRNet
// transposed conv and the FNet halo layers, pooled or not; see consumer_halo_pxn / consumer_convT_pxn /
// consumer_splitk) swap the GEMM's roles: M = the 64 output channels (the packed weight tile is the
// K-major A operand), N = the tile's 128 pixels (the halo view is the K-major B operand, 16 core groups
// of 8 pixels), so each (tap, k-step) is ONE m64n128k16 that reads 6 KB of smem instead of two m64n64k16
// that read 8 KB.  The epilogue works from registers: bias / act / residual -> fp16 -> stmatrix into a
// 16 KB tile in the TMA box image -> one TMA tensor store per tile (per parity for the transposed conv,
// into a 5-D view of its output); the residual arrives in that tile by one TMA load issued before the
// tile's MMAs.  With the pool, the 2x2 max is taken in registers and a 4 KB pooled tile is stored.
// On the conv3x3 and split-K paths the consumers take turns issuing their MMAs, so that one's epilogue
// runs under the others' MMAs.  The conv3x3 (consumer_halo_pxn) runs three consumer warpgroups (512
// threads) on one four-stage halo ring filled in tile order, so each epilogue has two other consumers'
// MMA turns to hide under; a bottom tile row with at most 8 rows inside the image issues m64n64k16 over
// its first 8 tile rows.  The transposed conv keeps two consumers with two halo stages each.  The
// mainloop and epilogue pieces (halo_pxn_mmas, convT_pxn_mmas, pxn_store_tile) are in tg_wgmma.cuh; the
// fused SRNet tail (tg_tail.cu) uses the same ones.
#include <cuda.h>

#include <cstdlib>
#include <type_traits>

#include "tg_common.cuh"
#include "tg_wgmma.cuh"

namespace {

constexpr int kMaxRing = 4;               // smem stages per ring
constexpr int kBiasBar = 4;               // named barrier of all consumer warpgroups (1 + cw: one consumer's)
constexpr uint32_t kHeaderBytes = 2048;   // barriers (first 1 KB) + bias (second 1 KB; 2 KB for cout = 384, 512)
constexpr uint32_t kTapABytes = TH * TW * 128;  // 16 KB
constexpr uint32_t kPoolTileBytes = kTapABytes / 4;   // the pooled 8x4 px x 64 ch output tile
// A-operand modes (template parameter MODE)
constexpr int MODE_TAP = 0;    // one 16x8 box per (tap, chunk)
constexpr int MODE_HALO = 1;   // one 18x10 halo box per (tile, chunk), taps = descriptor shifts
constexpr int MODE_TAPN = 2;   // thin heads: one 16x8 box per (tile, chunk), N = 9 taps x 4 couts,
                               // 3x3 shift-add in the epilogue; tiles overlap by one pixel ring
constexpr int MODE_SPLITK = 3; // forward conv3x3 with cin 128 / 256: the K chunks split over a cluster
                               // (see consumer_splitk)
constexpr int kTapnStepY = TH - 2, kTapnStepX = TW - 2;   // 14 x 6 valid outputs per TAPN tile
// fp32 staging tile of a consumer: 128 rows x (N + 4) floats (the pad keeps the per-row float4
// reads of the epilogue free of bank conflicts)
__host__ __device__ constexpr uint32_t stage_stride(int mode) { return mode == MODE_TAPN ? 52u : 68u; }
__host__ __device__ constexpr uint32_t scratch_bytes(int mode) { return 128u * stage_stride(mode) * 4u; }
// up to four tensor maps: [0] = the NHWC input; TG_CONV_3X3_S2 reads the input's four parity planes
struct TgMaps { CUtensorMap m[4]; };

struct KParams {
  tg_conv_desc d;
  int tiles_x, tiles_y, num_tiles;
  int chunks, n_acc;
  int halo, b_resident;
  int box_w, box_h, org_x, org_y;
  int step_y, step_x;              // output pixels a tile advances by (16x8; 14x6 for MODE_TAPN)
  int ring;                        // smem stages per ring
  int ksteps;                      // wgmma k-steps (16 channels) per 64-channel chunk that can hold non-zero input (1..4)
  int n_split, bn;                 // output channels are split over n_split CTAs of bn columns
  uint32_t stage_bytes, a_bytes, b_tile_bytes, b_stage_bytes;
  uint32_t off_b, off_stage, off_scratch;   // off_scratch: the consumers' fp32 staging or fp16 output tiles
  uint32_t epi_bytes;              // MODE_SPLITK: per-consumer receive buffer (the output tile overlaps it)
  int reverse;                     // schedule index t works on tile num_tiles - 1 - t (TG_AMODE_REVERSE)
};

// The mbarriers of the header (8 bytes each), every slot named once; c = consumer 0 / 1 (0..2 for res and turn).
// The three consumers of the pixels-on-N conv3x3 share ring 0.
struct ConvBars {
  uint32_t base;
  enum { kFull = 0, kEmpty = 2 * kMaxRing, kWeights = 4 * kMaxRing, kRes, kRecv = kRes + 3, kFree = kRecv + 2,
         kTurn = kFree + 2, kCount = kTurn + 3 };
  __device__ uint32_t at(int slot) const { return base + 8u * (uint32_t)slot; }
  // stage k of ring c: its TMA bytes have landed / its MMAs have read it (one arrival per warp of the consumer)
  __device__ uint32_t full(int c, int k) const { return at(kFull + c * kMaxRing + k); }
  __device__ uint32_t empty(int c, int k) const { return at(kEmpty + c * kMaxRing + k); }
  __device__ uint32_t weights() const { return at(kWeights); }       // the resident weights have landed
  __device__ uint32_t res(int c) const { return at(kRes + c); }      // consumer c's residual tile has landed
  __device__ uint32_t recv(int c) const { return at(kRecv + c); }    // MODE_SPLITK: consumer c's partials received
  __device__ uint32_t handback(int c) const { return at(kFree + c); }   // MODE_SPLITK: peers handed back their buffers
  __device__ uint32_t turn(int c) const { return at(kTurn + c); }    // pixels-on-N conv3x3 / split-K: c may issue
};
static_assert(8 * ConvBars::kCount <= 1024, "the barriers take the first 1 KB of the header");

// The forward halo conv / transposed conv with NHWC output (pooled or not) puts the roles of the GEMM the
// other way round: D[cout][pixel] = W . X^T, the 64 output channels on M and the tile's 128 pixels on N.
template <int KIND, int MODE, bool BWD>
__host__ __device__ constexpr bool pixels_on_n() {
  return (KIND == TG_CONV_3X3 || KIND == TG_CONVT_3X3_S2) && MODE == MODE_HALO && !BWD;
}
// Consumer warpgroups: three for the forward pixels-on-N conv3x3 (consumer_halo_pxn, one shared ring of halo stages),
// two, each with its own ring, for every other instantiation.  The producer warpgroup comes first.
template <int KIND, int MODE, bool BWD>
__host__ __device__ constexpr int conv_consumers() {
  return KIND == TG_CONV_3X3 && pixels_on_n<KIND, MODE, BWD>() ? 3 : 2;
}
template <int KIND, int MODE, bool BWD>
__host__ __device__ constexpr int conv_threads() {
  return 128 * (1 + conv_consumers<KIND, MODE, BWD>());
}

struct TileCoord { int n, y0, x0, nb; };
// Every role maps its schedule index to a tile here, so the walk direction is applied once for all of them.
__device__ __forceinline__ TileCoord tile_coord(const KParams& p, int tile) {
  TileCoord t;
  if (p.reverse) tile = p.num_tiles - 1 - tile;
  const int per_img = p.tiles_x * p.tiles_y;
  const int sp = tile / p.n_split;          // CTAs that share an A tile are adjacent (L2 reuse)
  t.nb = tile - sp * p.n_split;
  t.n = sp / per_img;
  const int r = sp - t.n * per_img;
  t.y0 = (r / p.tiles_x) * p.step_y;
  t.x0 = (r % p.tiles_x) * p.step_x;
  return t;
}

__device__ __forceinline__ void st_global_128x2(void* ptr, const uint4& a, const uint4& b) {
  uint4* q = reinterpret_cast<uint4*>(ptr);
  q[0] = a;
  q[1] = b;
}

// NHWC epilogue of one accumulator for the pixel of tile row r: 64 fp32 values in S[r] -> act(acc + bias)
// [+ residual] (or the derivative epilogue) -> fp16 -> the pixel's 128-byte NHWC row.
template <int KIND, bool BWD, bool POOL>
__device__ __forceinline__ void epilogue_nhwc(const KParams& p, const TileCoord& tc, int r, int lane, int acc,
                                              const float* S, const float* bias_s) {
  const tg_conv_desc& d = p.d;
  const int ty = r >> 3, tx = r & 7;
  const int py = tc.y0 + ty, px = tc.x0 + tx;
  const bool inb = py < d.h && px < d.w;
  constexpr bool kCanRes = KIND != TG_CONVT_3X3_S2;
  const bool has_res = kCanRes && !POOL && (d.residual != nullptr) && inb;
  const bool has_mask = BWD && kCanRes && d.act >= TG_ACT_DRELU && inb;
  const size_t in_off = (((size_t)tc.n * d.h + py) * d.w + px) * d.cout + tc.nb * p.bn;
  int oy = py, ox = px, OW = d.w, OH = d.h;
  if (KIND == TG_CONVT_3X3_S2) { oy = 2 * py + (acc >> 1); ox = 2 * px + (acc & 1); OW = 2 * d.w; OH = 2 * d.h; }
  if (POOL) { OH = d.h >> 1; OW = d.w >> 1; oy = py >> 1; ox = px >> 1; }
  uint4* orow = reinterpret_cast<uint4*>(reinterpret_cast<__half*>(d.y) +
                                         (((size_t)tc.n * OH + oy) * OW + ox) * d.cout + tc.nb * p.bn);
  const float* srow = S + (size_t)r * stage_stride(MODE_TAP);
#pragma unroll
  for (int pc = 0; pc < 2; ++pc) {                // bn == 64: two 32-column pieces
    uint4 res[4], msk[4];
    if (has_res) {
      const uint4* rp = reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(d.residual) + in_off) + pc * 4;
#pragma unroll
      for (int i = 0; i < 4; ++i) res[i] = __ldg(rp + i);
    }
    if (has_mask) {
      const uint4* mp = reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(d.mask) + in_off) + pc * 4;
#pragma unroll
      for (int i = 0; i < 4; ++i) msk[i] = __ldg(mp + i);
    }
    float v[32];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float4 f = reinterpret_cast<const float4*>(srow + pc * 32)[i];
      v[i * 4] = f.x; v[i * 4 + 1] = f.y; v[i * 4 + 2] = f.z; v[i * 4 + 3] = f.w;
    }
    const float4* bias4 = reinterpret_cast<const float4*>(bias_s + tc.nb * p.bn + pc * 32);
    uint4 ov[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __half2* o = reinterpret_cast<__half2*>(&ov[i]);
      const __half2* rh = reinterpret_cast<const __half2*>(&res[i]);
      const __half2* mh = reinterpret_cast<const __half2*>(&msk[i]);
      const float4 b0 = bias4[i * 2], b1 = bias4[i * 2 + 1];
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int cidx = i * 8 + j * 2;
        float a0, a1;
        if (!BWD) {
          a0 = tg_epi_val(v[cidx], bb[j * 2], d.act);
          a1 = tg_epi_val(v[cidx + 1], bb[j * 2 + 1], d.act);
          if (has_res) {
            const float2 rf = __half22float2(rh[j]);
            a0 += rf.x; a1 += rf.y;
          }
        } else {
          a0 = v[cidx] + bb[j * 2];
          a1 = v[cidx + 1] + bb[j * 2 + 1];
          if (has_res) {
            const float2 rf = __half22float2(rh[j]);
            a0 += rf.x; a1 += rf.y;
          }
          if (has_mask) {
            const float2 mf = __half22float2(mh[j]);
            a0 *= tg_dact(mf.x, d.act); a1 *= tg_dact(mf.y, d.act);
          }
        }
        o[j] = __floats2half2_rn(a0, a1);
      }
    }
    if (POOL) {
      // max over the 2x2 block (all 32 lanes take part: lane ^ 1 = x neighbour, lane ^ 8 = y neighbour;
      // floor pooling: blocks that reach outside the image are not stored)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        uint32_t* wv = reinterpret_cast<uint32_t*>(&ov[i]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          uint32_t o1 = __shfl_xor_sync(0xFFFFFFFFu, wv[j], 1);
          __half2 mx = __hmax2(*reinterpret_cast<__half2*>(&wv[j]), *reinterpret_cast<__half2*>(&o1));
          uint32_t m32 = *reinterpret_cast<uint32_t*>(&mx);
          uint32_t o8 = __shfl_xor_sync(0xFFFFFFFFu, m32, 8);
          mx = __hmax2(mx, *reinterpret_cast<__half2*>(&o8));
          wv[j] = *reinterpret_cast<uint32_t*>(&mx);
        }
      }
      if (((tx | ty) & 1) == 0 && py + 1 < d.h && px + 1 < d.w) {
        st_global_128x2(orow + pc * 4, ov[0], ov[1]);
        st_global_128x2(orow + pc * 4 + 2, ov[2], ov[3]);
      }
    } else if (inb) {
      st_global_128x2(orow + pc * 4, ov[0], ov[1]);
      st_global_128x2(orow + pc * 4 + 2, ov[2], ov[3]);
    }
  }
  (void)lane;
}

// ------------------------------------------------------------------ consumer of the pixels-on-N path
// One of the three consumer warpgroups (cw) of the forward 3x3 halo conv, NHWC fp16 output: for each of its tiles
//   D[64 cout][128 px] = sum over (tap, chunk, k-step) of m64n128k16(A = resident weight tile, K-major,
//                        SBO 1024; B = the tap's shifted view of the halo stage, K-major, SBO = one box row)
// then an epilogue from registers into a 16 KB tile in the TMA box image (16x8 px x 64 ch, 128B swizzle)
// that one TMA tensor store writes out (clipped at the image edge).  The residual, if any, is TMA-loaded
// into the same tile before the tile's MMAs and overwritten in place (pxn_store_tile).
// POOL (MaxPool2d(2, 2) folded in, pxn_store_tile_pool2): the pooled 8x4 px x 64 ch tile (4 KB) is stored through
// the pooled tensor's map; clipping at that map's edge is the floor pooling.
// The weights are one 64-channel chunk (cin = 64; wider inputs take the split-K path), so a tile is one halo stage.
template <bool POOL>
__device__ __forceinline__ void consumer_halo_pxn(const TgMaps& maps, const KParams& p, uint32_t base,
                                                  const float* bias_s, int cw) {
  constexpr int kNC = conv_consumers<TG_CONV_3X3, MODE_HALO, false>();
  const tg_conv_desc& d = p.d;
  const int r = threadIdx.x - 128 * (1 + cw);
  const int q = r >> 5, lane = threadIdx.x & 31;
  const ConvBars bars{base};
  const uint32_t bar_res = bars.res(cw);
  const uint32_t stage0 = base + p.off_stage;
  const uint32_t out_s = base + p.off_scratch + (uint32_t)cw * (POOL ? kPoolTileBytes : kTapABytes);
  const uint32_t w16 = gmma_addr16(base + p.off_b), btb16 = p.b_stage_bytes >> 4;
  const bool has_res = !POOL && d.residual != nullptr;
  const int bar_id = 1 + cw;
  // Turns on the tensor pipe.  The CTA's tiles blockIdx.x + i * gridDim.x, i = 0, 1, 2, ..., go to consumer i mod 3.
  // The owner of tile i > 0 issues its MMAs only after the owner of tile i - 1 has issued (and committed) it: it
  // waits on turn[cw], on which the previous consumer's four warps arrive after each of their commits.  The tensor
  // pipe then runs the consumers' MMAs one tile after the other instead of sharing it, and each epilogue runs under
  // the next two consumers' MMAs.  No deadlock: every tile i > 0 has its tile i - 1 in the same CTA, and issuing
  // tile i - 1 waits only for tile i - 2's issue and for memory (the stage, the store drain), never for anything of
  // tile i or later, whatever the consumers' tile counts (0, 1 or unequal).  Waits and arrivals on a barrier
  // alternate (an arrival on turn[c] needs the wait that preceded the arriving consumer's own issue), so a parity
  // wait is never more than one phase behind; the arrival after a consumer's last tile has no waiter and is harmless.
  // The shared ring: tile i is in stage i mod R with parity (i / R) & 1, filled by the producer in tile order.  A
  // parity wait never mistakes an older fill of the stage for tile i's: the owner of tile j + 3 also owned tile j,
  // and it issued tile j only after tile j - 1 had been issued, hence after tile j - 1's stage wait had returned.
  // With R >= 4, tile j + 3 shares its stage with tile j + 3 - R, which is tile j - 1 or earlier, so that fill's
  // phase has completed.  The invariant is ring depth >= consumers + 1 (the host requires R >= 4).
  const uint32_t turn_mine = bars.turn(cw), turn_next = bars.turn(cw + 1 == kNC ? 0 : cw + 1);
  uint32_t tphase = 0;
  const uint32_t mat_off = pxn_mat_off(lane, q, 128u, /*swizzled=*/true, POOL);
  uint32_t rphase = 0;
  float acc[64];

  for (int i = cw;; i += kNC) {
    const int tile = (int)blockIdx.x + i * (int)gridDim.x;
    if (tile >= p.num_tiles) break;
    const TileCoord tc = tile_coord(p, tile);
    if (r == 0) {
      bulk_wait_group_read0();           // the previous tile's store (three tiles back) has left the output tile
      if (has_res) {
        mbar_expect_tx(bar_res, kTapABytes);
        tma_load_4d(out_s, &maps.m[1], bar_res, tc.nb * 64, tc.x0, tc.y0, tc.n);
      }
    }
#pragma unroll
    for (int k = 0; k < 64; ++k) acc[k] = 0.f;
    const int s = i % p.ring;
    mbar_wait_mma(bars.full(0, s), (uint32_t)(i / p.ring) & 1u);
    // take the turn only once the tile's stage is here, so that it is never held while waiting on memory
    if (i > 0) { mbar_wait_mma(turn_mine, tphase); tphase ^= 1u; }
    const uint32_t x16 = gmma_addr16(stage0 + (uint32_t)s * p.stage_bytes);
    auto mmas = [&](auto n, auto ks) {   // each path waits for its own MMAs (see halo_pxn_mmas)
      wgmma_fence();
      halo_pxn_mmas<decltype(n)::value, decltype(ks)::value>(acc, x16, w16, btb16, 1, 0, p.ksteps);
      wgmma_commit();
      __syncwarp();
      if (lane == 0) mbar_arrive(turn_next);   // pass the turn
      wgmma_wait<0>();
    };
    // A bottom tile row with at most 8 rows inside the image: m64n64k16 over rows 0-7 (rows 8-15 keep the zeros).
    // Inputs with all 64 channels real (every layer but FNet's first) run 4 k-steps fixed at compile time.
    using Rows16 = std::integral_constant<int, 128>;
    using Rows8 = std::integral_constant<int, 64>;
    using KSteps4 = std::integral_constant<int, 4>;
    using KStepsRuntime = std::integral_constant<int, 0>;
    const bool half = d.h - tc.y0 <= TH / 2;
    if (p.ksteps == 4) half ? mmas(Rows8{}, KSteps4{}) : mmas(Rows16{}, KSteps4{});
    else half ? mmas(Rows8{}, KStepsRuntime{}) : mmas(Rows16{}, KStepsRuntime{});
    __syncwarp();
    if (lane == 0) mbar_arrive(bars.empty(0, s));

    // the output tile is free once thread 0 saw the previous store read it (it issued the residual load after)
    if (has_res) { mbar_wait_mma(bar_res, rphase); rphase ^= 1u; }
    else named_bar_sync(bar_id, 128);
    const float b0 = bias_s[tc.nb * 64 + 16 * q + (lane >> 2)], b1 = bias_s[tc.nb * 64 + 16 * q + (lane >> 2) + 8];
    if (POOL) pxn_store_tile_pool2(acc, out_s, 128u, mat_off, b0, b1, d.act);
    else pxn_store_tile(acc, out_s, 128u, mat_off, b0, b1, d.act, has_res);
    fence_proxy_async_smem();
    named_bar_sync(bar_id, 128);
    if (r == 0) {
      if (POOL) tma_store_4d(&maps.m[2], out_s, tc.nb * 64, tc.x0 >> 1, tc.y0 >> 1, tc.n);
      else tma_store_4d(&maps.m[2], out_s, tc.nb * 64, tc.x0, tc.y0, tc.n);
      bulk_commit_group();
    }
  }
  // the stores must be complete before the CTA exits (its shared memory goes, and a dependent kernel's
  // griddepcontrol.wait must see the data)
  if (r == 0) bulk_wait_group0();
}

// ------------------------------------------------------------------ consumer of the split-K path
// Forward 3x3 conv with cin = 64 * C (C = 2 or 4), NHWC output (pooled or not).  The C CTAs of a thread-block
// cluster share every (tile, N slice): CTA rank r keeps the weights of K chunk r resident, loads one halo box
// at channel offset 64 r and runs the 64->64 pixels-on-N mainloop of consumer_halo_pxn on it, giving a
// partial D_r[64 cout][128 px].  The partials are reduced through distributed shared memory, partitioned by
// output channel: warp q (couts 16q..16q+15) belongs to rank q / (4 / C).  Each thread of a warp that another
// rank owns sends its 64 accumulators with st.async to the same thread's slot in the owner's receive buffer
// (slot layout [sender slot][owner warp][16 float4][32 lanes]; transaction bytes complete the owner's
// per-consumer "full" barrier).  The owner adds the partials in rank order, p0 + p1 (+ p2 + p3), so the
// result does not depend on which CTA owns the couts or on the grid, then runs the register epilogue and
// stores its 64/C-channel slice of the tile with one TMA store (unswizzled box, 2 * 64/C bytes per pixel).
// The output tile overlaps the receive buffer: once a tile's store has read it, the owner's store thread
// hands the buffer back with a remote arrive on each peer's per-consumer "free" barrier (C - 1 arrivals),
// which a sender waits on before it sends its next tile.  All CTAs of a cluster walk the same tile sequence.
template <bool POOL>
__device__ __forceinline__ void consumer_splitk(const TgMaps& maps, const KParams& p, uint32_t base,
                                                const float* bias_s, int cw) {
  const tg_conv_desc& d = p.d;
  const int r = threadIdx.x - 128 * (1 + cw);
  const int q = r >> 5, lane = threadIdx.x & 31;
  const int C = p.chunks;
  const int rank = (int)cluster_ctarank();
  const int wpr = 4 / C;                   // warps (16 couts each) owned per rank
  const int owner = q / wpr;
  const bool own = owner == rank;
  const bool lead = r == rank * wpr * 32;  // first thread of the rank's first owned warp: stores, hand-backs
  const int sc = 64 / C;                   // output channels per rank
  const uint32_t sb = 2u * (uint32_t)sc;   // bytes per pixel of the rank's output slice tile
  const ConvBars bars{base};
  const uint32_t bar_rfull = bars.recv(cw), bar_free = bars.handback(cw);
  const uint32_t stage0 = base + p.off_stage + (uint32_t)(cw * p.ring) * p.stage_bytes;
  const uint32_t epi_s = base + p.off_scratch + (uint32_t)cw * p.epi_bytes;
  const uint32_t w16 = gmma_addr16(base + p.off_b), btb16 = p.b_stage_bytes >> 4;
  const int bar_id = 1 + cw;
  // where this thread's partial goes in the owner's receive buffer (senders only)
  const int my_slot = rank < owner ? rank : rank - 1;
  const uint32_t send_off = (uint32_t)((my_slot * wpr + (q - owner * wpr)) * 16) * 512u + (uint32_t)lane * 16u;
  const uint32_t peer_buf = mapa_shared(epi_s + send_off, (uint32_t)owner);
  const uint32_t peer_bar = mapa_shared(bar_rfull, (uint32_t)owner);
  const uint32_t recv_bytes = (uint32_t)((C - 1) * wpr) * 8192u;
  // in the rank's dense slice tile, warp q's chunks 2*q + m%2 are local chunks 2*(q - rank*wpr) + m%2 (owners only)
  const uint32_t mat_off = pxn_mat_off(lane, q - rank * wpr, sb, /*swizzled=*/false, POOL);
  const int t0 = (int)cluster_id_x(), tstep = (int)cluster_count_x();
  // turns on the tensor pipe as in consumer_halo_pxn, over the CTA's tiles t0 + i * tstep; the waits for
  // peer CTAs (hand-back, partials) come after a tile's MMAs are issued, so the argument there holds here too
  const uint32_t turn_mine = bars.turn(cw), turn_other = bars.turn(cw ^ 1);
  uint32_t tphase = 0;
  int stage = 0, it = 0;
  uint32_t phase = 0;
  float acc[64];

  for (int tile = t0 + cw * tstep; tile < p.num_tiles; tile += 2 * tstep, ++it) {
    const TileCoord tc = tile_coord(p, tile);
    if (lead) {
      bulk_wait_group_read0();           // the previous tile's store has left the output tile / receive buffer
      if (it > 0)
        for (int s = 0; s < C; ++s)
          if (s != rank) mbar_arrive_cluster(mapa_shared(bar_free, (uint32_t)s));
      mbar_expect_tx(bar_rfull, recv_bytes);
    }
    const int s = stage;
    mbar_wait_mma(bars.full(cw, s), phase);
    if (++stage == p.ring) { stage = 0; phase ^= 1u; }
    if (tile >= tstep) { mbar_wait_mma(turn_mine, tphase); tphase ^= 1u; }
    const uint32_t x16 = gmma_addr16(stage0 + (uint32_t)s * p.stage_bytes);
    wgmma_fence();
    halo_pxn_mmas(acc, x16, w16, btb16, 1, 0, 4);   // the rank's one chunk is resident: [tap][1]
    wgmma_commit();
    __syncwarp();
    if (lane == 0) mbar_arrive(turn_other);   // pass the turn
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(bars.empty(cw, s));

    if (!own) {
      // the owner has handed back the buffer its previous tile's partials went to
      if (it > 0) mbar_wait_cluster(bar_free, (uint32_t)(it - 1) & 1u);
#pragma unroll
      for (int j = 0; j < 16; ++j)
        st_async_v4(peer_buf + (uint32_t)j * 512u, make_float4(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]),
                    peer_bar);
    } else {
      mbar_wait_cluster(bar_rfull, (uint32_t)it & 1u);
      const uint32_t lq_off = (uint32_t)((q - rank * wpr) * 16) * 512u + (uint32_t)lane * 16u;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float4 mine = make_float4(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]);
        float4 sum = mine;
#pragma unroll
        for (int src = 0; src < 4; ++src) {
          if (src >= C) break;
          const int slot = src < rank ? src : src - 1;
          const float4 v = src == rank ? mine
                                       : ld_shared_v4(epi_s + (uint32_t)(slot * wpr * 16) * 512u + lq_off + (uint32_t)j * 512u);
          if (src == 0) sum = v;
          else { sum.x += v.x; sum.y += v.y; sum.z += v.z; sum.w += v.w; }
        }
        acc[4 * j] = sum.x; acc[4 * j + 1] = sum.y; acc[4 * j + 2] = sum.z; acc[4 * j + 3] = sum.w;
      }
    }
    named_bar_sync(bar_id, 128);         // the receive buffer is read: the output tile may overwrite it
    if (own) {
      const float b0 = bias_s[tc.nb * 64 + 16 * q + (lane >> 2)], b1 = bias_s[tc.nb * 64 + 16 * q + (lane >> 2) + 8];
      if (POOL) pxn_store_tile_pool2(acc, epi_s, sb, mat_off, b0, b1, d.act);
      else pxn_store_tile(acc, epi_s, sb, mat_off, b0, b1, d.act, /*residual=*/false);
      fence_proxy_async_smem();
    }
    named_bar_sync(bar_id, 128);
    if (lead) {
      if (POOL) tma_store_4d(&maps.m[2], epi_s, tc.nb * 64 + rank * sc, tc.x0 >> 1, tc.y0 >> 1, tc.n);
      else tma_store_4d(&maps.m[2], epi_s, tc.nb * 64 + rank * sc, tc.x0, tc.y0, tc.n);
      bulk_commit_group();
    }
  }
  if (lead) bulk_wait_group0();
}

// One consumer warpgroup of the forward stride-2 transposed conv (17x9 halo box, origin 0), pixels on N: for
// each of its tiles and each output parity a = (py, px), acc[64 cout][128 px] = convT_pxn_mmas(a), then
// bias / act -> fp16 -> stmatrix into one of the consumer's two 16 KB output tiles -> one TMA store of the
// parity's 16x8 output pixels (2*(y0+ty) + py, 2*(x0+tx) + px) through the 5-D output map (maps.m[2]).  The
// tiles alternate by parity, so parity a's store drains while parity a + 1 is computed.
__device__ __forceinline__ void consumer_convT_pxn(const TgMaps& maps, const KParams& p, uint32_t base,
                                                   const float* bias_s, int cw) {
  const tg_conv_desc& d = p.d;
  const int r = threadIdx.x - 128 * (1 + cw);
  const int q = r >> 5, lane = threadIdx.x & 31;
  const ConvBars bars{base};
  const uint32_t stage0 = base + p.off_stage + (uint32_t)(cw * p.ring) * p.stage_bytes;
  const uint32_t out0 = base + p.off_scratch + (uint32_t)cw * 2u * kTapABytes;
  const uint32_t w16 = gmma_addr16(base + p.off_b);
  const int bar_id = 1 + cw;
  const uint32_t mat_off = pxn_mat_off(lane, q, 128u, /*swizzled=*/true, /*pool=*/false);
  int stage = 0;
  uint32_t phase = 0;
  float acc[64];

  for (int tile = blockIdx.x + cw * (int)gridDim.x; tile < p.num_tiles; tile += 2 * (int)gridDim.x) {
    const TileCoord tc = tile_coord(p, tile);
    const float b0 = bias_s[tc.nb * 64 + 16 * q + (lane >> 2)], b1 = bias_s[tc.nb * 64 + 16 * q + (lane >> 2) + 8];
    const int s = stage;
    mbar_wait_mma(bars.full(cw, s), phase);
    if (++stage == p.ring) { stage = 0; phase ^= 1u; }
    const uint32_t x16 = gmma_addr16(stage0 + (uint32_t)s * p.stage_bytes);
#pragma unroll 1
    for (int a = 0; a < 4; ++a) {
      wgmma_fence();
      convT_pxn_mmas(acc, x16, w16, a);
      wgmma_commit();
      // the output tile of this parity was last read by the store before the previous one
      if (r == 0) bulk_wait_group_read1();
      named_bar_sync(bar_id, 128);
      wgmma_wait<0>();
      if (a == 3) { __syncwarp(); if (lane == 0) mbar_arrive(bars.empty(cw, s)); }
      const uint32_t out_s = out0 + (uint32_t)(a & 1) * kTapABytes;
      pxn_store_tile(acc, out_s, 128u, mat_off, b0, b1, d.act, /*residual=*/false);
      fence_proxy_async_smem();
      named_bar_sync(bar_id, 128);
      if (r == 0) {
        tma_store_5d(&maps.m[2], out_s, (a & 1) * d.cout + tc.nb * 64, tc.x0, a >> 1, tc.y0, tc.n);
        bulk_commit_group();
      }
    }
  }
  if (r == 0) bulk_wait_group0();
}

// ------------------------------------------------------------------ the kernel
// BWD = data-gradient instantiation: epilogue y = (acc + bias [+ residual]) * act'(mask)  (TG_ACT_DRELU /
// TG_ACT_DLRELU02; TG_ACT_NONE = no derivative).
// POOL = TG_EPI_NHWC_F16_POOL2 instantiation: 2x2 max over the tile's pixels (tap mode: by warp shuffles,
// one store per 2x2 block; halo mode: in registers, one TMA store of the pooled tile).
template <int KIND, int MODE, bool BWD = false, bool POOL = false>
__global__ void __launch_bounds__(conv_threads<KIND, MODE, BWD>(), 1)
conv_wgmma_kernel(const __grid_constant__ TgMaps maps, const KParams p) {
  constexpr int kThreads = conv_threads<KIND, MODE, BWD>();
  constexpr int kConsumers = conv_consumers<KIND, MODE, BWD>();
  constexpr bool kSharedRing = kConsumers == 3;   // one ring, filled in tile order (else one ring per consumer)
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;   // 128B swizzle atoms need 1024B alignment
  uint8_t* sm = smem_raw + (base - raw);
  constexpr int BN = MODE == MODE_TAPN ? TG_TAPN_ROWS : 64;
  constexpr int NF = BN / 2;                      // accumulator registers per m64 half

  const int warp = __shfl_sync(0xFFFFFFFFu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const tg_conv_desc& d = p.d;

  const ConvBars bars{base};
  const uint32_t bar_b = bars.weights();
  float* bias_s = reinterpret_cast<float*>(sm + 1024);
  static_assert(!(KIND == TG_CONV_3X3_S2 && MODE != MODE_TAP), "the stride-2 conv runs in tap mode only");
  constexpr bool kPxN = pixels_on_n<KIND, MODE, BWD>();
  constexpr bool kSplitK = MODE == MODE_SPLITK;
  static_assert(!kSplitK || (KIND == TG_CONV_3X3 && !BWD), "split-K: forward conv3x3 only");

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&maps.m[0]);
    if (KIND == TG_CONV_3X3_S2) { tma_prefetch_desc(&maps.m[1]); tma_prefetch_desc(&maps.m[2]); tma_prefetch_desc(&maps.m[3]); }
    if (kPxN) { tma_prefetch_desc(&maps.m[1]); tma_prefetch_desc(&maps.m[2]); }
    if (kSplitK) tma_prefetch_desc(&maps.m[2]);
  }
  if (warp == 1 && lane == 0) {
    mbar_init(bar_b, 1);
    for (int c = 0; c < (kSharedRing ? 1 : 2); ++c)
      for (int k = 0; k < kMaxRing; ++k) {
        mbar_init(bars.full(c, k), 1);
        mbar_init(bars.empty(c, k), 4);    // one arrival per warp of the consumer that read the stage
      }
    for (int c = 0; c < kConsumers; ++c) {
      mbar_init(bars.res(c), 1);
      if (kSplitK) {
        mbar_init(bars.recv(c), 1);               // the owner's expect_tx; the bytes come from the peers
        mbar_init(bars.handback(c), p.chunks - 1);    // one hand-back per peer
      }
      if (kSplitK || kConsumers == 3) mbar_init(bars.turn(c), 4);   // one arrival per warp of the previous consumer
    }
    fence_barrier_init();
  }
  // split-K: the peers' barriers must be initialised before any remote arrive or st.async reaches them
  if constexpr (kSplitK) cluster_sync();
  else __syncthreads();

  const uint32_t smem_b = base + p.off_b;
  const uint32_t smem_stage0 = base + p.off_stage;
  const unsigned char* wglob = reinterpret_cast<const unsigned char*>(d.weights);
  const int n_tiles_w = (MODE == MODE_TAPN ? 1 : 9) * (kSplitK ? 1 : p.chunks);
  // tile schedule: CTA i of the grid, or cluster i of the grid for split-K (all CTAs of a cluster take the
  // same tiles; CTA rank r of the cluster works on K chunk r)
  const int sched0 = kSplitK ? (int)cluster_id_x() : (int)blockIdx.x;
  const int sched_step = kSplitK ? (int)cluster_count_x() : (int)gridDim.x;
  const int k_rank = kSplitK ? (int)cluster_ctarank() : 0;

  // Resident weights do not depend on the previous kernel (static during graph replay; the eager path
  // separates tg_pack_* from the conv by a bias copy): start their load, then join the
  // programmatic-dependent-launch wait.  The previous kernel's OUTPUT is only read after tg_pdl_wait().
  if (warp == 0 && lane == 0 && p.b_resident) {
    // fixed per CTA: the number of CTAs (clusters for split-K) and num_tiles are multiples of n_split
    const uint32_t nb = (uint32_t)tile_coord(p, sched0).nb;
    mbar_expect_tx(bar_b, (uint32_t)n_tiles_w * p.b_stage_bytes);
    for (int t = 0; t < n_tiles_w; ++t) {
      const int src = kSplitK ? t * p.chunks + k_rank : t;   // split-K: the 9 taps of chunk k_rank
      bulk_load(smem_b + t * p.b_stage_bytes, wglob + (size_t)src * p.b_tile_bytes + (size_t)nb * p.b_stage_bytes,
                p.b_stage_bytes, bar_b);
    }
  }
  tg_pdl_wait();
  tg_pdl_trigger();
  // Only the consumer warpgroups read the bias.  They load it among themselves, so the producer issues its
  // first TMA loads right after the wait, and their latency overlaps the bias load's.
  if (warp >= 4) {
    for (int i = threadIdx.x - 128; i < d.cout; i += kThreads - 128) bias_s[i] = d.bias[i];
    named_bar_sync(kBiasBar, kThreads - 128);
  }

  if (warp == 0) {
    // ============================================================ TMA producer
    if (lane == 0) {
      int stage[2] = {0, 0};
      uint32_t phase[2] = {0, 0};
      int it = 0;
      for (int tile = sched0; tile < p.num_tiles; tile += sched_step, ++it) {
        const int cw = kSharedRing ? 0 : it & 1;   // the ring the tile goes to
        const TileCoord tc = tile_coord(p, tile);
        const int n_loads = MODE == MODE_TAP ? 9 * p.chunks : kSplitK ? 1 : p.chunks;
        for (int l = 0; l < n_loads; ++l) {
          const uint32_t full = bars.full(cw, stage[cw]);
          mbar_wait_mma(bars.empty(cw, stage[cw]), phase[cw] ^ 1);
          const uint32_t sa = smem_stage0 + (uint32_t)(cw * p.ring + stage[cw]) * p.stage_bytes;
          if (MODE != MODE_TAP) {
            mbar_expect_tx(full, p.a_bytes);
            tma_load_4d(sa, &maps.m[0], full, (l + k_rank) * 64, tc.x0 + p.org_x, tc.y0 + p.org_y, tc.n);
          } else {
            const int g = l / p.chunks, c = l - g * p.chunks;
            const TgGroup gr = tg_group(KIND, g);
            mbar_expect_tx(full, p.a_bytes + (p.b_resident ? 0u : p.b_stage_bytes));
            tma_load_4d(sa, &maps.m[KIND == TG_CONV_3X3_S2 ? tg_s2_plane(g) : 0], full, c * 64,
                        tc.x0 + gr.dx, tc.y0 + gr.dy, tc.n);
            if (!p.b_resident)
              bulk_load(sa + kTapABytes,
                        wglob + (size_t)(g * p.chunks + c) * p.b_tile_bytes + (size_t)tc.nb * p.b_stage_bytes,
                        p.b_stage_bytes, full);
          }
          if (++stage[cw] == p.ring) { stage[cw] = 0; phase[cw] ^= 1u; }
        }
      }
    }
  } else if (kSplitK) {
    // ============================================================ consumers, split-K over the cluster
    if (warp >= 4) {
      mbar_wait_mma(bar_b, 0);
      consumer_splitk<POOL>(maps, p, base, bias_s, (warp - 4) >> 2);
    }
  } else if (kPxN) {
    // ============================================================ consumers, pixels on N
    if (warp >= 4) {
      if (p.b_resident) mbar_wait_mma(bar_b, 0);
      if constexpr (KIND == TG_CONVT_3X3_S2) consumer_convT_pxn(maps, p, base, bias_s, (warp - 4) >> 2);
      else consumer_halo_pxn<POOL>(maps, p, base, bias_s, (warp - 4) >> 2);
    }
  } else if (warp >= 4) {
    // ============================================================ consumers
    const int cw = (warp - 4) >> 2;
    const int r = threadIdx.x - 128 * (1 + cw);        // 0..127: tile row in the epilogue
    const int q = r >> 5;                              // warp of the warpgroup
    float* S = reinterpret_cast<float*>(sm + p.off_scratch + (uint32_t)cw * scratch_bytes(MODE));
    if (p.b_resident) mbar_wait_mma(bar_b, 0);

    constexpr int kBoxW = (KIND == TG_CONV_3X3) ? TW + 2 : TW + 1;
    constexpr int kOrg = (KIND == TG_CONV_3X3) ? -1 : 0;
    const uint32_t a_sbo = (MODE == MODE_HALO ? (uint32_t)kBoxW : (uint32_t)TW) * 128u;
    const uint64_t a_hi = gmma_desc_hi(a_sbo), b_hi = gmma_desc_hi(1024u);
    const uint32_t half16 = (8u * a_sbo) >> 4;         // tile rows 8..15 = the second m64 half
    const uint32_t btb16 = p.b_stage_bytes >> 4;
    const uint32_t smem_b16 = gmma_addr16(smem_b);
    int stage = 0;
    uint32_t phase = 0;
    int pend = -1;                                     // stage whose MMAs may still be reading it

    float acc[2][NF];
    auto mma_group = [&](uint32_t a16, uint32_t b16, bool first) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (k < p.ksteps) {
          const uint32_t sc = (first && k == 0) ? 0u : 1u;
          wgmma_k16<NF>(acc[0], a_hi | (uint64_t)(a16 + 2u * k), b_hi | (uint64_t)(b16 + 2u * k), sc);
          wgmma_k16<NF>(acc[1], a_hi | (uint64_t)(a16 + half16 + 2u * k), b_hi | (uint64_t)(b16 + 2u * k), sc);
        }
      }
    };
    auto release = [&](int s) {
      __syncwarp();
      if (lane == 0) mbar_arrive(bars.empty(cw, s));
    };
    auto next_stage = [&]() -> int {   // wait for the next stage of this consumer's ring; returns its index
      const int s = stage;
      mbar_wait_mma(bars.full(cw, s), phase);
      if (++stage == p.ring) { stage = 0; phase ^= 1u; }
      return s;
    };
    auto stage_addr = [&](int s) { return smem_stage0 + (uint32_t)(cw * p.ring + s) * p.stage_bytes; };
    // accumulators -> S (fp32, row-major [128][stride]); the caller synchronises the warpgroup around it
    auto stash = [&]() {
      constexpr uint32_t ST = stage_stride(MODE);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int i = 0; i < NF; i += 2) {
          const int row = h * 64 + q * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
          const int col = 8 * (i >> 2) + 2 * (lane & 3);
          *reinterpret_cast<float2*>(S + (size_t)row * ST + col) = make_float2(acc[h][i], acc[h][i + 1]);
        }
      }
    };
    const int bar_id = 1 + cw;

    int it = cw;
    for (int tile = blockIdx.x + cw * (int)gridDim.x; tile < p.num_tiles; tile += 2 * (int)gridDim.x, it += 2) {
      const TileCoord tc = tile_coord(p, tile);
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < NF; ++i) acc[h][i] = 0.f;

      if (MODE == MODE_TAPN) {
        // D[pos][tap*4+co] = x[pos] . W[tap][co]; out[p] = sum_taps D[p+off(tap)][tap]
        for (int c = 0; c < p.chunks; ++c) {
          const int s = next_stage();
          wgmma_fence();
          mma_group(gmma_addr16(stage_addr(s)), smem_b16 + (uint32_t)c * btb16, c == 0);
          wgmma_commit();
          wgmma_wait<1>();
          if (pend >= 0) release(pend);
          pend = s;
        }
        wgmma_wait<0>();
        release(pend);
        pend = -1;
        stash();
        named_bar_sync(bar_id, 128);
        const int ty = r >> 3, tx = r & 7;
        const int py = tc.y0 + ty - 1, px = tc.x0 + tx - 1;
        const bool inb = ty >= 1 && ty <= TH - 2 && tx >= 1 && tx <= TW - 2 && py < d.h && px < d.w;
        if (inb) {
          constexpr uint32_t ST = stage_stride(MODE_TAPN);
          float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int tap = 0; tap < 9; ++tap) {
            const float4 e = *reinterpret_cast<const float4*>(S + (size_t)(r + (tap / 3 - 1) * TW + (tap % 3 - 1)) * ST + tap * 4);
            a.x += e.x; a.y += e.y; a.z += e.z; a.w += e.w;
          }
          const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
          for (int ch = 0; ch < 4; ++ch) {
            if (d.epilogue == TG_EPI_FLOW_NCHW_F32) {
              tg_epi_flow(d, tc.n, py, px, d.h, d.w, ch, av[ch]);
            } else {
              tg_epi_out(d, tc.n, py, px, d.h, d.w, ch, av[ch]);
            }
          }
        }
        named_bar_sync(bar_id, 128);
      } else if (MODE == MODE_HALO) {
        for (int c = 0; c < p.chunks; ++c) {
          const int s = next_stage();
          const uint32_t sa16 = gmma_addr16(stage_addr(s));
          wgmma_fence();
#pragma unroll
          for (int g = 0; g < 9; ++g) {
            const TgGroup gr = tg_group(KIND, g);
            mma_group(sa16 + (uint32_t)((gr.dy - kOrg) * kBoxW + (gr.dx - kOrg)) * 8u,
                      smem_b16 + (uint32_t)(g * p.chunks + c) * btb16, g == 0 && c == 0);
          }
          wgmma_commit();
          wgmma_wait<1>();
          if (pend >= 0) release(pend);
          pend = s;
        }
        wgmma_wait<0>();
        release(pend);
        pend = -1;
        stash();
        named_bar_sync(bar_id, 128);
        epilogue_nhwc<KIND, BWD, POOL>(p, tc, r, lane, 0, S, bias_s);
        named_bar_sync(bar_id, 128);
      } else {
        // MODE_TAP: one stage per (tap, chunk); the groups of one accumulator are consecutive
#pragma unroll 1
        for (int g = 0; g < 9; ++g) {
          const TgGroup gr = tg_group(KIND, g);
          const bool first_of_acc = g == 0 || tg_group(KIND, g - 1).acc != gr.acc;
          const bool last_of_acc = g == 8 || tg_group(KIND, g + 1).acc != gr.acc;
          for (int c = 0; c < p.chunks; ++c) {
            const int s = next_stage();
            const uint32_t sa = stage_addr(s);
            const uint32_t b16 = p.b_resident ? smem_b16 + (uint32_t)(g * p.chunks + c) * btb16
                                              : gmma_addr16(sa + kTapABytes);
            wgmma_fence();
            mma_group(gmma_addr16(sa), b16, first_of_acc && c == 0);
            wgmma_commit();
            wgmma_wait<1>();
            if (pend >= 0) release(pend);
            pend = s;
          }
          if (last_of_acc) {
            wgmma_wait<0>();
            release(pend);
            pend = -1;
            stash();
            named_bar_sync(bar_id, 128);
            epilogue_nhwc<KIND, BWD, POOL>(p, tc, r, lane, gr.acc, S, bias_s);
            named_bar_sync(bar_id, 128);
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int i = 0; i < NF; ++i) acc[h][i] = 0.f;
          }
        }
      }
    }
  }
  // split-K: no CTA leaves (and frees its shared memory) while a peer may still arrive on its barriers
  if constexpr (kSplitK) cluster_sync();
}

// ------------------------------------------------------------------ host side
// Output [n][2h][2w][c] of the transposed conv with input size h x w, as the 5-D tensor (2c, w, 2, h, n):
// element (px*c + ch, x, py, y, n) is output pixel (2y + py, 2x + px).  Parity (py, px) of the 16x8 input
// pixels at (y0, x0) is the box (64, 8, 1, 16, 1) at (px*c + nb*64, x0, py, y0, n); it clips at the right and
// bottom image edges, and never crosses into the next image.
int encode_convT_out(CUtensorMap* m, const void* ptr, int c, int w, int h, int n) {
  const size_t C = (size_t)c, W = (size_t)w;
  const cuuint64_t dims[5] = {2 * (cuuint64_t)c, (cuuint64_t)w, 2, (cuuint64_t)h, (cuuint64_t)n};
  const size_t strides[4] = {2 * C, 2 * W * C, 4 * W * C, 4 * (size_t)h * W * C};
  const cuuint32_t box[5] = {64, TW, 1, TH, 1};
  return encode_f16(m, ptr, 5, dims, strides, box);
}

template <int K, int M, bool B, bool P>
cudaError_t set_smem_attr() {
  return cudaFuncSetAttribute(conv_wgmma_kernel<K, M, B, P>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              (int)kSmemLimit);
}

template <int K, int M, bool B = false, bool P = false>
cudaError_t launch_conv(dim3 grid, cudaStream_t st, const TgMaps& maps, const KParams& p) {
  return tg_launch(conv_wgmma_kernel<K, M, B, P>, grid, dim3(conv_threads<K, M, B>()), kSmemLimit, st, maps, p);
}

// Clusters of `cluster` split-K CTAs (one per SM) that can be resident at once, per device; 0 if the query fails.
template <bool P>
int splitk_max_clusters(int cluster) {
  static int cache[64][5] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
  int& v = cache[dev][cluster];
  if (v == 0) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(cluster);
    cfg.blockDim = dim3(conv_threads<TG_CONV_3X3, MODE_SPLITK, false>());
    cfg.dynamicSmemBytes = kSmemLimit;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)cluster;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, conv_wgmma_kernel<TG_CONV_3X3, MODE_SPLITK, false, P>, &cfg) != cudaSuccess) {
      (void)cudaGetLastError();
      n = 0;
    }
    v = n;
  }
  return v;
}

}  // namespace

extern "C" {

int tg_debug_set_conv_timers(void* device_buffer) {
  TG_REQUIRE(device_buffer == nullptr, TG_E_UNSUPPORTED,
             "debug_set_conv_timers: the sm_90a kernels record no role timers");
  return TG_OK;
}

int tg_conv_validate(const tg_conv_desc* d, const char* who) {
  TG_REQUIRE(d != nullptr, TG_E_INVALID, "%s: null descriptor", who);
  TG_REQUIRE(d->x && d->weights && d->bias && d->y, TG_E_INVALID, "%s: null pointer", who);
  TG_REQUIRE(d->n > 0 && d->h > 0 && d->w > 0, TG_E_INVALID, "%s: bad size n=%d h=%d w=%d", who, d->n, d->h, d->w);
  TG_REQUIRE(d->kind == TG_CONV_3X3 || d->kind == TG_CONVT_3X3_S2 || d->kind == TG_CONV_3X3_S2, TG_E_INVALID,
             "%s: kind", who);
  TG_REQUIRE(d->act >= TG_ACT_NONE && d->act <= TG_ACT_DLRELU02, TG_E_INVALID, "%s: act", who);
  TG_REQUIRE((d->act >= TG_ACT_DRELU) == (d->mask != nullptr), TG_E_INVALID,
             "%s: mask must be given exactly for TG_ACT_DRELU / TG_ACT_DLRELU02", who);
  TG_REQUIRE(!(d->act >= TG_ACT_DRELU && (d->epilogue != TG_EPI_NHWC_F16 || d->kind == TG_CONVT_3X3_S2)),
             TG_E_UNSUPPORTED, "%s: derivative epilogues need NHWC output and a conv3x3 / conv3x3s2 layer", who);
  TG_REQUIRE(!(d->kind == TG_CONV_3X3_S2 && d->epilogue != TG_EPI_NHWC_F16), TG_E_UNSUPPORTED,
             "%s: conv3x3s2 needs the NHWC epilogue", who);
  TG_REQUIRE(d->cin == 64 || d->cin == 128 || d->cin == 192 || d->cin == 256 || d->cin == 384 || d->cin == 512,
             TG_E_UNSUPPORTED, "%s: cin=%d (stored channels must be 64, 128, 192, 256, 384 or 512)", who, d->cin);
  if (d->epilogue == TG_EPI_NHWC_F16_POOL2)
    TG_REQUIRE(d->kind == TG_CONV_3X3 && d->residual == nullptr && d->act <= TG_ACT_LRELU02 && d->h >= 2 && d->w >= 2,
               TG_E_UNSUPPORTED, "%s: the pooled epilogue needs a conv3x3 without residual / derivative epilogue", who);
  if (d->epilogue == TG_EPI_NHWC_F16 || d->epilogue == TG_EPI_NHWC_F16_POOL2) {
    TG_REQUIRE(d->cout == 64 || d->cout == 128 || d->cout == 192 || d->cout == 256 || d->cout == 384 ||
                   d->cout == 512,
               TG_E_UNSUPPORTED, "%s: cout=%d (64, 128, 192, 256, 384 or 512 for the NHWC epilogue)", who, d->cout);
    TG_REQUIRE(!(d->residual && d->kind == TG_CONVT_3X3_S2), TG_E_UNSUPPORTED, "%s: residual with convT", who);
    TG_REQUIRE(!(d->kind == TG_CONVT_3X3_S2 && d->cout != 64), TG_E_UNSUPPORTED,
               "%s: convT needs cout == 64 (4 parity accumulators per tile)", who);
  } else if (d->epilogue == TG_EPI_FLOW_NCHW_F32 || d->epilogue == TG_EPI_OUT_NCHW_F32) {
    TG_REQUIRE(d->kind == TG_CONV_3X3 && d->cout == TG_TAPN_ROWS && d->cout_real >= 1 && d->cout_real <= 4,
               TG_E_UNSUPPORTED, "%s: NCHW epilogues need conv3x3, cout=48 (tap-major N), cout_real<=4", who);
    TG_REQUIRE(d->residual == nullptr, TG_E_UNSUPPORTED, "%s: residual with NCHW epilogue", who);
  } else {
    TG_REQUIRE(false, TG_E_INVALID, "%s: epilogue %d", who, d->epilogue);
  }
  return TG_OK;
}

int tg_conv_tcgen05(const tg_conv_desc* d, void* stream) {
  int rc = tg_conv_validate(d, "conv");
  if (rc != TG_OK) return rc;
  const int a_mode = d->a_mode & ~TG_AMODE_REVERSE;
  TG_REQUIRE(a_mode >= TG_AMODE_AUTO && a_mode <= TG_AMODE_TAP, TG_E_INVALID, "conv: a_mode");
  TG_REQUIRE(((uintptr_t)d->x & 15) == 0 && ((uintptr_t)d->weights & 15) == 0 && ((uintptr_t)d->y & 15) == 0,
             TG_E_INVALID, "conv: pointers must be 16-byte aligned");

  KParams p;
  p.d = *d;
  p.d.a_mode = a_mode;
  p.reverse = (d->a_mode & TG_AMODE_REVERSE) != 0;
  const bool tapn = d->epilogue == TG_EPI_FLOW_NCHW_F32 || d->epilogue == TG_EPI_OUT_NCHW_F32;
  const bool pool = d->epilogue == TG_EPI_NHWC_F16_POOL2;
  p.step_y = tapn ? kTapnStepY : TH;
  p.step_x = tapn ? kTapnStepX : TW;
  p.tiles_x = tg_ceil_div(d->w, p.step_x);
  p.tiles_y = tg_ceil_div(d->h, p.step_y);
  p.num_tiles = p.tiles_x * p.tiles_y * d->n;
  p.chunks = d->cin / 64;
  TG_REQUIRE(d->cin_real >= 0 && d->cin_real <= d->cin, TG_E_INVALID, "conv: cin_real=%d outside [0, cin=%d]",
             d->cin_real, d->cin);
  p.ksteps = (p.chunks == 1 && d->cin_real > 0) ? (d->cin_real + 15) / 16 : 4;
  p.n_acc = d->kind == TG_CONVT_3X3_S2 ? 4 : 1;
  p.b_tile_bytes = (uint32_t)d->cout * 128u;

  // Output channels beyond 64 are split over CTAs (N = 64 per CTA): cout/64 x more CTAs on the
  // low-resolution FNet layers, and each CTA only needs its own 64-row slice of every weight tile.
  p.n_split = (!tapn && d->cout > 64) ? d->cout / 64 : 1;
  p.bn = d->cout / p.n_split;
  p.b_stage_bytes = (uint32_t)p.bn * 128u;
  const bool bwd = d->act >= TG_ACT_DRELU || d->kind == TG_CONV_3X3_S2;
  const bool convT = d->kind == TG_CONVT_3X3_S2;
  // Forward 3x3 convs with 128 / 256 input channels (NHWC output, pooled or not) split K over a cluster of
  // cin/64 CTAs (MODE_SPLITK), each with one chunk's weights resident; TG_AMODE_TAP keeps the tap kernel.
  // consumer_splitk partitions the four 16-cout warps among the ranks, so 192 / 384 input channels (3 / 6 chunks)
  // stream their weights in tap mode.
  const bool splitk = a_mode == TG_AMODE_AUTO && d->kind == TG_CONV_3X3 && !bwd && !tapn &&
                      (p.chunks == 2 || p.chunks == 4) && d->residual == nullptr;
  // the bias follows the barriers: 1 KB holds 256 output channels, 384 and 512 take a second KB
  const uint32_t header = kHeaderBytes + (d->cout > 256 ? 1024u : 0u);
  const uint32_t b_total = (tapn ? 1u : 9u) * (splitk ? 1u : (uint32_t)p.chunks) * p.b_stage_bytes;   // resident slice per CTA
  const int hbox_w = d->kind != TG_CONVT_3X3_S2 ? TW + 2 : TW + 1;
  const int hbox_h = d->kind != TG_CONVT_3X3_S2 ? TH + 2 : TH + 1;
  const uint32_t halo_bytes = (uint32_t)hbox_w * hbox_h * 128u;
  const uint32_t halo_stage = (halo_bytes + 1023u) & ~1023u;
  const uint32_t scratch = 2u * scratch_bytes(tapn ? MODE_TAPN : MODE_TAP);
  const uint32_t fixed = 1024u /*align slack*/ + header + scratch;

  // every consumer needs at least one stage of its own
  const bool can_resident_halo = fixed + b_total + 2u * halo_stage <= kSmemLimit &&
                                 !(d->kind == TG_CONVT_3X3_S2 && p.chunks != 1);
  const bool can_resident_tap = fixed + b_total + 2u * kTapABytes <= kSmemLimit;
  int mode = a_mode;
  TG_REQUIRE(!(d->kind == TG_CONV_3X3_S2 && mode == TG_AMODE_HALO), TG_E_UNSUPPORTED,
             "conv: conv3x3s2 runs in tap mode (a stride-2 view is not a wgmma descriptor)");
  if (d->kind == TG_CONV_3X3_S2 || tapn) mode = TG_AMODE_TAP;   // thin heads run MODE_TAPN below
  if (mode == TG_AMODE_AUTO) mode = (splitk || can_resident_halo) ? TG_AMODE_HALO : TG_AMODE_TAP;
  TG_REQUIRE(!(mode == TG_AMODE_HALO && !splitk && !can_resident_halo), TG_E_UNSUPPORTED,
             "conv: halo mode needs the weights resident in smem (cin=%d cout=%d)", d->cin, d->cout);
  p.halo = mode == TG_AMODE_HALO;
  p.b_resident = p.halo ? 1 : (can_resident_tap ? 1 : 0);
  p.num_tiles *= p.n_split;
  TG_REQUIRE(p.bn == 64 || (tapn && p.bn == TG_TAPN_ROWS), TG_E_UNSUPPORTED,
             "conv: per-CTA N must be 64 (48 for the thin heads)");
  TG_REQUIRE(!tapn || p.b_resident, TG_E_UNSUPPORTED, "conv: thin head weights must fit in smem");
  if (tapn) {
    p.box_w = TW; p.box_h = TH; p.org_x = -1; p.org_y = -1;
    p.a_bytes = kTapABytes;
    p.stage_bytes = kTapABytes;
  } else if (p.halo) {
    p.box_w = hbox_w; p.box_h = hbox_h;
    p.org_x = d->kind == TG_CONV_3X3 ? -1 : 0;
    p.org_y = p.org_x;
    p.a_bytes = halo_bytes;
    p.stage_bytes = halo_stage;
  } else {
    p.box_w = TW; p.box_h = TH; p.org_x = 0; p.org_y = 0;
    p.a_bytes = kTapABytes;
    p.stage_bytes = kTapABytes + (p.b_resident ? 0u : p.b_stage_bytes);
  }
  // the consumers' epilogue tiles on the pixels-on-N path: one fp16 output / residual tile (16 KB) each, two
  // per consumer for the transposed conv (alternating parities), one 4 KB pooled tile each with the pool;
  // fp32 accumulator staging otherwise
  // Split-K: a receive buffer per consumer for the peers' partials of the couts this CTA owns ((C - 1) x 4/C
  // warps x 8 KB: 16 KB for C = 2, 24 KB for C = 4); the consumer's output slice tile overlaps it.
  // The forward pixels-on-N conv3x3 has three consumers, one output tile each, and one ring shared in tile order: the
  // ring must be at least consumers + 1 = 4 stages deep (consumer_halo_pxn), which the 72 KB weight slice of a cin = 64
  // layer always leaves room for: 1024 + 2048 + 73,728 + 4 x 23,552 + 3 x 16,384 = 220,160 B.
  const bool pxn = p.halo && !bwd && !tapn && !splitk;
  const bool three = pxn && !convT;
  p.epi_bytes = splitk ? (uint32_t)((p.chunks - 1) * (4 / p.chunks)) * 8192u : 0u;
  const uint32_t epi_tiles = splitk  ? 2u * p.epi_bytes
                             : !pxn  ? scratch
                             : convT ? 4u * kTapABytes
                                     : 3u * (pool ? kPoolTileBytes : kTapABytes);
  const uint32_t avail = kSmemLimit - 1024u - header - epi_tiles - (p.b_resident ? b_total : 0u);
  const int rings = three ? 1 : 2;
  int ring = (int)(avail / p.stage_bytes) / rings;
  if (ring > kMaxRing) ring = kMaxRing;
  TG_REQUIRE(ring >= 1, TG_E_UNSUPPORTED, "conv: shared memory budget (cin=%d cout=%d)", d->cin, d->cout);
  TG_REQUIRE(!three || (ring >= 4 && p.chunks == 1), TG_E_UNSUPPORTED,
             "conv: the three-consumer halo conv needs cin = 64 and 4 halo stages (cin=%d cout=%d: %d)", d->cin,
             d->cout, ring);
  p.ring = ring;
  p.off_b = header;
  p.off_stage = header + (p.b_resident ? b_total : 0u);
  p.off_scratch = p.off_stage + (uint32_t)(rings * ring) * p.stage_bytes;   // ring c: stages [c*ring, (c+1)*ring)
  const uint32_t smem_bytes = 1024u + p.off_scratch + epi_tiles;
  TG_REQUIRE(smem_bytes <= kSmemLimit, TG_E_UNSUPPORTED, "conv: smem %u > limit", smem_bytes);

  // tensor maps
  TgMaps map_a;
  if (d->kind != TG_CONV_3X3_S2) {
    rc = encode_nhwc(&map_a.m[0], d->x, d->cin, d->w, d->h, d->n, (size_t)d->cin, (size_t)d->w * d->cin,
                     (size_t)d->h * d->w * d->cin, 64, p.box_w, p.box_h);
    if (rc != TG_OK) return rc;
    map_a.m[1] = map_a.m[2] = map_a.m[3] = map_a.m[0];
    const size_t C = (size_t)d->cout;
    if (splitk) {
      // [2] = the output (pooled or not), one box per tile, N slice and rank: 64/C channels x 16x8 px (8x4 pooled),
      // unswizzled (the rank's slice tile is dense, 2 * 64/C bytes per pixel)
      const int sc = 64 / p.chunks;
      const int ow = pool ? d->w / 2 : d->w, oh = pool ? d->h / 2 : d->h;
      rc = encode_nhwc(&map_a.m[2], d->y, d->cout, ow, oh, d->n, C, (size_t)ow * C, (size_t)oh * ow * C, sc,
                       pool ? TW / 2 : TW, pool ? TH / 2 : TH, /*swizzle=*/false);
      if (rc != TG_OK) return rc;
    } else if (pxn && convT) {
      rc = encode_convT_out(&map_a.m[2], d->y, d->cout, d->w, d->h, d->n);
      if (rc != TG_OK) return rc;
    } else if (pxn && pool) {
      // [2] = the pooled output [n][h/2][w/2][cout], one 8x4 px x 64 ch box per tile and N slice
      const int pw = d->w / 2, ph = d->h / 2;
      rc = encode_nhwc(&map_a.m[2], d->y, d->cout, pw, ph, d->n, C, (size_t)pw * C, (size_t)ph * pw * C, 64,
                       TW / 2, TH / 2);
      if (rc != TG_OK) return rc;
    } else if (pxn) {
      // [1] = residual, [2] = output: NHWC [n][h][w][cout], one 16x8 px x 64 ch box per tile and N slice
      if (d->residual) {
        TG_REQUIRE(((uintptr_t)d->residual & 15) == 0, TG_E_INVALID, "conv: residual must be 16-byte aligned");
        rc = encode_nhwc(&map_a.m[1], d->residual, d->cout, d->w, d->h, d->n, C, (size_t)d->w * C,
                         (size_t)d->h * d->w * C, 64, TW, TH);
        if (rc != TG_OK) return rc;
      }
      rc = encode_nhwc(&map_a.m[2], d->y, d->cout, d->w, d->h, d->n, C, (size_t)d->w * C,
                       (size_t)d->h * d->w * C, 64, TW, TH);
      if (rc != TG_OK) return rc;
    }
  } else {
    // x [n,2h,2w,cin]: parity plane (py,px) = pixels (2i+py, 2j+px), each an [n,h,w,cin] strided view
    const size_t W2 = (size_t)2 * d->w, C = (size_t)d->cin;
    for (int pl = 0; pl < 4; ++pl) {
      const __half* base = reinterpret_cast<const __half*>(d->x) + ((size_t)(pl >> 1) * W2 + (pl & 1)) * C;
      rc = encode_nhwc(&map_a.m[pl], base, d->cin, d->w, d->h, d->n, 2 * C, 2 * W2 * C,
                       (size_t)4 * d->h * d->w * C, 64, p.box_w, p.box_h);
      if (rc != TG_OK) return rc;
    }
  }

  static TgPerDeviceOnce attr_once;
  const cudaError_t attr_err = attr_once.run([] {
    const cudaError_t errs[] = {
        set_smem_attr<TG_CONV_3X3, MODE_HALO, false, false>(), set_smem_attr<TG_CONV_3X3, MODE_TAP, false, false>(),
        set_smem_attr<TG_CONV_3X3, MODE_TAPN, false, false>(), set_smem_attr<TG_CONVT_3X3_S2, MODE_HALO, false, false>(),
        set_smem_attr<TG_CONVT_3X3_S2, MODE_TAP, false, false>(), set_smem_attr<TG_CONV_3X3, MODE_HALO, false, true>(),
        set_smem_attr<TG_CONV_3X3, MODE_TAP, false, true>(), set_smem_attr<TG_CONV_3X3, MODE_HALO, true, false>(),
        set_smem_attr<TG_CONV_3X3, MODE_TAP, true, false>(), set_smem_attr<TG_CONV_3X3_S2, MODE_TAP, true, false>(),
        set_smem_attr<TG_CONV_3X3, MODE_SPLITK, false, false>(), set_smem_attr<TG_CONV_3X3, MODE_SPLITK, false, true>()};
    for (cudaError_t e : errs)
      if (e != cudaSuccess) return e;
    return cudaSuccess;
  });
  TG_REQUIRE(attr_err == cudaSuccess, (int)attr_err, "conv: cudaFuncSetAttribute: %s",
             cudaGetErrorString(attr_err));

  int sms = 0;
  rc = tg_device_sm_count(&sms);
  if (rc != TG_OK) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t lerr = cudaSuccess;
  if (splitk) {
    // clusters of C = cin/64 CTAs, as many as can be resident (max_ctas: at most that many CTAs); every
    // cluster keeps one fixed N slice, so the cluster count is a multiple of n_split
    const int C = p.chunks;
    const int resident = pool ? splitk_max_clusters<true>(C) : splitk_max_clusters<false>(C);
    TG_REQUIRE(resident > 0, TG_E_DRIVER, "conv: cudaOccupancyMaxActiveClusters found no room for a %d-CTA cluster", C);
    int ncl = d->max_ctas > 0 ? d->max_ctas / C : resident;
    if (ncl > p.num_tiles) ncl = p.num_tiles;
    ncl -= ncl % p.n_split;
    if (ncl < p.n_split) ncl = p.n_split;
    const dim3 g(ncl * C), b(conv_threads<TG_CONV_3X3, MODE_SPLITK, false>());
    lerr = pool ? tg_launch_cluster(conv_wgmma_kernel<TG_CONV_3X3, MODE_SPLITK, false, true>, g, b, kSmemLimit, st, C,
                                    map_a, p)
                : tg_launch_cluster(conv_wgmma_kernel<TG_CONV_3X3, MODE_SPLITK, false, false>, g, b, kSmemLimit, st, C,
                                    map_a, p);
    TG_REQUIRE(lerr == cudaSuccess, (int)lerr, "conv: launch failed: %s", cudaGetErrorString(lerr));
    TG_CUDA_LAUNCH_CHECK("conv");
    return TG_OK;
  }
  int grid = d->max_ctas > 0 ? d->max_ctas : sms;
  if (grid > p.num_tiles) grid = p.num_tiles;
  grid -= grid % p.n_split;             // every CTA keeps one fixed N slice (resident weights)
  if (grid < p.n_split) grid = p.n_split;
  const dim3 g(grid);
  if (pool) {
    lerr = p.halo ? launch_conv<TG_CONV_3X3, MODE_HALO, false, true>(g, st, map_a, p)
                  : launch_conv<TG_CONV_3X3, MODE_TAP, false, true>(g, st, map_a, p);
  } else if (bwd) {
    if (d->kind == TG_CONV_3X3_S2)
      lerr = launch_conv<TG_CONV_3X3_S2, MODE_TAP, true>(g, st, map_a, p);
    else if (p.halo)
      lerr = launch_conv<TG_CONV_3X3, MODE_HALO, true>(g, st, map_a, p);
    else
      lerr = launch_conv<TG_CONV_3X3, MODE_TAP, true>(g, st, map_a, p);
  } else if (tapn) {
    lerr = launch_conv<TG_CONV_3X3, MODE_TAPN>(g, st, map_a, p);
  } else if (d->kind == TG_CONV_3X3) {
    lerr = p.halo ? launch_conv<TG_CONV_3X3, MODE_HALO>(g, st, map_a, p)
                  : launch_conv<TG_CONV_3X3, MODE_TAP>(g, st, map_a, p);
  } else {
    lerr = p.halo ? launch_conv<TG_CONVT_3X3_S2, MODE_HALO>(g, st, map_a, p)
                  : launch_conv<TG_CONVT_3X3_S2, MODE_TAP>(g, st, map_a, p);
  }
  TG_REQUIRE(lerr == cudaSuccess, (int)lerr, "conv: launch failed: %s", cudaGetErrorString(lerr));
  TG_CUDA_LAUNCH_CHECK("conv");
  return TG_OK;
}


}  // extern "C"
