// 3x3 convolution / stride-2 transposed convolution / stride-2 convolution as a persistent,
// warp-specialised wgmma implicit GEMM for sm_90a (H100).
//
//   M tile  = 128 output pixels = a 16x8 patch of one image (row m <-> pixel (m>>3, m&7)), issued as
//             two m64 wgmmas (tile rows 0-7 and 8-15)
//   N       = 64 output channels per CTA (layers with 128 / 256 are split over 2 / 4 CTAs); 48 for
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
//             CTA's tiles alternately, each with its own ring of smem stages: wgmma -> accumulators
//             staged to a per-consumer fp32 smem tile -> one thread per pixel applies bias / act /
//             residual (or the derivative, pool, pixel-shuffle and thin-head epilogues) and writes
//             the pixel's 128-byte NHWC row.  On the forward halo and split-K paths the consumers take
//             turns issuing their MMAs, so that one's epilogue runs under the other's MMAs.
//             The tap-mode transposed conv keeps 4 parity accumulators (1/2/2/4 taps), computed and
//             stored one after the other; each stores its pixel's output of that parity (pixel shuffle).
//
// The forward halo conv and transposed conv with NHWC output (the SRNet body, the first SRNet
// transposed conv and the FNet halo layers, pooled or not; see consumer_halo_pxn / consumer_convT_pxn)
// swap the GEMM's roles: M = the 64 output channels (the packed weight tile is the K-major A operand),
// N = the tile's 128 pixels (the halo view is the K-major B operand, 16 core groups of 8 pixels), so
// each (tap, k-step) is ONE m64n128k16 that reads 6 KB of smem instead of two m64n64k16 that read 8 KB.
// The epilogue works from registers: bias / act / residual -> fp16 -> stmatrix into a 16 KB tile in the
// TMA box image -> one TMA tensor store per tile (per parity for the transposed conv, into a 5-D view
// of its output); the residual arrives in that tile by one TMA load issued before the tile's MMAs.  With
// the pool, the 2x2 max is taken in registers and a 4 KB pooled tile is stored.  Without the fp32
// staging tiles each consumer's ring holds two halo stages or more.
#include <cuda.h>

#include <cstdlib>
#include <mutex>

#include "tg_common.cuh"
#include "tg_epilogue.cuh"
#include "tg_wgmma.cuh"

namespace {

constexpr int TH = 16, TW = 8;
constexpr int kThreads = 384;             // producer warpgroup + 2 consumer warpgroups
constexpr int kMaxRing = 4;               // smem stages per consumer ring
constexpr int kBiasBar = 3;               // named barrier of both consumer warpgroups (1 + cw: one consumer's)
constexpr uint32_t kHeaderBytes = 2048;   // barriers (first 1 KB) + bias (second 1 KB)
constexpr uint32_t kTapABytes = TH * TW * 128;  // 16 KB
constexpr uint32_t kPoolTileBytes = kTapABytes / 4;   // the pooled 8x4 px x 64 ch output tile
constexpr uint32_t kSmemLimit = 232448;   // 227 KB opt-in limit per CTA
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
  int ring;                        // smem stages per consumer
  int ksteps;                      // wgmma k-steps (16 channels) per 64-channel chunk that can hold non-zero input (1..4)
  int n_split, bn;                 // output channels are split over n_split CTAs of bn columns
  uint32_t stage_bytes, a_bytes, b_tile_bytes, b_stage_bytes;
  uint32_t off_b, off_stage, off_scratch;   // off_scratch: the consumers' fp32 staging or fp16 output tiles
  uint32_t epi_bytes;              // MODE_SPLITK: per-consumer receive buffer (the output tile overlaps it)
};

// The forward halo conv / transposed conv with NHWC output (pooled or not) puts the roles of the GEMM the
// other way round: D[cout][pixel] = W . X^T, the 64 output channels on M and the tile's 128 pixels on N.
template <int KIND, int MODE, bool BWD>
__host__ __device__ constexpr bool pixels_on_n() {
  return (KIND == TG_CONV_3X3 || KIND == TG_CONVT_3X3_S2) && MODE == MODE_HALO && !BWD;
}

struct TileCoord { int n, y0, x0, nb; };
__device__ __forceinline__ TileCoord tile_coord(const KParams& p, int tile) {
  TileCoord t;
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
// One consumer warpgroup (cw) of the forward 3x3 halo conv, NHWC fp16 output: for each of its tiles
//   D[64 cout][128 px] = sum over (tap, chunk, k-step) of m64n128k16(A = resident weight tile, K-major,
//                        SBO 1024; B = the tap's shifted view of the halo stage, K-major, SBO = one box row)
// then an epilogue from registers into a 16 KB tile in the TMA box image (16x8 px x 64 ch, 128B swizzle)
// that one TMA tensor store writes out (clipped at the image edge).  The residual, if any, is TMA-loaded
// into the same tile before the tile's MMAs and overwritten in place.  Thread t of the warpgroup holds
// rows (couts) 16*(t/32) + (t%32)/4 + {0, 8} and pixel columns 8*j + 2*(t%4) + {0, 1}, j = 0..15.
// POOL (MaxPool2d(2, 2) folded in): the 2x2 block (tile rows 2i, 2i+1; columns 2*(t%4), +1) of a cout lies in
// four registers of one thread, so the pooled 8x4 px x 64 ch tile (4 KB) is formed without shuffles and
// stored through the pooled tensor's map; clipping at that map's edge is the floor pooling.
template <bool POOL>
__device__ __forceinline__ void consumer_halo_pxn(const TgMaps& maps, const KParams& p, uint32_t base,
                                                  const float* bias_s, int cw) {
  const tg_conv_desc& d = p.d;
  const int r = threadIdx.x - 128 * (1 + cw);
  const int q = r >> 5, lane = threadIdx.x & 31;
  const uint32_t bar_full = base + 8u * (cw * kMaxRing), bar_empty = base + 16 * kMaxRing + 8u * (cw * kMaxRing);
  const uint32_t bar_res = base + 32 * kMaxRing + 8 + 8u * cw;
  const uint32_t stage0 = base + p.off_stage + (uint32_t)(cw * p.ring) * p.stage_bytes;
  const uint32_t out_s = base + p.off_scratch + (uint32_t)cw * (POOL ? kPoolTileBytes : kTapABytes);
  constexpr uint32_t kBoxW = TW + 2;
  const uint64_t w_hi = gmma_desc_hi(1024u), x_hi = gmma_desc_hi(kBoxW * 128u);
  const uint32_t w16 = gmma_addr16(base + p.off_b), btb16 = p.b_stage_bytes >> 4;
  const bool has_res = !POOL && d.residual != nullptr;
  const int bar_id = 1 + cw;
  // Turns on the tensor pipe.  The CTA's tiles blockIdx.x + i * gridDim.x, i = 0, 1, 2, ..., go to consumer i & 1.
  // The owner of tile i > 0 issues its MMAs only after the other consumer has issued (and committed) tile i - 1:
  // it waits on turn[cw], on which the other consumer's four warps arrive after each of their commits.  The
  // tensor pipe then runs the two consumers' MMAs one tile after the other instead of sharing it, so one
  // consumer's epilogue runs under the other's MMAs rather than both epilogues leaving the pipe idle together.
  // No deadlock: every tile i > 0 has its tile i - 1 in the same CTA, and issuing tile i - 1 waits only for
  // tile i - 2's issue and for memory (the stage, the store drain), never for anything of tile i or later,
  // whatever the tile counts of the two consumers (1 / 0, or unequal).  Waits and arrivals on a barrier
  // alternate (an arrival on turn[c] needs the wait that preceded the arriving consumer's own issue), so a parity
  // wait is never more than one phase behind; the arrival after a consumer's last tile has no waiter and is harmless.
  const uint32_t turn_mine = base + 32 * kMaxRing + 56 + 8u * cw, turn_other = base + 32 * kMaxRing + 56 + 8u * (cw ^ 1);
  uint32_t tphase = 0;
  // stmatrix / ldmatrix: lane l addresses pixel row l%8 of 8x8 matrix m = l/8 = (tile row 2*jp + m/2,
  // 8-channel chunk 2*q + m%2); the swizzled offset of (pixel px, chunk) is px*128 + ((chunk ^ px%8) << 4).
  // POOL: matrix m = (pooled row pair 2*ip + m/2, chunk 2*q + m%2), its column 2*c + e = pooled pixel
  // (row 2*(2*ip + m/2) + e, column c), i.e. lane l addresses tile pixel 8*(m/2) + kk, kk = 4*(l%2) + (l%8)/2.
  const uint32_t kk = POOL ? 4u * (lane & 1) + ((lane & 7) >> 1) : (uint32_t)(lane & 7);
  const uint32_t mat_off = (uint32_t)(8 * ((lane >> 3) >> 1) + kk) * 128u +
                           ((uint32_t)((2 * q + ((lane >> 3) & 1)) ^ kk) << 4);
  int stage = 0;
  uint32_t phase = 0, rphase = 0;
  float acc[64];

  for (int tile = blockIdx.x + cw * (int)gridDim.x; tile < p.num_tiles; tile += 2 * (int)gridDim.x) {
    const TileCoord tc = tile_coord(p, tile);
    if (r == 0) {
      bulk_wait_group_read0();           // the previous tile's store has left the output tile
      if (has_res) {
        mbar_expect_tx(bar_res, kTapABytes);
        tma_load_4d(out_s, &maps.m[1], bar_res, tc.nb * 64, tc.x0, tc.y0, tc.n);
      }
    }
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    int pend = -1;                       // stage whose MMAs may still be reading it
    for (int c = 0; c < p.chunks; ++c) {
      const int s = stage;
      mbar_wait_mma(bar_full + 8 * s, phase);
      if (++stage == p.ring) { stage = 0; phase ^= 1u; }
      // take the turn only once the tile's first stage is here, so that it is never held while waiting on memory
      if (c == 0 && tile >= (int)gridDim.x) { mbar_wait_mma(turn_mine, tphase); tphase ^= 1u; }
      const uint32_t x16 = gmma_addr16(stage0 + (uint32_t)s * p.stage_bytes);
      wgmma_fence();
#pragma unroll
      for (int g = 0; g < 9; ++g) {
        const TgGroup gr = tg_group(TG_CONV_3X3, g);
        const uint32_t a16 = w16 + (uint32_t)(g * p.chunks + c) * btb16;
        const uint32_t b16 = x16 + (uint32_t)((gr.dy + 1) * (int)kBoxW + (gr.dx + 1)) * 8u;
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (k < p.ksteps)
            wgmma_n128(acc, w_hi | (uint64_t)(a16 + 2u * k), x_hi | (uint64_t)(b16 + 2u * k),
                       (g == 0 && c == 0 && k == 0) ? 0u : 1u);
      }
      wgmma_commit();
      if (c == p.chunks - 1) { __syncwarp(); if (lane == 0) mbar_arrive(turn_other); }   // pass the turn
      wgmma_wait<1>();
      if (pend >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(bar_empty + 8 * pend); }
      pend = s;
    }
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_empty + 8 * pend);

    // the output tile is free once thread 0 saw the previous store read it (it issued the residual load after)
    if (has_res) { mbar_wait_mma(bar_res, rphase); rphase ^= 1u; }
    else named_bar_sync(bar_id, 128);
    const float b0 = bias_s[tc.nb * 64 + 16 * q + (lane >> 2)], b1 = bias_s[tc.nb * 64 + 16 * q + (lane >> 2) + 8];
    if (POOL) {
#pragma unroll
      for (int ip = 0; ip < 2; ++ip) {
        uint32_t ov[4];
#pragma unroll
        for (int m = 0; m < 4; ++m) {
          const float bb = (m & 1) ? b1 : b0;
          __half v[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            // pooled row pr = tile rows 2*pr, 2*pr + 1; the same fp16 values the unpooled epilogue stores
            const int pr = 2 * (2 * ip + (m >> 1)) + e;
            const int i0 = 4 * (2 * pr) + 2 * (m & 1), i1 = i0 + 4;
            const __half2 r0 = __floats2half2_rn(tg_epi_val(acc[i0], bb, d.act), tg_epi_val(acc[i0 + 1], bb, d.act));
            const __half2 r1 = __floats2half2_rn(tg_epi_val(acc[i1], bb, d.act), tg_epi_val(acc[i1 + 1], bb, d.act));
            const __half2 mx = __hmax2(r0, r1);
            v[e] = __hmax(__low2half(mx), __high2half(mx));
          }
          const __half2 o = __halves2half2(v[0], v[1]);
          ov[m] = *reinterpret_cast<const uint32_t*>(&o);
        }
        stmatrix_x4_trans(out_s + (uint32_t)ip * 2048u + mat_off, ov);
      }
    } else {
#pragma unroll
      for (int jp = 0; jp < 8; ++jp) {
        const uint32_t addr = out_s + (uint32_t)jp * 2048u + mat_off;
        uint32_t rv[4], ov[4];
        if (has_res) ldmatrix_x4_trans(addr, rv);
#pragma unroll
        for (int m = 0; m < 4; ++m) {
          const int i = 4 * (2 * jp + (m >> 1)) + 2 * (m & 1);
          const float bb = (m & 1) ? b1 : b0;
          float a0 = tg_epi_val(acc[i], bb, d.act), a1 = tg_epi_val(acc[i + 1], bb, d.act);
          if (has_res) {
            const float2 rf = __half22float2(*reinterpret_cast<const __half2*>(&rv[m]));
            a0 += rf.x; a1 += rf.y;
          }
          const __half2 o = __floats2half2_rn(a0, a1);
          ov[m] = *reinterpret_cast<const uint32_t*>(&o);
        }
        stmatrix_x4_trans(addr, ov);
      }
    }
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
  const uint32_t bar_full = base + 8u * (cw * kMaxRing), bar_empty = base + 16 * kMaxRing + 8u * (cw * kMaxRing);
  const uint32_t bar_rfull = base + 32 * kMaxRing + 24 + 8u * cw, bar_free = base + 32 * kMaxRing + 40 + 8u * cw;
  const uint32_t stage0 = base + p.off_stage + (uint32_t)(cw * p.ring) * p.stage_bytes;
  const uint32_t epi_s = base + p.off_scratch + (uint32_t)cw * p.epi_bytes;
  constexpr uint32_t kBoxW = TW + 2;
  const uint64_t w_hi = gmma_desc_hi(1024u), x_hi = gmma_desc_hi(kBoxW * 128u);
  const uint32_t w16 = gmma_addr16(base + p.off_b), btb16 = p.b_stage_bytes >> 4;
  const int bar_id = 1 + cw;
  // where this thread's partial goes in the owner's receive buffer (senders only)
  const int my_slot = rank < owner ? rank : rank - 1;
  const uint32_t send_off = (uint32_t)((my_slot * wpr + (q - owner * wpr)) * 16) * 512u + (uint32_t)lane * 16u;
  const uint32_t peer_buf = mapa_shared(epi_s + send_off, (uint32_t)owner);
  const uint32_t peer_bar = mapa_shared(bar_rfull, (uint32_t)owner);
  const uint32_t recv_bytes = (uint32_t)((C - 1) * wpr) * 8192u;
  // stmatrix: lane l addresses pixel row kk of matrix m = l/8 = (tile row pair, 8-channel chunk 2*q + m%2); in the
  // rank's slice tile that chunk is local chunk 2*(q - rank*wpr) + m%2 (owners only)
  const uint32_t kk = POOL ? 4u * (lane & 1) + ((lane & 7) >> 1) : (uint32_t)(lane & 7);
  const uint32_t mat_off = (uint32_t)(8 * ((lane >> 3) >> 1) + kk) * sb +
                           ((uint32_t)(2 * (q - rank * wpr) + ((lane >> 3) & 1)) << 4);
  const int t0 = (int)cluster_id_x(), tstep = (int)cluster_count_x();
  // turns on the tensor pipe as in consumer_halo_pxn, over the CTA's tiles t0 + i * tstep; the waits for
  // peer CTAs (hand-back, partials) come after a tile's MMAs are issued, so the argument there holds here too
  const uint32_t turn_mine = base + 32 * kMaxRing + 56 + 8u * cw, turn_other = base + 32 * kMaxRing + 56 + 8u * (cw ^ 1);
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
    mbar_wait_mma(bar_full + 8 * s, phase);
    if (++stage == p.ring) { stage = 0; phase ^= 1u; }
    if (tile >= tstep) { mbar_wait_mma(turn_mine, tphase); tphase ^= 1u; }
    const uint32_t x16 = gmma_addr16(stage0 + (uint32_t)s * p.stage_bytes);
    wgmma_fence();
#pragma unroll
    for (int g = 0; g < 9; ++g) {
      const TgGroup gr = tg_group(TG_CONV_3X3, g);
      const uint32_t a16 = w16 + (uint32_t)g * btb16;
      const uint32_t b16 = x16 + (uint32_t)((gr.dy + 1) * (int)kBoxW + (gr.dx + 1)) * 8u;
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_n128(acc, w_hi | (uint64_t)(a16 + 2u * k), x_hi | (uint64_t)(b16 + 2u * k), (g == 0 && k == 0) ? 0u : 1u);
    }
    wgmma_commit();
    __syncwarp();
    if (lane == 0) mbar_arrive(turn_other);   // pass the turn
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_empty + 8 * s);

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
      if (POOL) {
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
              const __half2 r0 = __floats2half2_rn(tg_epi_val(acc[i0], bb, d.act), tg_epi_val(acc[i0 + 1], bb, d.act));
              const __half2 r1 = __floats2half2_rn(tg_epi_val(acc[i1], bb, d.act), tg_epi_val(acc[i1 + 1], bb, d.act));
              const __half2 mx = __hmax2(r0, r1);
              v[e] = __hmax(__low2half(mx), __high2half(mx));
            }
            const __half2 o = __halves2half2(v[0], v[1]);
            ov[m] = *reinterpret_cast<const uint32_t*>(&o);
          }
          stmatrix_x4_trans(epi_s + (uint32_t)ip * 16u * sb + mat_off, ov);
        }
      } else {
#pragma unroll
        for (int jp = 0; jp < 8; ++jp) {
          uint32_t ov[4];
#pragma unroll
          for (int m = 0; m < 4; ++m) {
            const int i = 4 * (2 * jp + (m >> 1)) + 2 * (m & 1);
            const float bb = (m & 1) ? b1 : b0;
            const __half2 o = __floats2half2_rn(tg_epi_val(acc[i], bb, d.act), tg_epi_val(acc[i + 1], bb, d.act));
            ov[m] = *reinterpret_cast<const uint32_t*>(&o);
          }
          stmatrix_x4_trans(epi_s + (uint32_t)jp * 16u * sb + mat_off, ov);
        }
      }
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
  const uint32_t bar_full = base + 8u * (cw * kMaxRing), bar_empty = base + 16 * kMaxRing + 8u * (cw * kMaxRing);
  const uint32_t stage0 = base + p.off_stage + (uint32_t)(cw * p.ring) * p.stage_bytes;
  const uint32_t out0 = base + p.off_scratch + (uint32_t)cw * 2u * kTapABytes;
  const uint32_t w16 = gmma_addr16(base + p.off_b);
  const int bar_id = 1 + cw;
  // as in consumer_halo_pxn: lane l addresses pixel row l%8 of matrix l/8 = (tile row 2*jp + m/2, chunk 2*q + m%2)
  const uint32_t mat_off = (uint32_t)(8 * ((lane >> 3) >> 1) + (lane & 7)) * 128u +
                           ((uint32_t)((2 * q + ((lane >> 3) & 1)) ^ (lane & 7)) << 4);
  int stage = 0;
  uint32_t phase = 0;
  float acc[64];

  for (int tile = blockIdx.x + cw * (int)gridDim.x; tile < p.num_tiles; tile += 2 * (int)gridDim.x) {
    const TileCoord tc = tile_coord(p, tile);
    const float b0 = bias_s[tc.nb * 64 + 16 * q + (lane >> 2)], b1 = bias_s[tc.nb * 64 + 16 * q + (lane >> 2) + 8];
    const int s = stage;
    mbar_wait_mma(bar_full + 8 * s, phase);
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
      if (a == 3) { __syncwarp(); if (lane == 0) mbar_arrive(bar_empty + 8 * s); }
      const uint32_t out_s = out0 + (uint32_t)(a & 1) * kTapABytes;
#pragma unroll
      for (int jp = 0; jp < 8; ++jp) {
        uint32_t ov[4];
#pragma unroll
        for (int m = 0; m < 4; ++m) {
          const int i = 4 * (2 * jp + (m >> 1)) + 2 * (m & 1);
          const float bb = (m & 1) ? b1 : b0;
          const __half2 o = __floats2half2_rn(tg_epi_val(acc[i], bb, d.act), tg_epi_val(acc[i + 1], bb, d.act));
          ov[m] = *reinterpret_cast<const uint32_t*>(&o);
        }
        stmatrix_x4_trans(out_s + (uint32_t)jp * 2048u + mat_off, ov);
      }
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
__global__ void __launch_bounds__(kThreads, 1)
conv_wgmma_kernel(const __grid_constant__ TgMaps maps, const KParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;   // 128B swizzle atoms need 1024B alignment
  uint8_t* sm = smem_raw + (base - raw);
  constexpr int BN = MODE == MODE_TAPN ? TG_TAPN_ROWS : 64;
  constexpr int NF = BN / 2;                      // accumulator registers per m64 half

  const int warp = __shfl_sync(0xFFFFFFFFu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const tg_conv_desc& d = p.d;

  // header: barriers, ring k of consumer c at index c * kMaxRing + k
  const uint32_t bar_full = base;                          // [2 * kMaxRing]
  const uint32_t bar_empty = base + 16 * kMaxRing;         // [2 * kMaxRing]
  const uint32_t bar_b = base + 32 * kMaxRing;             // [1]
  const uint32_t bar_res = bar_b + 8;                      // [2] residual tile of consumer c
  const uint32_t bar_rfull = bar_b + 24;                   // [2] MODE_SPLITK: partials received, consumer c
  const uint32_t bar_free = bar_b + 40;                    // [2] MODE_SPLITK: peers handed back their buffers
  const uint32_t bar_turn = bar_b + 56;                    // [2] pixels-on-N conv3x3 / split-K: consumer c may issue
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
    for (int s = 0; s < 2 * kMaxRing; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, 4);     // one arrival per consumer warp
    }
    mbar_init(bar_b, 1);
    mbar_init(bar_res, 1);
    mbar_init(bar_res + 8, 1);
    if (kSplitK) {
      for (int c = 0; c < 2; ++c) {
        mbar_init(bar_rfull + 8 * c, 1);             // the owner's expect_tx; the bytes come from the peers
        mbar_init(bar_free + 8 * c, p.chunks - 1);   // one hand-back per peer
      }
    }
    if (kSplitK || (kPxN && KIND == TG_CONV_3X3)) {
      mbar_init(bar_turn, 4);              // one arrival per warp of the other consumer
      mbar_init(bar_turn + 8, 4);
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
    // fixed per CTA: the number of CTAs (clusters for split-K) is a multiple of n_split
    const uint32_t nb = (uint32_t)sched0 % (uint32_t)p.n_split;
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
        const int cw = it & 1;
        const TileCoord tc = tile_coord(p, tile);
        const int n_loads = MODE == MODE_TAP ? 9 * p.chunks : kSplitK ? 1 : p.chunks;
        for (int l = 0; l < n_loads; ++l) {
          const int s = cw * kMaxRing + stage[cw];
          mbar_wait_mma(bar_empty + 8 * s, phase[cw] ^ 1);
          const uint32_t sa = smem_stage0 + (uint32_t)(cw * p.ring + stage[cw]) * p.stage_bytes;
          if (MODE != MODE_TAP) {
            mbar_expect_tx(bar_full + 8 * s, p.a_bytes);
            tma_load_4d(sa, &maps.m[0], bar_full + 8 * s, (l + k_rank) * 64, tc.x0 + p.org_x, tc.y0 + p.org_y, tc.n);
          } else {
            const int g = l / p.chunks, c = l - g * p.chunks;
            const TgGroup gr = tg_group(KIND, g);
            mbar_expect_tx(bar_full + 8 * s, p.a_bytes + (p.b_resident ? 0u : p.b_stage_bytes));
            tma_load_4d(sa, &maps.m[KIND == TG_CONV_3X3_S2 ? tg_s2_plane(g) : 0], bar_full + 8 * s, c * 64,
                        tc.x0 + gr.dx, tc.y0 + gr.dy, tc.n);
            if (!p.b_resident)
              bulk_load(sa + kTapABytes,
                        wglob + (size_t)(g * p.chunks + c) * p.b_tile_bytes + (size_t)tc.nb * p.b_stage_bytes,
                        p.b_stage_bytes, bar_full + 8 * s);
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
      if (lane == 0) mbar_arrive(bar_empty + 8 * (cw * kMaxRing + s));
    };
    auto next_stage = [&]() -> int {   // wait for the next stage of this consumer's ring; returns its index
      const int s = stage;
      mbar_wait_mma(bar_full + 8 * (cw * kMaxRing + s), phase);
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
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
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
int encode_f16(CUtensorMap* m, const void* ptr, int rank, const cuuint64_t* dims, const size_t* elem_strides,
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
int encode_nhwc(CUtensorMap* m, const void* ptr, int c, int w, int h, int n, size_t sw, size_t sh,
                size_t sn, int box_c, int box_w, int box_h, bool swizzle = true) {
  const cuuint64_t dims[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
  const size_t strides[3] = {sw, sh, sn};
  const cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
  return encode_f16(m, ptr, 4, dims, strides, box, swizzle);
}

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
    cfg.blockDim = dim3(kThreads);
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
  TG_REQUIRE(d->cin == 64 || d->cin == 128 || d->cin == 256, TG_E_UNSUPPORTED,
             "%s: cin=%d (stored channels must be 64, 128 or 256)", who, d->cin);
  if (d->epilogue == TG_EPI_NHWC_F16_POOL2)
    TG_REQUIRE(d->kind == TG_CONV_3X3 && d->residual == nullptr && d->act <= TG_ACT_LRELU02 && d->h >= 2 && d->w >= 2,
               TG_E_UNSUPPORTED, "%s: the pooled epilogue needs a conv3x3 without residual / derivative epilogue", who);
  if (d->epilogue == TG_EPI_NHWC_F16 || d->epilogue == TG_EPI_NHWC_F16_POOL2) {
    TG_REQUIRE(d->cout == 64 || d->cout == 128 || d->cout == 256, TG_E_UNSUPPORTED,
               "%s: cout=%d (64, 128 or 256 for the NHWC epilogue)", who, d->cout);
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
  TG_REQUIRE(d->a_mode >= TG_AMODE_AUTO && d->a_mode <= TG_AMODE_TAP, TG_E_INVALID, "conv: a_mode");
  TG_REQUIRE(((uintptr_t)d->x & 15) == 0 && ((uintptr_t)d->weights & 15) == 0 && ((uintptr_t)d->y & 15) == 0,
             TG_E_INVALID, "conv: pointers must be 16-byte aligned");

  KParams p;
  p.d = *d;
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
  const bool splitk = d->a_mode == TG_AMODE_AUTO && d->kind == TG_CONV_3X3 && !bwd && !tapn && p.chunks >= 2 &&
                      d->residual == nullptr;
  const uint32_t b_total = (tapn ? 1u : 9u) * (splitk ? 1u : (uint32_t)p.chunks) * p.b_stage_bytes;   // resident slice per CTA
  const int hbox_w = d->kind != TG_CONVT_3X3_S2 ? TW + 2 : TW + 1;
  const int hbox_h = d->kind != TG_CONVT_3X3_S2 ? TH + 2 : TH + 1;
  const uint32_t halo_bytes = (uint32_t)hbox_w * hbox_h * 128u;
  const uint32_t halo_stage = (halo_bytes + 1023u) & ~1023u;
  const uint32_t scratch = 2u * scratch_bytes(tapn ? MODE_TAPN : MODE_TAP);
  const uint32_t fixed = 1024u /*align slack*/ + kHeaderBytes + scratch;

  // every consumer needs at least one stage of its own
  const bool can_resident_halo = fixed + b_total + 2u * halo_stage <= kSmemLimit &&
                                 !(d->kind == TG_CONVT_3X3_S2 && p.chunks != 1);
  const bool can_resident_tap = fixed + b_total + 2u * kTapABytes <= kSmemLimit;
  int mode = d->a_mode;
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
  const bool pxn = p.halo && !bwd && !tapn && !splitk;
  p.epi_bytes = splitk ? (uint32_t)((p.chunks - 1) * (4 / p.chunks)) * 8192u : 0u;
  const uint32_t epi_tiles = splitk ? 2u * p.epi_bytes
                             : !pxn ? scratch : convT ? 4u * kTapABytes : pool ? 2u * kPoolTileBytes : 2u * kTapABytes;
  const uint32_t avail = kSmemLimit - 1024u - kHeaderBytes - epi_tiles - (p.b_resident ? b_total : 0u);
  int ring = (int)(avail / p.stage_bytes) / 2;
  if (ring > kMaxRing) ring = kMaxRing;
  TG_REQUIRE(ring >= 1, TG_E_UNSUPPORTED, "conv: shared memory budget (cin=%d cout=%d)", d->cin, d->cout);
  p.ring = ring;
  p.off_b = kHeaderBytes;
  p.off_stage = kHeaderBytes + (p.b_resident ? b_total : 0u);
  p.off_scratch = p.off_stage + 2u * (uint32_t)ring * p.stage_bytes;   // consumer c's ring: stages [c*ring, (c+1)*ring)
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
  const dim3 b(kThreads);
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
    const dim3 g(ncl * C);
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
    lerr = p.halo ? tg_launch(conv_wgmma_kernel<TG_CONV_3X3, MODE_HALO, false, true>, g, b, kSmemLimit, st, map_a, p)
                  : tg_launch(conv_wgmma_kernel<TG_CONV_3X3, MODE_TAP, false, true>, g, b, kSmemLimit, st, map_a, p);
  } else if (bwd) {
    if (d->kind == TG_CONV_3X3_S2)
      lerr = tg_launch(conv_wgmma_kernel<TG_CONV_3X3_S2, MODE_TAP, true>, g, b, kSmemLimit, st, map_a, p);
    else if (p.halo)
      lerr = tg_launch(conv_wgmma_kernel<TG_CONV_3X3, MODE_HALO, true>, g, b, kSmemLimit, st, map_a, p);
    else
      lerr = tg_launch(conv_wgmma_kernel<TG_CONV_3X3, MODE_TAP, true>, g, b, kSmemLimit, st, map_a, p);
  } else if (tapn) {
    lerr = tg_launch(conv_wgmma_kernel<TG_CONV_3X3, MODE_TAPN>, g, b, kSmemLimit, st, map_a, p);
  } else if (d->kind == TG_CONV_3X3) {
    lerr = p.halo ? tg_launch(conv_wgmma_kernel<TG_CONV_3X3, MODE_HALO>, g, b, kSmemLimit, st, map_a, p)
                  : tg_launch(conv_wgmma_kernel<TG_CONV_3X3, MODE_TAP>, g, b, kSmemLimit, st, map_a, p);
  } else {
    lerr = p.halo ? tg_launch(conv_wgmma_kernel<TG_CONVT_3X3_S2, MODE_HALO>, g, b, kSmemLimit, st, map_a, p)
                  : tg_launch(conv_wgmma_kernel<TG_CONVT_3X3_S2, MODE_TAP>, g, b, kSmemLimit, st, map_a, p);
  }
  TG_REQUIRE(lerr == cudaSuccess, (int)lerr, "conv: launch failed: %s", cudaGetErrorString(lerr));
  TG_CUDA_LAUNCH_CHECK("conv");
  return TG_OK;
}


}  // extern "C"
