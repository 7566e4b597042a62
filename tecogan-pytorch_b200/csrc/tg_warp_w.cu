// Fused backward_warp + space_to_depth + concat, warp-autonomous version (C = 3).
//
// Same arithmetic as warp_s2d_concat_kernel (tg_elementwise.cu; net_utils.py:36-82, tecogan_nets.py:141,
// 239-247) but every WARP is its own pipeline: one unit = 32 consecutive HR columns (= 32/S LR pixels) of
// one LR row; the warp stages its flow neighbourhood, gathers, transposes through a warp-private
// shared-memory tile and stores -- synchronised with __syncwarp only.  The CTA-wide version runs its four
// warps in lock step (two __syncthreads per LR row), so while one phase waits on DRAM nothing else of that
// CTA is in flight.  Here warps drift apart and the gathers of one overlap the stores / flow staging of the
// others; units are handed out grid-stride, and the small flow / lr reads of the next unit are prefetched
// into registers so a unit costs one dependent DRAM round trip.
#include "tg_common.cuh"

#include <cstdlib>

namespace {

constexpr int kWarpsPerCta = 4;
constexpr int kDefaultOcc = 5;

// FLOW: 0 = HR flow given; 1 / 2 = LR flow upsampled inline with the bicubic / bilinear upsample_func
template <int S, int FLOW, int OCC>
__global__ void __launch_bounds__(32 * kWarpsPerCta, OCC)
warp_s2d_concat_w_kernel(const float* __restrict__ hr_prev, const float* __restrict__ flow,
                         const float* __restrict__ lr_curr, __half* __restrict__ out, int n, int h, int w,
                         int h8, int w8, int cpad) {
  tg_pdl_wait();
  tg_pdl_trigger();
  constexpr bool LRFLOW = FLOW != 0;
  constexpr int up_mode = FLOW == 2 ? TG_UP_BILINEAR : TG_UP_BICUBIC;
  constexpr int LRW = 32 / S;                 // LR pixels per unit
  constexpr int FW = LRW + 3, FH = 4;         // flow neighbourhood: LR cols x0-1 .. x0+LRW+1, rows y-1 .. y+2
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tstride = cpad + 8;               // halves per tile pixel (+16 B: conflict-free 2-byte stores)
  const int tile_bytes = LRW * tstride * 2;
  const int per_warp = (tile_bytes + 2 * FH * FW * 4 + 15) & ~15;
  __half* tile = reinterpret_cast<__half*>(smem_raw + warp * per_warp);
  float* fsrc = reinterpret_cast<float*>(smem_raw + warp * per_warp + tile_bytes);   // [comp][row][col]

  const int H = h * S, W = w * S;
  const int xblocks = (w + LRW - 1) / LRW;
  const long long units = (long long)n * h * xblocks;
  const int lx = lane / S, sx = lane - lx * S;
  // pad channels [(S*S+1)*3, cpad) are never written again: zero the warp's tile once
  for (int i = lane; i < LRW * tstride / 8; i += 32) reinterpret_cast<uint4*>(tile)[i] = make_uint4(0u, 0u, 0u, 0u);
  __syncwarp();

  const long long wstride = (long long)gridDim.x * kWarpsPerCta;
  // Software pipeline over units: the (small) flow and lr_curr reads of unit u+1 are issued while unit u gathers,
  // so a unit costs ONE dependent DRAM round trip (the gathers) instead of two.
  constexpr int NF = LRFLOW ? (2 * FH * FW + 31) / 32 : 2 * S;     // prefetched flow values per lane
  constexpr int NL = (LRW * 3 + 31) / 32;                         // prefetched lr_curr values per lane
  float pf[NF], pl[NL];
  // unit -> (image, LR row, column block), walked incrementally: no (64-bit) divisions per unit -- the kernel is
  // close to issue-bound (~870 warp instructions per unit in the ncu capture), index arithmetic included
  struct UnitPos { int nn, y, xb; };
  const int step_x = (int)(wstride % xblocks), step_y = (int)(wstride / xblocks);
  auto advance = [&](UnitPos& c) {
    c.xb += step_x;
    c.y += step_y;
    if (c.xb >= xblocks) { c.xb -= xblocks; ++c.y; }
    while (c.y >= h) { c.y -= h; ++c.nn; }
  };
  // lane-constant decompositions of the prefetch indices (hoisted out of the unit loop)
  int f_col[NF], f_row[NF], f_comp[NF], l_k[NL], l_p[NL];
#pragma unroll
  for (int j = 0; j < NF; ++j) {
    const int i = lane + 32 * j;
    f_col[j] = i % FW; f_row[j] = (i / FW) % FH; f_comp[j] = i / (FH * FW);
  }
#pragma unroll
  for (int j = 0; j < NL; ++j) {
    const int i = lane + 32 * j;
    l_k[j] = i / LRW; l_p[j] = i - l_k[j] * LRW;
  }
  auto prefetch = [&](const UnitPos& c) {
    const int xb = c.xb, y = c.y, nn = c.nn;
    const int x0 = xb * LRW;
    if (LRFLOW) {
      // hr_flow = S * upsample_func(reflect_pad(lr_flow))   (tecogan_nets.py:239-244)
#pragma unroll
      for (int j = 0; j < NF; ++j) {
        const int i = lane + 32 * j;
        float v = 0.f;
        if (i < 2 * FH * FW) {
          const int yy = tg_reflect_hi(tg_clampi(y - 1 + f_row[j], 0, h - 1), h8);
          const int xx = tg_reflect_hi(tg_clampi(x0 - 1 + f_col[j], 0, w - 1), w8);
          v = __ldg(flow + (((size_t)nn * 2 + f_comp[j]) * h8 + yy) * w8 + xx);
        }
        pf[j] = v;
      }
    } else {
      const int X = x0 * S + lane;
#pragma unroll
      for (int j = 0; j < NF; ++j) pf[j] = 0.f;
      if (X < W) {
        const float* f0 = flow + (((size_t)nn * 2 + 0) * H + (size_t)y * S) * W + X;
        const float* f1 = flow + (((size_t)nn * 2 + 1) * H + (size_t)y * S) * W + X;
#pragma unroll
        for (int sy = 0; sy < S; ++sy) {
          pf[sy] = __ldg(f0 + (size_t)sy * W);
          pf[S + sy] = __ldg(f1 + (size_t)sy * W);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < NL; ++j) {
      const int i = lane + 32 * j;
      float v = 0.f;
      if (i < LRW * 3 && x0 + l_p[j] < w) v = __ldg(lr_curr + (((size_t)nn * 3 + l_k[j]) * h + y) * w + x0 + l_p[j]);
      pl[j] = v;
    }
  };
  const long long u_first = (long long)blockIdx.x * kWarpsPerCta + warp;
  UnitPos cur, nxt;
  cur.xb = (int)(u_first % xblocks);
  cur.y = (int)((u_first / xblocks) % h);
  cur.nn = (int)(u_first / ((long long)xblocks * h));
  nxt = cur;
  if (u_first < units) prefetch(cur);
  for (long long u = u_first; u < units; u += wstride, cur = nxt) {
    const int xb = cur.xb, y = cur.y, nn = cur.nn;
    const int x0 = xb * LRW;
    const int X = x0 * S + lane;
    float uu[S], vv[S];
    // hand the prefetched values over (shared memory for the LR flow neighbourhood and the lr channels) ...
    if (LRFLOW) {
#pragma unroll
      for (int j = 0; j < NF; ++j)
        if (lane + 32 * j < 2 * FH * FW) fsrc[lane + 32 * j] = pf[j];
    } else {
#pragma unroll
      for (int sy = 0; sy < S; ++sy) { uu[sy] = pf[sy]; vv[sy] = pf[S + sy]; }
    }
#pragma unroll
    for (int j = 0; j < NL; ++j) {
      if (lane + 32 * j < LRW * 3) tile[l_p[j] * tstride + l_k[j]] = __float2half(pl[j]);
    }
    // ... and start the next unit's reads before this unit's gathers
    advance(nxt);
    if (u + wstride < units) prefetch(nxt);
    if (LRFLOW) {
      __syncwarp();
      float kx[4], hx[2][FH];
      tg_up_taps(up_mode, sx, S, kx);
#pragma unroll
      for (int comp = 0; comp < 2; ++comp)
#pragma unroll
        for (int row = 0; row < FH; ++row) {
          const float* f = fsrc + (comp * FH + row) * FW + lx;
          hx[comp][row] = kx[0] * f[0] + kx[1] * f[1] + kx[2] * f[2] + kx[3] * f[3];
        }
#pragma unroll
      for (int sy = 0; sy < S; ++sy) {
        float ky[4];
        tg_up_taps(up_mode, sy, S, ky);
        uu[sy] = (float)S * (ky[0] * hx[0][0] + ky[1] * hx[0][1] + ky[2] * hx[0][2] + ky[3] * hx[0][3]);
        vv[sy] = (float)S * (ky[0] * hx[1][0] + ky[1] * hx[1][1] + ky[2] * hx[1][2] + ky[3] * hx[1][3]);
      }
    }
    if (X < W) {
      int o00[S];
      float ax[S], ay[S];
#pragma unroll
      for (int sy = 0; sy < S; ++sy) {
        float fx = (float)X + uu[sy];
        float fy = (float)(y * S + sy) + vv[sy];
        fx = fminf(fmaxf(fx, 0.f), (float)(W - 1));
        fy = fminf(fmaxf(fy, 0.f), (float)(H - 1));
        // corner pair shifted left / up at the far border, fraction 1: bit-identical to padding_mode='border'
        const int xa = min((int)floorf(fx), W - 2), ya = min((int)floorf(fy), H - 2);
        ax[sy] = fx - (float)xa; ay[sy] = fy - (float)ya;
        o00[sy] = ya * W + xa;
      }
      float g[S][3][4];
      const float* img = hr_prev + (size_t)nn * 3 * H * W;
#pragma unroll
      for (int sy = 0; sy < S; ++sy)
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const float* r0 = img + (size_t)k * H * W + o00[sy];
          const float* r1 = r0 + W;
          g[sy][k][0] = __ldg(r0); g[sy][k][1] = __ldg(r0 + 1);
          g[sy][k][2] = __ldg(r1); g[sy][k][3] = __ldg(r1 + 1);
        }
#pragma unroll
      for (int sy = 0; sy < S; ++sy) {
        __half* dst = tile + lx * tstride + 3 + (sy * S + sx) * 3;     // s2d channel (sy*S+sx)*3 + k, after lr
        const float w00 = (1.f - ax[sy]) * (1.f - ay[sy]), w01 = ax[sy] * (1.f - ay[sy]);
        const float w10 = (1.f - ax[sy]) * ay[sy], w11 = ax[sy] * ay[sy];
#pragma unroll
        for (int k = 0; k < 3; ++k)
          dst[k] = __float2half(g[sy][k][0] * w00 + g[sy][k][1] * w01 + g[sy][k][2] * w10 + g[sy][k][3] * w11);
      }
    }
    __syncwarp();
    const int npx = min(LRW, w - x0);
    const int vec_per_px = cpad / 8;
    uint4* dstg = reinterpret_cast<uint4*>(out + (((size_t)nn * h + y) * w + x0) * cpad);
    for (int i = lane; i < npx * vec_per_px; i += 32) {
      const int px = i / vec_per_px, v8 = i - px * vec_per_px;
      dstg[i] = *reinterpret_cast<const uint4*>(tile + px * tstride + v8 * 8);
    }
    __syncwarp();        // the tile and fsrc are rewritten by the next unit
  }
}


}  // namespace

// launcher used by warp_launch() in tg_elementwise.cu (C == 3 only); returns cudaSuccess or the launch error
cudaError_t tg_warp_w_launch(const float* hr_prev, const float* flow, const float* lr_curr, __half* out, int n, int h,
                             int w, int h8, int w8, int s, int fm, int cpad, cudaStream_t st) {
  const int lrw = 32 / s;
  const size_t per_warp = ((size_t)lrw * (cpad + 8) * 2 + 2 * 4 * (lrw + 3) * 4 + 15) & ~(size_t)15;
  const size_t smem = per_warp * kWarpsPerCta;
  const long long units = (long long)n * h * ((w + lrw - 1) / lrw);
  long long ctas = (units + kWarpsPerCta - 1) / kWarpsPerCta;
  // resident CTAs per SM (register cap 65536 / (128 * OCC)): TG_WARP_OCC = 5..8 for A/B measurements
  static int occ = 0;
  if (occ == 0) {
    const char* e = getenv("TG_WARP_OCC");
    occ = e != nullptr ? atoi(e) : kDefaultOcc;
    if (occ < 5 || occ > 8) occ = kDefaultOcc;
  }
  const long long cap = (long long)tg_sms() * occ;            // one resident wave: every warp walks several units and the warps
                                                 // of an SM drift out of phase
  if (ctas > cap) ctas = cap;
  if (ctas < 1) ctas = 1;
  dim3 grid((unsigned)ctas), block(32 * kWarpsPerCta);
#define TG_W3(SS, FM, OC) return tg_launch(warp_s2d_concat_w_kernel<SS, FM, OC>, grid, block, smem, st, hr_prev, flow, lr_curr, out, n, h, w, h8, w8, cpad)
#define TG_W(SS, FM) do { if (occ == 5) TG_W3(SS, FM, 5); if (occ == 6) TG_W3(SS, FM, 6); if (occ == 7) TG_W3(SS, FM, 7); TG_W3(SS, FM, 8); } while (0)
  if (s == 4) { if (fm == 0) TG_W(4, 0); if (fm == 1) TG_W(4, 1); TG_W(4, 2); }
  if (fm == 0) TG_W(2, 0);
  if (fm == 1) TG_W(2, 1);
  TG_W(2, 2);
#undef TG_W
#undef TG_W3
}
