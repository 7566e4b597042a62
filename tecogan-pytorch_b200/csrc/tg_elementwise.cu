// HBM-bound kernels of the FRNet hot path: fused warp + space_to_depth + concat, FNet's
// pool / x2-upsample, layout packs, module-boundary NCHW fp32 ops, uint8 quantisation.
// Reference call sites are cited per entry point in include/tecogan_b200.h.
#include "tg_common.cuh"

#include <cstdlib>

namespace {

// =====================================================================================
// fused backward_warp + space_to_depth + concat
//
// One CTA produces the SRNet input of LRW = 128/S consecutive LR pixels of one LR row:
//   - 128 threads = 128 consecutive HR columns; each thread walks the S HR rows of the
//     LR row (flow reads are 512-byte coalesced row segments per plane, the 4-corner
//     gathers of hr_prev stay within a few 128B lines because the flow is smooth),
//   - results are transposed through shared memory into NHWC pixels (cpad fp16 each) so
//     the CTA stores one contiguous LRW*cpad*2-byte run with 16-byte vectors.
// Warp arithmetic follows net_utils.py:50-82 in closed form: sample at (X+u, Y+v), clamp to
// the border, x1=min(x0+1,W-1)  (SURVEY.md 8-a4).
// =====================================================================================
__device__ __forceinline__ float bilerp_border(const float* __restrict__ plane, int H, int W,
                                               float fx, float fy) {
  fx = fminf(fmaxf(fx, 0.f), (float)(W - 1));
  fy = fminf(fmaxf(fy, 0.f), (float)(H - 1));
  const float x0f = floorf(fx), y0f = floorf(fy);
  const int x0 = (int)x0f, y0 = (int)y0f;
  const int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
  const float ax = fx - x0f, ay = fy - y0f;
  const float* r0 = plane + (size_t)y0 * W;
  const float* r1 = plane + (size_t)y1 * W;
  const float v00 = __ldg(r0 + x0), v01 = __ldg(r0 + x1);
  const float v10 = __ldg(r1 + x0), v11 = __ldg(r1 + x1);
  return v00 * (1.f - ax) * (1.f - ay) + v01 * ax * (1.f - ay) + v10 * (1.f - ax) * ay +
         v11 * ax * ay;
}

// One CTA = RY LR rows x LRW=128/S LR pixels; 128 threads, thread t owns HR column X = x0*S + t and
// walks the S HR rows of each LR row in passes of SP rows (SP*12 independent gathers in flight per
// thread; SP = 2 keeps the kernel at <= 64 registers -> 8 CTAs = 32 warps per SM, twice the bytes in
// flight per SM of the SP = S version that ncu showed latency-bound at 29 % occupancy).
//   LRFLOW: the LR flow neighbourhood ((RY+3) rows x LRW+3 cols, reflect-padded + replicate-clamped)
//   is staged in smem once; each thread evaluates the x-pass of the separable 4-tap upsampler for its
//   own column into registers (RY+3 values per component) and the y-pass per HR row.
//   FLOW: 0 = HR flow given; 1 / 2 = LR flow, upsampled inline with the bicubic / bilinear
//   upsample_func (compile time, so the y-pass taps are immediates).
//   The NHWC transpose goes through a shared-memory tile whose pixel stride is cpad*2 + 16 bytes:
//   with the natural 128-byte stride the 8 LR pixels of a warp hit the same bank (8-way conflict on
//   every 2-byte store -- the top stall of the round-1 capture); +16 B spreads them over all banks
//   and keeps the 16-byte alignment of the vector read-out.
template <int S, int FLOW, int RY, int SP>
__global__ void __launch_bounds__(128, SP == S ? 5 : 8)
warp_s2d_concat_kernel(const float* __restrict__ hr_prev, const float* __restrict__ flow,
                       const float* __restrict__ lr_curr, __half* __restrict__ out, int C, int h,
                       int w, int h8, int w8, int cpad) {
  tg_pdl_wait();
  tg_pdl_trigger();
  constexpr bool LRFLOW = FLOW != 0;
  constexpr int up_mode = FLOW == 2 ? TG_UP_BILINEAR : TG_UP_BICUBIC;
  constexpr int LRW = 128 / S;
  constexpr int FW = LRW + 3;                 // LR columns x0-1 .. x0+LRW+1
  constexpr int FH = RY + 3;                  // LR rows    y0-1 .. y0+RY+1
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int tstride = cpad + 8;               // halves per tile pixel (cpad*2 + 16 bytes)
  __half* tile = reinterpret_cast<__half*>(smem_raw);  // [LRW][tstride]
  __shared__ float fsrc[LRFLOW ? 2 * FH * FW : 1];     // [comp][row][col]

  const int t = threadIdx.x;
  const int x0 = blockIdx.x * LRW;      // first LR column of the tile
  const int y0 = blockIdx.y * RY;       // first LR row
  const int n = blockIdx.z;
  const int H = h * S, W = w * S;
  const int X = x0 * S + t;             // HR column of this thread
  const int lx = t / S, sx = t - lx * S;

  // the pad channels [(S*S+1)*C, cpad) are never written again: zero the whole tile once
  for (int i = t; i < LRW * tstride / 8; i += 128) reinterpret_cast<uint4*>(tile)[i] = make_uint4(0u, 0u, 0u, 0u);

  float hx[2][FH];                      // x-pass of the flow upsampler, this thread's column
  if (LRFLOW) {
    // hr_flow = S * upsample_func(reflect_pad(lr_flow))   (tecogan_nets.py:239-244)
    for (int i = t; i < 2 * FH * FW; i += 128) {
      const int col = i % FW, row = (i / FW) % FH, comp = i / (FH * FW);
      const int yy = tg_reflect_hi(tg_clampi(y0 - 1 + row, 0, h - 1), h8);
      const int xx = tg_reflect_hi(tg_clampi(x0 - 1 + col, 0, w - 1), w8);
      fsrc[i] = __ldg(flow + (((size_t)n * 2 + comp) * h8 + yy) * w8 + xx);
    }
    __syncthreads();
    float kx[4];
    tg_up_taps(up_mode, sx, S, kx);
#pragma unroll
    for (int comp = 0; comp < 2; ++comp)
#pragma unroll
      for (int row = 0; row < FH; ++row) {
        const float* f = fsrc + (comp * FH + row) * FW + lx;   // taps at LR cols lx-1 .. lx+2
        hx[comp][row] = kx[0] * f[0] + kx[1] * f[1] + kx[2] * f[2] + kx[3] * f[3];
      }
  }

#pragma unroll
  for (int ry = 0; ry < RY; ++ry) {
    const int y = y0 + ry;
    if (y >= h) break;                  // uniform over the CTA
    if (ry == 0) __syncthreads();       // (tile zeroing / flow staging above) before the first channel writes
    // stage lr_curr
    for (int i = t; i < LRW * C; i += 128) {
      const int k = i / LRW, p = i - k * LRW;
      const int xx = x0 + p;
      float v = 0.f;
      if (xx < w) v = __ldg(lr_curr + (((size_t)n * C + k) * h + y) * w + xx);
      tile[p * tstride + k] = __float2half(v);
    }
    if (X < W) {
#pragma unroll
      for (int s0 = 0; s0 < S; s0 += SP) {
        float u[SP], v[SP];
        if (LRFLOW) {
#pragma unroll
          for (int j = 0; j < SP; ++j) {
            float ky[4];
            tg_up_taps(up_mode, s0 + j, S, ky);
            u[j] = (float)S * (ky[0] * hx[0][ry] + ky[1] * hx[0][ry + 1] + ky[2] * hx[0][ry + 2] + ky[3] * hx[0][ry + 3]);
            v[j] = (float)S * (ky[0] * hx[1][ry] + ky[1] * hx[1][ry + 1] + ky[2] * hx[1][ry + 2] + ky[3] * hx[1][ry + 3]);
          }
        } else {
          const float* f0 = flow + (((size_t)n * 2 + 0) * H + (size_t)y * S + s0) * W + X;
          const float* f1 = flow + (((size_t)n * 2 + 1) * H + (size_t)y * S + s0) * W + X;
#pragma unroll
          for (int j = 0; j < SP; ++j) {
            u[j] = __ldg(f0 + (size_t)j * W);
            v[j] = __ldg(f1 + (size_t)j * W);
          }
        }
        if (C == 3) {
          // two-phase gather: compute the corner offsets of the SP pixels, issue all 12*SP loads,
          // then combine -- independent loads in flight per thread hide the L2/DRAM latency
          int o00[SP];
          float ax[SP], ay[SP];
#pragma unroll
          for (int j = 0; j < SP; ++j) {
            float fx = (float)X + u[j];
            float fy = (float)(y * S + s0 + j) + v[j];
            fx = fminf(fmaxf(fx, 0.f), (float)(W - 1));
            fy = fminf(fmaxf(fy, 0.f), (float)(H - 1));
            // The four corners are (ya,xa),(ya,xa+1),(ya+1,xa),(ya+1,xa+1) with xa <= W-2, ya <= H-2:
            // at the far border (fx == W-1) the pair is shifted one to the left and the fraction
            // becomes 1, which selects the same sample with weight exactly 1 (bit-identical result,
            // net_utils.py:76 padding_mode='border') -- and the corner addresses are immediates of
            // two base addresses instead of four independent ones.
            const int xa = min((int)floorf(fx), W - 2), ya = min((int)floorf(fy), H - 2);
            ax[j] = fx - (float)xa; ay[j] = fy - (float)ya;
            o00[j] = ya * W + xa;
          }
          float g[SP][3][4];
          const float* img = hr_prev + (size_t)n * 3 * H * W;
#pragma unroll
          for (int j = 0; j < SP; ++j)
#pragma unroll
            for (int k = 0; k < 3; ++k) {
              const float* r0 = img + (size_t)k * H * W + o00[j];
              const float* r1 = r0 + W;
              g[j][k][0] = __ldg(r0); g[j][k][1] = __ldg(r0 + 1);
              g[j][k][2] = __ldg(r1); g[j][k][3] = __ldg(r1 + 1);
            }
#pragma unroll
          for (int j = 0; j < SP; ++j) {
            // space_to_depth channel (sy*S+sx)*C + k  (net_utils.py:36-47), after the C lr channels
            __half* dst = tile + lx * tstride + 3 + ((s0 + j) * S + sx) * 3;
            const float w00 = (1.f - ax[j]) * (1.f - ay[j]), w01 = ax[j] * (1.f - ay[j]);
            const float w10 = (1.f - ax[j]) * ay[j], w11 = ax[j] * ay[j];
#pragma unroll
            for (int k = 0; k < 3; ++k)
              dst[k] = __float2half(g[j][k][0] * w00 + g[j][k][1] * w01 + g[j][k][2] * w10 + g[j][k][3] * w11);
          }
        } else {
#pragma unroll
          for (int j = 0; j < SP; ++j) {
            const float fx = (float)X + u[j];
            const float fy = (float)(y * S + s0 + j) + v[j];
            __half* dst = tile + lx * tstride + C + ((s0 + j) * S + sx) * C;
            for (int k = 0; k < C; ++k) {
              const float* plane = hr_prev + ((size_t)n * C + k) * H * W;
              dst[k] = __float2half(bilerp_border(plane, H, W, fx, fy));
            }
          }
        }
      }
    }
    __syncthreads();
    // coalesced store of min(LRW, w-x0) pixels * cpad halves (cpad*2 bytes, multiple of 16)
    const int npx = min(LRW, w - x0);
    const int vec_per_px = cpad / 8;  // uint4 per pixel
    uint4* dstg = reinterpret_cast<uint4*>(out + (((size_t)n * h + y) * w + x0) * cpad);
    for (int i = t; i < npx * vec_per_px; i += 128) {
      const int px = i / vec_per_px, vv = i - px * vec_per_px;
      dstg[i] = *reinterpret_cast<const uint4*>(tile + px * tstride + vv * 8);
    }
    __syncthreads();
  }
}

// =====================================================================================
// FNet helpers on NHWC fp16 (8 channels = one 16-byte vector per thread)
// =====================================================================================
__global__ void maxpool2x2_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int n, int h,
                                  int w, int c8) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int ho = h / 2, wo = w / 2;
  const size_t total = (size_t)n * ho * wo * c8;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % c8);
    size_t p = i / c8;
    const int xo = (int)(p % wo); p /= wo;
    const int yo = (int)(p % ho);
    const int nn = (int)(p / ho);
    const size_t base = (((size_t)nn * h + 2 * yo) * w + 2 * xo) * c8 + cv;
    uint4 a = __ldg(x + base), b = __ldg(x + base + c8);
    uint4 c = __ldg(x + base + (size_t)w * c8), d = __ldg(x + base + (size_t)w * c8 + c8);
    uint4 r;
    const __half2* ah = reinterpret_cast<const __half2*>(&a);
    const __half2* bh = reinterpret_cast<const __half2*>(&b);
    const __half2* ch = reinterpret_cast<const __half2*>(&c);
    const __half2* dh = reinterpret_cast<const __half2*>(&d);
    __half2* rh = reinterpret_cast<__half2*>(&r);
#pragma unroll
    for (int k = 0; k < 4; ++k) rh[k] = __hmax2(__hmax2(ah[k], bh[k]), __hmax2(ch[k], dh[k]));
    y[i] = r;
  }
}

// F.interpolate(scale_factor=2, bilinear, align_corners=False):
// out[2i] = .25*in[max(i-1,0)] + .75*in[i], out[2i+1] = .75*in[i] + .25*in[min(i+1,L-1)]
// One thread = one INPUT position (8 channels): 9 independent 16-byte loads of its 3x3 clamped
// neighbourhood, four 16-byte outputs (the 2x2 block it expands to) -- 9 loads per 4 outputs
// instead of 16, all in flight together, 32-bit index arithmetic.
__device__ __forceinline__ void up2_mix(const uint4& a, const uint4& b, float wa, float wb, float2 o[4]) {
  const __half2* pa = reinterpret_cast<const __half2*>(&a);
  const __half2* pb = reinterpret_cast<const __half2*>(&b);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 fa = __half22float2(pa[k]), fb = __half22float2(pb[k]);
    o[k].x = wa * fa.x + wb * fb.x;
    o[k].y = wa * fa.y + wb * fb.y;
  }
}
__device__ __forceinline__ uint4 up2_out(const float2 a[4], const float2 b[4], float wa, float wb) {
  uint4 r;
  __half2* rh = reinterpret_cast<__half2*>(&r);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float2 o;
    o.x = wa * a[k].x + wb * b[k].x;
    o.y = wa * a[k].y + wb * b[k].y;
    rh[k] = __float22half2_rn(o);
  }
  return r;
}
__global__ void __launch_bounds__(256)
upsample2x_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int n, int h, int w, int c8) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int total = n * h * w * c8;
  const int wo = 2 * w;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int cv = i % c8;
    int p = i / c8;
    const int xi = p % w; p /= w;
    const int yi = p % h;
    const int nn = p / h;
    const int ya = max(yi - 1, 0), yc = min(yi + 1, h - 1);
    const int xa = max(xi - 1, 0), xc = min(xi + 1, w - 1);
    const uint4* r0 = x + ((size_t)(nn * h + ya) * w) * c8 + cv;
    const uint4* r1 = x + ((size_t)(nn * h + yi) * w) * c8 + cv;
    const uint4* r2 = x + ((size_t)(nn * h + yc) * w) * c8 + cv;
    const uint4 v00 = __ldg(r0 + xa * c8), v01 = __ldg(r0 + xi * c8), v02 = __ldg(r0 + xc * c8);
    const uint4 v10 = __ldg(r1 + xa * c8), v11 = __ldg(r1 + xi * c8), v12 = __ldg(r1 + xc * c8);
    const uint4 v20 = __ldg(r2 + xa * c8), v21 = __ldg(r2 + xi * c8), v22 = __ldg(r2 + xc * c8);
    // x pass per row: even output column = .25*in[x-1] + .75*in[x], odd = .75*in[x] + .25*in[x+1]
    float2 e0[4], o0[4], e1[4], o1[4], e2[4], o2[4];
    up2_mix(v00, v01, 0.25f, 0.75f, e0); up2_mix(v01, v02, 0.75f, 0.25f, o0);
    up2_mix(v10, v11, 0.25f, 0.75f, e1); up2_mix(v11, v12, 0.75f, 0.25f, o1);
    up2_mix(v20, v21, 0.25f, 0.75f, e2); up2_mix(v21, v22, 0.75f, 0.25f, o2);
    uint4* out0 = y + ((size_t)(nn * 2 * h + 2 * yi) * wo + 2 * xi) * c8 + cv;   // output row 2*yi
    uint4* out1 = out0 + (size_t)wo * c8;                                       // output row 2*yi+1
    out0[0] = up2_out(e0, e1, 0.25f, 0.75f);
    out0[c8] = up2_out(o0, o1, 0.25f, 0.75f);
    out1[0] = up2_out(e1, e2, 0.75f, 0.25f);
    out1[c8] = up2_out(o1, o2, 0.75f, 0.25f);
  }
}

// FNet input: cat([x1,x2],1) of two 3-channel NCHW fp32 images -> NHWC fp16 c64 (tecogan_nets.py:71).
// One thread = one pixel: 2*c coalesced plane loads, then the pixel's whole 128-byte row (six
// values + zeros) in eight 128-bit stores.
__global__ void __launch_bounds__(256)
pack_pair_c64_kernel(const float* __restrict__ x1, const float* __restrict__ x2, uint4* __restrict__ y,
                     int n, int c, int hw) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int total = n * hw;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int nn = i / hw, sp = i - nn * hw;
    __align__(16) __half vals[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      float v = 0.f;
      if (k < c) v = __ldg(x1 + ((size_t)nn * c + k) * hw + sp);
      else if (k < 2 * c) v = __ldg(x2 + ((size_t)nn * c + (k - c)) * hw + sp);
      vals[k] = __float2half(v);
    }
    const uint4 v0 = *reinterpret_cast<const uint4*>(vals), z = make_uint4(0u, 0u, 0u, 0u);
    uint4* row = y + (size_t)i * 8;
    row[0] = v0;
#pragma unroll
    for (int q = 1; q < 8; ++q) row[q] = z;
  }
}

// cat([x1,x2],1) + NCHW fp32 -> NHWC fp16 (cpad channels, zero padded). One thread per
// (pixel, 8-channel vector); plane reads are coalesced across pixels.
__global__ void pack_pair_kernel(const float* __restrict__ x1, const float* __restrict__ x2,
                                 uint4* __restrict__ y, int n, int c, int h, int w, int c8,
                                 int c_offset, int zero_fill) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const size_t hw = (size_t)h * w;
  const size_t total = (size_t)n * hw * c8;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    // pixel-fastest mapping inside a vector index so that plane loads coalesce
    const size_t px = i % ((size_t)n * hw);
    const int cv = (int)(i / ((size_t)n * hw));
    const int nn = (int)(px / hw);
    const size_t sp = px % hw;
    __align__(16) __half vals[8];
    bool any = false;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int ch = cv * 8 + k - c_offset;
      float v = 0.f;
      if (ch >= 0 && ch < c) { v = __ldg(x1 + ((size_t)nn * c + ch) * hw + sp); any = true; }
      else if (x2 != nullptr && ch >= c && ch < 2 * c) {
        v = __ldg(x2 + ((size_t)nn * c + (ch - c)) * hw + sp); any = true;
      }
      vals[k] = __float2half(v);
    }
    if (any || zero_fill) y[px * c8 + cv] = *reinterpret_cast<const uint4*>(vals);
  }
}

__global__ void nhwc_to_nchw_kernel(const __half* __restrict__ x, float* __restrict__ y, int n,
                                    int c, int h, int w, int cpad) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const size_t hw = (size_t)h * w;
  const size_t total = (size_t)n * c * hw;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const size_t sp = i % hw;
    const int ch = (int)((i / hw) % c);
    const int nn = (int)(i / (hw * c));
    y[i] = __half2float(x[((size_t)nn * hw + sp) * cpad + ch]);
  }
}

// =====================================================================================
// module-boundary NCHW fp32 ops
// =====================================================================================
__global__ void backward_warp_kernel(const float* __restrict__ x, const float* __restrict__ flow,
                                     float* __restrict__ y, int n, int c, int h, int w) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const size_t hw = (size_t)h * w;
  const size_t total = (size_t)n * hw;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int nn = (int)(i / hw);
    const size_t sp = i % hw;
    const int yy = (int)(sp / w), xx = (int)(sp % w);
    const float fx = (float)xx + __ldg(flow + ((size_t)nn * 2 + 0) * hw + sp);
    const float fy = (float)yy + __ldg(flow + ((size_t)nn * 2 + 1) * hw + sp);
    for (int k = 0; k < c; ++k)
      y[((size_t)nn * c + k) * hw + sp] = bilerp_border(x + ((size_t)nn * c + k) * hw, h, w, fx, fy);
  }
}

__global__ void space_to_depth_kernel(const float* __restrict__ x, float* __restrict__ y, int n,
                                      int c, int h, int w, int s) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int oh = h / s, ow = w / s;
  const size_t total = (size_t)n * c * s * s * oh * ow;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    size_t p = i;
    const int xo = (int)(p % ow); p /= ow;
    const int yo = (int)(p % oh); p /= oh;
    const int oc = (int)(p % (c * s * s));
    const int nn = (int)(p / (c * s * s));
    const int k = oc % c, blk = oc / c, sy = blk / s, sx = blk % s;
    y[i] = __ldg(x + (((size_t)nn * c + k) * h + (yo * s + sy)) * w + (xo * s + sx));
  }
}

// y = mul * upsample_func(reflect_pad(x)): one CTA = RY LR rows x 128/S LR pixels of one plane ->
// RY*S HR rows x 128 HR columns; thread t owns HR column X: x-pass of the separable 4-tap filter
// (tg_up_taps) for RY+3 source rows into registers, then RY*S outputs (512-byte coalesced rows).
template <int S, int RY>
__global__ void __launch_bounds__(128)
upsample_nchw_kernel(const float* __restrict__ x, float* __restrict__ y, int hin, int win, int h,
                     int w, int up_mode, float mul, int accumulate) {
  tg_pdl_wait();
  tg_pdl_trigger();
  constexpr int LRW = 128 / S;
  constexpr int FW = LRW + 3, FH = RY + 3;
  __shared__ float fsrc[FH * FW];
  const int t = threadIdx.x;
  const int x0 = blockIdx.x * LRW, y0 = blockIdx.y * RY;
  const size_t pl = blockIdx.z;
  const float* src = x + pl * hin * win;
  for (int i = t; i < FH * FW; i += 128) {
    const int col = i % FW, row = i / FW;
    const int yy = tg_reflect_hi(tg_clampi(y0 - 1 + row, 0, h - 1), hin);
    const int xx = tg_reflect_hi(tg_clampi(x0 - 1 + col, 0, w - 1), win);
    fsrc[i] = __ldg(src + (size_t)yy * win + xx);
  }
  __syncthreads();
  const int X = x0 * S + t;
  if (X >= w * S) return;
  float kx[4], hx[FH];
  tg_up_taps(up_mode, t % S, S, kx);
#pragma unroll
  for (int row = 0; row < FH; ++row) {
    const float* f = fsrc + row * FW + t / S;
    hx[row] = kx[0] * f[0] + kx[1] * f[1] + kx[2] * f[2] + kx[3] * f[3];
  }
  float* dst = y + (pl * h * S + (size_t)y0 * S) * ((size_t)w * S) + X;
#pragma unroll
  for (int ry = 0; ry < RY; ++ry) {
    if (y0 + ry >= h) break;
#pragma unroll
    for (int sy = 0; sy < S; ++sy) {
      float ky[4];
      tg_up_taps(up_mode, sy, S, ky);
      float* o = dst + (size_t)(ry * S + sy) * ((size_t)w * S);
      const float up = mul * (ky[0] * hx[ry] + ky[1] * hx[ry + 1] + ky[2] * hx[ry + 2] + ky[3] * hx[ry + 3]);
      *o = accumulate ? *o + up : up;
    }
  }
}

// float32_to_uint8 + CHW->HWC: uint8(clip(rint(x*255),0,255)), rint = round-half-even
__device__ __forceinline__ uint32_t tg_q8(float v) {
  return (uint32_t)fminf(fmaxf(rintf(v * 255.f), 0.f), 255.f);
}
__global__ void to_uint8_kernel(const float* __restrict__ x, uint8_t* __restrict__ y, int n, int c,
                                int h, int w) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const size_t hw = (size_t)h * w;
  const size_t total = (size_t)n * hw;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int nn = (int)(i / hw);
    const size_t sp = i % hw;
    for (int k = 0; k < c; ++k) y[i * c + k] = (uint8_t)tg_q8(__ldg(x + ((size_t)nn * c + k) * hw + sp));
  }
}
// c == 3, hw % 4 == 0: one thread = 4 pixels = three float4 loads -> 12 bytes = three u32 stores
__global__ void to_uint8_c3x4_kernel(const float4* __restrict__ x, uint32_t* __restrict__ y, int n,
                                     size_t hw4) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const size_t total = (size_t)n * hw4;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const size_t nn = i / hw4, sp = i % hw4;
    const float4 r = __ldg(x + (nn * 3 + 0) * hw4 + sp);
    const float4 g = __ldg(x + (nn * 3 + 1) * hw4 + sp);
    const float4 b = __ldg(x + (nn * 3 + 2) * hw4 + sp);
    // bytes: r0 g0 b0 r1 | g1 b1 r2 g2 | b2 r3 g3 b3
    const uint32_t w0 = tg_q8(r.x) | (tg_q8(g.x) << 8) | (tg_q8(b.x) << 16) | (tg_q8(r.y) << 24);
    const uint32_t w1 = tg_q8(g.y) | (tg_q8(b.y) << 8) | (tg_q8(r.z) << 16) | (tg_q8(g.z) << 24);
    const uint32_t w2 = tg_q8(b.z) | (tg_q8(r.w) << 8) | (tg_q8(g.w) << 16) | (tg_q8(b.w) << 24);
    uint32_t* o = y + i * 3;
    o[0] = w0; o[1] = w1; o[2] = w2;
  }
}

// Gaussian blur + subsample of the BD degradation (data_utils.py:30-53).  One CTA = 32 x 8 outputs:
// the (7s+k) x (31s+k) input patch (reflect-padded when pad_data) is staged in shared memory once,
// every thread then accumulates its k*k taps from it.
__global__ void __launch_bounds__(256)
downsample_bd_kernel(const float* __restrict__ x, const float* __restrict__ k2d, float* __restrict__ y,
                     int H, int W, int oh, int ow, int k, int s, int pad) {
  tg_pdl_wait();
  tg_pdl_trigger();
  extern __shared__ float bd_smem[];
  const int tw = 31 * s + k, th = 7 * s + k;
  float* taps = bd_smem;                 // [k*k]
  float* tile = bd_smem + k * k;         // [th][tw]
  const int plane = blockIdx.z;
  const int ox0 = blockIdx.x * 32, oy0 = blockIdx.y * 8;
  const float* xp = x + (size_t)plane * H * W;
  for (int i = threadIdx.x; i < k * k; i += 256) taps[i] = __ldg(k2d + i);
  for (int i = threadIdx.x; i < th * tw; i += 256) {
    const int ty = i / tw, tx = i - ty * tw;
    int iy = oy0 * s + ty - pad, ix = ox0 * s + tx - pad;
    // F.pad(..., 'reflect'): -i -> i, H-1+i -> H-1-i; positions beyond what any valid output of
    // this tile needs are clamped (never used)
    iy = iy < 0 ? -iy : (iy >= H ? 2 * (H - 1) - iy : iy);
    ix = ix < 0 ? -ix : (ix >= W ? 2 * (W - 1) - ix : ix);
    iy = tg_clampi(iy, 0, H - 1);
    ix = tg_clampi(ix, 0, W - 1);
    tile[i] = __ldg(xp + (size_t)iy * W + ix);
  }
  __syncthreads();
  const int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;
  const int ox = ox0 + lx, oy = oy0 + ly;
  if (ox >= ow || oy >= oh) return;
  float acc = 0.f;
  const float* t0 = tile + (ly * s) * tw + lx * s;
  for (int i = 0; i < k; ++i)
    for (int j = 0; j < k; ++j) acc += taps[i * k + j] * t0[i * tw + j];
  y[((size_t)plane * oh + oy) * ow + ox] = acc;
}

}  // namespace
cudaError_t tg_warp_w_launch(const float* hr_prev, const float* flow, const float* lr_curr, __half* out, int n, int h,
                             int w, int h8, int w8, int s, int fm, int cpad, cudaStream_t st);   // tg_warp_w.cu
namespace {

inline int grid_for(size_t total, int block) {
  size_t g = (total + block - 1) / block;
  const size_t cap = (size_t)tg_sms() * 32;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace

// =====================================================================================
// C ABI
// =====================================================================================
extern "C" {

static int warp_launch(const float* hr_prev, const float* flow, const float* lr_curr, void* out,
                       int n, int c, int h, int w, int h8, int w8, int s, int up_mode, int cpad,
                       bool lrflow, void* stream) {
  TG_REQUIRE(hr_prev && flow && lr_curr && out, TG_E_INVALID, "warp_s2d_concat: null pointer");
  TG_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0, TG_E_INVALID, "warp_s2d_concat: bad size");
  TG_REQUIRE(s == 2 || s == 4, TG_E_UNSUPPORTED, "warp_s2d_concat: scale %d (2 or 4)", s);
  TG_REQUIRE(cpad % 8 == 0 && (s * s + 1) * c <= cpad, TG_E_UNSUPPORTED,
             "warp_s2d_concat: (s*s+1)*c=%d does not fit cpad=%d", (s * s + 1) * c, cpad);
  TG_REQUIRE(n <= 65535 && h <= 65535, TG_E_UNSUPPORTED, "warp_s2d_concat: grid too large");
  if (lrflow) {
    TG_REQUIRE(h8 > 0 && w8 > 0 && h8 <= h && w8 <= w && (h - h8) < h8 && (w - w8) < w8,
               TG_E_INVALID, "warp_s2d_concat: bad reflect pad %dx%d -> %dx%d", h8, w8, h, w);
    TG_REQUIRE(up_mode == TG_UP_BICUBIC || up_mode == TG_UP_BILINEAR, TG_E_INVALID,
               "warp_s2d_concat: up_mode");
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int lrw = 128 / s;
  constexpr int RY = 2;
  dim3 grid(tg_ceil_div(w, lrw), tg_ceil_div(h, RY), n);
  const size_t smem = (size_t)lrw * (cpad + 8) * sizeof(__half);   // tile pixel stride = cpad*2 + 16 bytes
  __half* o = (__half*)out;
  TG_REQUIRE(s * h >= 2 && s * w >= 2, TG_E_UNSUPPORTED, "warp_s2d_concat: HR image smaller than 2x2");
  const int fm = !lrflow ? 0 : (up_mode == TG_UP_BICUBIC ? 1 : 2);
  // default: the warp-autonomous kernel (tg_warp_w.cu); TG_WARP_KERNEL=cta selects the CTA-lock-step one
  static int use_cta = -1;
  if (use_cta < 0) { const char* e = getenv("TG_WARP_KERNEL"); use_cta = (e && e[0] == 'c') ? 1 : 0; }
  if (c == 3 && !use_cta) {
    cudaError_t le = tg_warp_w_launch(hr_prev, flow, lr_curr, o, n, h, w, h8, w8, s, fm, cpad, st);
    TG_REQUIRE(le == cudaSuccess, (int)le, "warp_s2d_concat: launch failed: %s", cudaGetErrorString(le));
    TG_CUDA_LAUNCH_CHECK("warp_s2d_concat");
    return TG_OK;
  }
  // Default: all S HR rows of an LR row per pass (12*S gathers in flight per thread, 5 CTAs/SM).
  // TG_WARP_SP=2: two rows per pass at <= 64 registers (8 CTAs/SM), for A/B measurements.
  static int sp_full = -1;
  if (sp_full < 0) { const char* e = getenv("TG_WARP_SP"); sp_full = (e && e[0] == '2') ? 0 : 1; }
#define TG_WARP_LAUNCH(SS, FM)                                                                                 \
  do {                                                                                                         \
    if (sp_full) tg_launch(warp_s2d_concat_kernel<SS, FM, RY, SS>, dim3(grid), dim3(128), smem, st, hr_prev,    \
                           flow, lr_curr, o, c, h, w, h8, w8, cpad);                                           \
    else tg_launch(warp_s2d_concat_kernel<SS, FM, RY, 2>, dim3(grid), dim3(128), smem, st, hr_prev, flow,       \
                   lr_curr, o, c, h, w, h8, w8, cpad);                                                         \
  } while (0)
  if (s == 4) {
    if (fm == 0) TG_WARP_LAUNCH(4, 0); else if (fm == 1) TG_WARP_LAUNCH(4, 1); else TG_WARP_LAUNCH(4, 2);
  } else {
    if (fm == 0) TG_WARP_LAUNCH(2, 0); else if (fm == 1) TG_WARP_LAUNCH(2, 1); else TG_WARP_LAUNCH(2, 2);
  }
#undef TG_WARP_LAUNCH
  TG_CUDA_LAUNCH_CHECK("warp_s2d_concat");
  return TG_OK;
}

int tg_warp_s2d_concat_hrflow(const float* hr_prev, const float* hr_flow, const float* lr_curr,
                              void* out, int n, int c, int h, int w, int s, int cpad,
                              void* stream) {
  return warp_launch(hr_prev, hr_flow, lr_curr, out, n, c, h, w, 0, 0, s, 0, cpad, false, stream);
}

int tg_warp_s2d_concat_lrflow(const float* hr_prev, const float* lr_flow, const float* lr_curr,
                              void* out, int n, int c, int h, int w, int h8, int w8, int s,
                              int up_mode, int cpad, void* stream) {
  return warp_launch(hr_prev, lr_flow, lr_curr, out, n, c, h, w, h8, w8, s, up_mode, cpad, true,
                     stream);
}

int tg_downsample_bd_nchw_f32(const float* x, const float* k2d, float* y, int n, int c, int H, int W,
                              int k, int s, int pad_data, void* stream) {
  TG_REQUIRE(x && k2d && y, TG_E_INVALID, "downsample_bd: null pointer");
  TG_REQUIRE(n > 0 && c > 0 && H > 0 && W > 0 && k >= 1 && s >= 1, TG_E_INVALID, "downsample_bd: bad size");
  TG_REQUIRE(k <= 31 && s <= 8, TG_E_UNSUPPORTED, "downsample_bd: kernel %d / stride %d too large", k, s);
  const int pad = pad_data ? (k - 1) / 2 : 0;
  const int Hp = H + (pad_data ? k - 1 : 0), Wp = W + (pad_data ? k - 1 : 0);
  TG_REQUIRE(Hp >= k && Wp >= k, TG_E_INVALID, "downsample_bd: image smaller than the kernel");
  TG_REQUIRE(!pad_data || (k - 1 - pad < H && k - 1 - pad < W), TG_E_INVALID,
             "downsample_bd: reflect padding needs pad < size");
  const int oh = (Hp - k) / s + 1, ow = (Wp - k) / s + 1;
  TG_REQUIRE((size_t)n * c <= 65535, TG_E_UNSUPPORTED, "downsample_bd: n*c too large");
  const size_t smem = ((size_t)k * k + (size_t)(7 * s + k) * (31 * s + k)) * sizeof(float);
  static TgPerDeviceOnce attr_once;
  attr_once.run([] {
    return cudaFuncSetAttribute(downsample_bd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
  });
  TG_REQUIRE(smem <= 160 * 1024, TG_E_UNSUPPORTED, "downsample_bd: tile does not fit in shared memory");
  dim3 grid(tg_ceil_div(ow, 32), tg_ceil_div(oh, 8), n * c);
  tg_launch(downsample_bd_kernel, grid, dim3(256), smem, (cudaStream_t)stream, x, k2d, y, H, W, oh, ow, k, s, pad);
  TG_CUDA_LAUNCH_CHECK("downsample_bd");
  return TG_OK;
}

int tg_maxpool2x2_nhwc_f16(const void* x, void* y, int n, int h, int w, int c, void* stream) {
  TG_REQUIRE(x && y, TG_E_INVALID, "maxpool2x2: null pointer");
  TG_REQUIRE(n > 0 && h >= 2 && w >= 2 && c > 0 && c % 8 == 0, TG_E_INVALID,
             "maxpool2x2: bad shape n=%d h=%d w=%d c=%d", n, h, w, c);
  const size_t total = (size_t)n * (h / 2) * (w / 2) * (c / 8);
  tg_launch(maxpool2x2_kernel, dim3(grid_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, (const uint4*)x, (uint4*)y, n, h, w, c / 8);
  TG_CUDA_LAUNCH_CHECK("maxpool2x2");
  return TG_OK;
}

int tg_upsample2x_bilinear_nhwc_f16(const void* x, void* y, int n, int h, int w, int c,
                                    void* stream) {
  TG_REQUIRE(x && y, TG_E_INVALID, "upsample2x: null pointer");
  TG_REQUIRE(n > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0, TG_E_INVALID, "upsample2x: bad shape");
  TG_REQUIRE((size_t)n * h * w * (c / 8) < (size_t)1 << 30, TG_E_UNSUPPORTED, "upsample2x: tensor too large");
  const size_t total = (size_t)n * h * w * (c / 8);    // one thread per input position and 8-channel vector
  tg_launch(upsample2x_kernel, dim3(grid_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, (const uint4*)x, (uint4*)y, n, h, w, c / 8);
  TG_CUDA_LAUNCH_CHECK("upsample2x");
  return TG_OK;
}

int tg_pack_pair_nhwc_f16(const float* x1, const float* x2, void* y, int n, int c, int h, int w,
                          int cpad, void* stream) {
  TG_REQUIRE(x1 && x2 && y, TG_E_INVALID, "pack_pair: null pointer");
  TG_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0 && cpad % 8 == 0 && 2 * c <= cpad, TG_E_INVALID,
             "pack_pair: bad shape");
  if (cpad == 64 && 2 * c <= 8 && (size_t)n * h * w < (size_t)1 << 30 && ((uintptr_t)y & 31) == 0) {
    tg_launch(pack_pair_c64_kernel, dim3(grid_for((size_t)n * h * w, 256)), dim3(256), 0, (cudaStream_t)stream, x1, x2, (uint4*)y, n, c, h * w);
  } else {
    const size_t total = (size_t)n * h * w * (cpad / 8);
    tg_launch(pack_pair_kernel, dim3(grid_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, x1, x2, (uint4*)y, n, c, h, w, cpad / 8, 0, 1);
  }
  TG_CUDA_LAUNCH_CHECK("pack_pair");
  return TG_OK;
}

int tg_nchw_f32_to_nhwc_f16(const float* x, void* y, int n, int c, int h, int w, int cpad,
                            int c_offset, void* stream) {
  TG_REQUIRE(x && y, TG_E_INVALID, "nchw_to_nhwc: null pointer");
  TG_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0 && cpad % 8 == 0 && c_offset >= 0 &&
                 c_offset + c <= cpad, TG_E_INVALID, "nchw_to_nhwc: bad shape");
  // c_offset == 0: writes every channel vector (zero padded); c_offset > 0: only the vectors it
  // touches, which must not be shared with other sources (c_offset % 8 == 0).
  TG_REQUIRE(c_offset % 8 == 0, TG_E_UNSUPPORTED, "nchw_to_nhwc: c_offset must be a multiple of 8");
  const size_t total = (size_t)n * h * w * (cpad / 8);
  tg_launch(pack_pair_kernel, dim3(grid_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, x, nullptr, (uint4*)y, n, c, h, w, cpad / 8, c_offset, c_offset == 0 ? 1 : 0);
  TG_CUDA_LAUNCH_CHECK("nchw_to_nhwc");
  return TG_OK;
}

int tg_nhwc_f16_to_nchw_f32(const void* x, float* y, int n, int c, int h, int w, int cpad,
                            void* stream) {
  TG_REQUIRE(x && y, TG_E_INVALID, "nhwc_to_nchw: null pointer");
  TG_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0 && c <= cpad, TG_E_INVALID, "nhwc_to_nchw: bad shape");
  const size_t total = (size_t)n * c * h * w;
  tg_launch(nhwc_to_nchw_kernel, dim3(grid_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, (const __half*)x, y, n, c, h, w, cpad);
  TG_CUDA_LAUNCH_CHECK("nhwc_to_nchw");
  return TG_OK;
}

int tg_backward_warp_nchw_f32(const float* x, const float* flow, float* y, int n, int c, int h,
                              int w, void* stream) {
  TG_REQUIRE(x && flow && y, TG_E_INVALID, "backward_warp: null pointer");
  TG_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0, TG_E_INVALID, "backward_warp: bad shape");
  const size_t total = (size_t)n * h * w;
  tg_launch(backward_warp_kernel, dim3(grid_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, x, flow, y, n, c, h, w);
  TG_CUDA_LAUNCH_CHECK("backward_warp");
  return TG_OK;
}

int tg_space_to_depth_nchw_f32(const float* x, float* y, int n, int c, int h, int w, int s,
                               void* stream) {
  TG_REQUIRE(x && y, TG_E_INVALID, "space_to_depth: null pointer");
  TG_REQUIRE(n > 0 && c > 0 && s > 0 && h >= s && w >= s, TG_E_INVALID, "space_to_depth: bad shape");
  const size_t total = (size_t)n * c * s * s * (h / s) * (w / s);
  tg_launch(space_to_depth_kernel, dim3(grid_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, x, y, n, c, h, w, s);
  TG_CUDA_LAUNCH_CHECK("space_to_depth");
  return TG_OK;
}

int tg_upsample_nchw_f32(const float* x, float* y, int n, int c, int hin, int win, int h, int w,
                         int s, int up_mode, float mul, int accumulate, void* stream) {
  TG_REQUIRE(x && y, TG_E_INVALID, "upsample: null pointer");
  TG_REQUIRE(n > 0 && c > 0 && hin > 0 && win > 0 && h >= hin && w >= win, TG_E_INVALID,
             "upsample: bad shape");
  TG_REQUIRE((h - hin) < hin && (w - win) < win, TG_E_INVALID, "upsample: reflect pad too large");
  TG_REQUIRE(up_mode == TG_UP_BICUBIC || up_mode == TG_UP_BILINEAR, TG_E_INVALID, "upsample: up_mode");
  TG_REQUIRE(s == 2 || s == 4, TG_E_UNSUPPORTED, "upsample: scale %d (2 or 4)", s);
  TG_REQUIRE(h <= 65535 && (size_t)n * c <= 65535, TG_E_UNSUPPORTED, "upsample: grid too large");
  constexpr int RY = 4;
  dim3 grid(tg_ceil_div(w, 128 / s), tg_ceil_div(h, RY), n * c);
  if (s == 4) tg_launch(upsample_nchw_kernel<4, RY>, dim3(grid), dim3(128), 0, (cudaStream_t)stream, x, y, hin, win, h, w, up_mode, mul, accumulate);
  else        tg_launch(upsample_nchw_kernel<2, RY>, dim3(grid), dim3(128), 0, (cudaStream_t)stream, x, y, hin, win, h, w, up_mode, mul, accumulate);
  TG_CUDA_LAUNCH_CHECK("upsample");
  return TG_OK;
}

int tg_float_to_uint8_nhwc(const float* x, uint8_t* y, int n, int c, int h, int w, void* stream) {
  TG_REQUIRE(x && y, TG_E_INVALID, "float_to_uint8: null pointer");
  TG_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0, TG_E_INVALID, "float_to_uint8: bad shape");
  const size_t total = (size_t)n * h * w;
  if (c == 3 && ((size_t)h * w) % 4 == 0 && ((uintptr_t)x & 15) == 0 && ((uintptr_t)y & 3) == 0)
    tg_launch(to_uint8_c3x4_kernel, dim3(grid_for(total / 4, 256)), dim3(256), 0, (cudaStream_t)stream, (const float4*)x, (uint32_t*)y, n, (size_t)h * w / 4);
  else
    tg_launch(to_uint8_kernel, dim3(grid_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, x, y, n, c, h, w);
  TG_CUDA_LAUNCH_CHECK("float_to_uint8");
  return TG_OK;
}

}  // extern "C"
