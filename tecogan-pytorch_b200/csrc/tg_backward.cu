// Backward (training) kernels of the FRNet generator that are not convolutions: gradients of the
// fused warp + space_to_depth + concat, of backward_warp / upsample_func at the module boundary, of
// FNet's maxpool / x2-bilinear / 24*tanh head, gradient packing with the loss scale, bias gradients.
// Reference: autograd through codes/models/networks/tecogan_nets.py:174-225 (forward_sequence),
// codes/utils/net_utils.py:50-156; call sites cited per entry point in include/tecogan_b200.h.
//
// Precision design (DESIGN.md section 4): activations and their gradients travel between conv
// layers as NHWC fp16; because raw loss gradients are far below the fp16 range (a mean over 1e8
// elements), every fp16 gradient is stored multiplied by a power-of-two LOSS SCALE that lives in
// device memory (`scale[0]` = scale, `scale[1]` = 1/scale, written by tg_grad_scale_from_amax) --
// fp32 results (parameter gradients, flow / state gradients) are multiplied by 1/scale on the way
// out.  No host round trip: the scale is chosen on the device.
#include "tg_common.cuh"

namespace {

inline int bgrid(size_t total, int block) {
  size_t g = (total + block - 1) / block;
  const size_t cap = (size_t)tg_sms() * 32;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// ------------------------------------------------------------------ loss scale
// amax over up to two fp32 tensors (uint compare of |x| bit patterns), then
// scale = 2^floor(log2(target / amax)) clamped to [2^-24, 2^24]; amax == 0 or not finite -> scale 1.
__global__ void amax_kernel(const float* __restrict__ a, size_t na, const float* __restrict__ b, size_t nb,
                            unsigned int* __restrict__ amax_bits) {
  tg_pdl_wait();
  unsigned int m = 0;
  const size_t stride = (size_t)gridDim.x * blockDim.x, i0 = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  for (size_t i = i0; i < na; i += stride) m = max(m, __float_as_uint(a[i]) & 0x7FFFFFFFu);
  if (b != nullptr)
    for (size_t i = i0; i < nb; i += stride) m = max(m, __float_as_uint(b[i]) & 0x7FFFFFFFu);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
  if ((threadIdx.x & 31) == 0 && m != 0) atomicMax(amax_bits, m);
}
__global__ void scale_from_amax_kernel(unsigned int* __restrict__ amax_bits, float target, float* __restrict__ scale) {
  tg_pdl_wait();
  const float amax = __uint_as_float(*amax_bits);
  float s = 1.f;
  if (amax > 0.f && isfinite(amax)) {
    // the exponent exactly, without rounding target / amax or its log2 (floorf(log2f(target / amax)) is one
    // too large when the quotient falls just below a power of two): with amax = ma * 2^ea and
    // target = mt * 2^et, ma and mt in [0.5, 1) (frexpf, exact for denormals too), target / amax =
    // (mt / ma) * 2^(et - ea) with mt / ma in (0.5, 2), below 1 exactly when mt < ma.
    int ea, et;
    const float ma = frexpf(amax, &ea), mt = frexpf(target, &et);
    int e = et - ea - (mt < ma ? 1 : 0);
    e = e < -24 ? -24 : (e > 24 ? 24 : e);
    s = exp2f((float)e);
  }
  scale[0] = s;
  scale[1] = 1.f / s;
  *amax_bits = 0;            // ready for the next use of the workspace
}

// ------------------------------------------------------------------ gradient packing
// g = (a [+ b]) * scale : NCHW fp32 [n,c,h,w] -> NHWC fp16 [n,h,w,cpad] (pad channels zero)
__global__ void grad_pack_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                 const float* __restrict__ scale, uint4* __restrict__ y, int n, int c, int hw, int c8) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const float s = scale ? __ldg(scale) : 1.f;
  const size_t total = (size_t)n * hw * c8;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t px = i % ((size_t)n * hw);          // pixel-fastest inside a vector index: plane loads coalesce
    const int cv = (int)(i / ((size_t)n * hw));
    const int nn = (int)(px / hw);
    const size_t sp = px % hw;
    __align__(16) __half vals[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int ch = cv * 8 + k;
      float v = 0.f;
      if (ch < c) {
        const size_t off = ((size_t)nn * c + ch) * hw + sp;
        v = __ldg(a + off);
        if (b != nullptr) v += __ldg(b + off);
      }
      vals[k] = __float2half(v * s);
    }
    y[px * c8 + cv] = *reinterpret_cast<const uint4*>(vals);
  }
}

// NHWC fp16 [n,h,w,cpad] channels [c0, c0+c) -> NCHW fp32 [n,c,h,w], times inv_scale (accumulate opt.)
__global__ void grad_unpack_kernel(const __half* __restrict__ x, const float* __restrict__ scale,
                                   float* __restrict__ y, int n, int c, int hw, int cpad, int c0, int accumulate) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const float inv = scale ? __ldg(scale + 1) : 1.f;
  const size_t total = (size_t)n * c * hw;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t sp = i % hw;
    const int ch = (int)((i / hw) % c);
    const int nn = (int)(i / ((size_t)hw * c));
    const float v = __half2float(x[((size_t)nn * hw + sp) * cpad + c0 + ch]) * inv;
    y[i] = accumulate ? y[i] + v : v;
  }
}

// ------------------------------------------------------------------ bias gradient
// db[c] += inv_scale * sum over pixels of dz[p][c]; one thread = 8 channels of a strided pixel set,
// block reduction in shared memory, one atomic per channel per block.
__global__ void __launch_bounds__(256)
bias_grad_kernel(const uint4* __restrict__ dz, size_t npix, int c8, int c_real, const float* __restrict__ scale,
                 float* __restrict__ db) {
  tg_pdl_wait();
  tg_pdl_trigger();
  extern __shared__ float red[];                      // [rows][c8*8]
  const int cv = threadIdx.x % c8, row = threadIdx.x / c8, rows = blockDim.x / c8;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (row < rows)
    for (size_t p = (size_t)blockIdx.x * rows + row; p < npix; p += (size_t)gridDim.x * rows) {
      const uint4 v = __ldg(dz + p * c8 + cv);
      const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = __half22float2(h[k]);
        acc[2 * k] += f.x; acc[2 * k + 1] += f.y;
      }
    }
  if (row < rows)
#pragma unroll
    for (int k = 0; k < 8; ++k) red[row * c8 * 8 + cv * 8 + k] = acc[k];
  __syncthreads();
  const float inv = scale ? __ldg(scale + 1) : 1.f;
  for (int ch = threadIdx.x; ch < c8 * 8; ch += blockDim.x) {
    if (ch >= c_real) continue;
    float s = 0.f;
    for (int r = 0; r < rows; ++r) s += red[r * c8 * 8 + ch];
    atomicAdd(db + ch, s * inv);
  }
}

// ------------------------------------------------------------------ warp backward (shared math)
// grid_sample(bilinear, border, align_corners=True) backward as PyTorch computes it
// (grid_sampler_2d_backward): the coordinate gradient is zeroed where the un-clipped coordinate
// lies at or beyond the border (clip_coordinates_set_grad: x <= 0 or x >= size-1 -> 0); corners
// that fall outside contribute nothing (their weight is 0 there anyway).  The reference's
// normalise / un-normalise round trip (net_utils.py:62-72, grid_sample align_corners) has a
// combined derivative of exactly 1.
struct WarpCorners { int xa, ya; float ax, ay; float mx, my; };
__device__ __forceinline__ WarpCorners warp_corners(float fx, float fy, int H, int W) {
  WarpCorners c;
  c.mx = (fx > 0.f && fx < (float)(W - 1)) ? 1.f : 0.f;
  c.my = (fy > 0.f && fy < (float)(H - 1)) ? 1.f : 0.f;
  fx = fminf(fmaxf(fx, 0.f), (float)(W - 1));
  fy = fminf(fmaxf(fy, 0.f), (float)(H - 1));
  c.xa = min((int)floorf(fx), W - 2);
  c.ya = min((int)floorf(fy), H - 2);
  c.ax = fx - (float)c.xa;
  c.ay = fy - (float)c.ya;
  return c;
}

// standalone: x [n,c,h,w], flow [n,2,h,w], gy [n,c,h,w] -> gx (atomic accumulate, caller zeroes) and
// gflow (plain store); either output may be null.
__global__ void backward_warp_bwd_kernel(const float* __restrict__ x, const float* __restrict__ flow,
                                         const float* __restrict__ gy, float* __restrict__ gx,
                                         float* __restrict__ gflow, int n, int c, int h, int w) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const size_t hw = (size_t)h * w;
  const size_t total = (size_t)n * hw;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int nn = (int)(i / hw);
    const size_t sp = i % hw;
    const int yy = (int)(sp / w), xx = (int)(sp % w);
    const float fx = (float)xx + __ldg(flow + ((size_t)nn * 2 + 0) * hw + sp);
    const float fy = (float)yy + __ldg(flow + ((size_t)nn * 2 + 1) * hw + sp);
    const WarpCorners cc = warp_corners(fx, fy, h, w);
    const float w00 = (1.f - cc.ax) * (1.f - cc.ay), w01 = cc.ax * (1.f - cc.ay);
    const float w10 = (1.f - cc.ax) * cc.ay, w11 = cc.ax * cc.ay;
    float gu = 0.f, gv = 0.f;
    for (int k = 0; k < c; ++k) {
      const size_t pl = ((size_t)nn * c + k) * hw;
      const float g = __ldg(gy + pl + sp);
      const size_t o = pl + (size_t)cc.ya * w + cc.xa;
      if (gflow != nullptr) {
        const float v00 = __ldg(x + o), v01 = __ldg(x + o + 1), v10 = __ldg(x + o + w), v11 = __ldg(x + o + w + 1);
        gu += g * ((v01 - v00) * (1.f - cc.ay) + (v11 - v10) * cc.ay);
        gv += g * ((v10 - v00) * (1.f - cc.ax) + (v11 - v01) * cc.ax);
      }
      if (gx != nullptr) {
        if (w00 != 0.f) atomicAdd(gx + o, g * w00);
        if (w01 != 0.f) atomicAdd(gx + o + 1, g * w01);
        if (w10 != 0.f) atomicAdd(gx + o + w, g * w10);
        if (w11 != 0.f) atomicAdd(gx + o + w + 1, g * w11);
      }
    }
    if (gflow != nullptr) {
      gflow[((size_t)nn * 2 + 0) * hw + sp] = gu * cc.mx;
      gflow[((size_t)nn * 2 + 1) * hw + sp] = gv * cc.my;
    }
  }
}

// fused: gradient of warp_s2d_concat (hr flow given).  gx NHWC fp16 [n,h,w,cpad] is the (loss-
// scaled) gradient of the SRNet input: channels [0,C) -> lr_curr, channel C + (sy*S+sx)*C + k ->
// warp(hr_prev)[k, y*S+sy, x*S+sx].  One thread = one HR pixel.
//   d_hr_prev (fp32 NCHW, atomic accumulate)  += inv_scale * g * bilinear weights
//   d_hr_flow (fp32 [n,2,H,W], plain store)    = inv_scale * sum_k g_k * d(sample)/d(coord)
template <int S>
__global__ void warp_s2d_concat_bwd_kernel(const __half* __restrict__ gx, const float* __restrict__ hr_prev,
                                           const float* __restrict__ hr_flow, const float* __restrict__ scale,
                                           float* __restrict__ d_hr_prev, float* __restrict__ d_hr_flow,
                                           int n, int C, int h, int w, int cpad) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int H = h * S, W = w * S;
  const size_t HW = (size_t)H * W;
  const size_t total = (size_t)n * HW;
  const float inv = scale ? __ldg(scale + 1) : 1.f;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int nn = (int)(i / HW);
    const size_t sp = i % HW;
    const int Y = (int)(sp / W), X = (int)(sp % W);
    const int y = Y / S, sy = Y - y * S, x = X / S, sx = X - x * S;
    const float fx = (float)X + __ldg(hr_flow + ((size_t)nn * 2 + 0) * HW + sp);
    const float fy = (float)Y + __ldg(hr_flow + ((size_t)nn * 2 + 1) * HW + sp);
    const WarpCorners cc = warp_corners(fx, fy, H, W);
    const float w00 = (1.f - cc.ax) * (1.f - cc.ay), w01 = cc.ax * (1.f - cc.ay);
    const float w10 = (1.f - cc.ax) * cc.ay, w11 = cc.ax * cc.ay;
    const __half* gp = gx + (((size_t)nn * h + y) * w + x) * cpad + C + (sy * S + sx) * C;
    float gu = 0.f, gv = 0.f;
    for (int k = 0; k < C; ++k) {
      const float g = __half2float(gp[k]) * inv;
      const size_t o = ((size_t)nn * C + k) * HW + (size_t)cc.ya * W + cc.xa;
      const float v00 = __ldg(hr_prev + o), v01 = __ldg(hr_prev + o + 1);
      const float v10 = __ldg(hr_prev + o + W), v11 = __ldg(hr_prev + o + W + 1);
      gu += g * ((v01 - v00) * (1.f - cc.ay) + (v11 - v10) * cc.ay);
      gv += g * ((v10 - v00) * (1.f - cc.ax) + (v11 - v01) * cc.ax);
      if (d_hr_prev != nullptr && g != 0.f) {
        if (w00 != 0.f) atomicAdd(d_hr_prev + o, g * w00);
        if (w01 != 0.f) atomicAdd(d_hr_prev + o + 1, g * w01);
        if (w10 != 0.f) atomicAdd(d_hr_prev + o + W, g * w10);
        if (w11 != 0.f) atomicAdd(d_hr_prev + o + W + 1, g * w11);
      }
    }
    if (d_hr_flow != nullptr) {
      d_hr_flow[((size_t)nn * 2 + 0) * HW + sp] = gu * cc.mx;
      d_hr_flow[((size_t)nn * 2 + 1) * HW + sp] = gv * cc.my;
    }
  }
}

// ------------------------------------------------------------------ upsample_func backward
// y = mul * upsample(x) with the separable 4-tap filter of tg_up_taps over clamped source indices
// (bicubic: BicubicUpsampler, bilinear: F.interpolate align_corners=False).  Transposed filter as a
// gather: gx[y][x] = mul * sum_{Y,X} gy[Y][X] * wy(Y->y) * wx(X->x), where wy(Y->y) = sum_i ky_{Y%S}[i]
// * [clamp(Y/S - 1 + i) == y].  One CTA = TY x TX LR outputs of one plane: the HR gradient patch
// ((TY+3)*S x (TX+3)*S, rows/cols that can reach the tile) is staged in shared memory, reduced along
// x into [(TY+3)*S][TX], then along y.
template <int S>
__global__ void __launch_bounds__(256)
upsample_bwd_kernel(const float* __restrict__ gy, float* __restrict__ gx, int h, int w, int up_mode, float mul,
                    int accumulate) {
  tg_pdl_wait();
  tg_pdl_trigger();
  constexpr int TY = 8, TX = 32;
  constexpr int PH = (TY + 3) * S, PW = (TX + 3) * S;       // source rows y0-2 .. y0+TY (LR units), times S
  __shared__ float patch[PH][PW + 1];
  __shared__ float rowred[PH][TX + 1];
  const int x0 = blockIdx.x * TX, y0 = blockIdx.y * TY;
  const size_t pl = blockIdx.z;
  const int H = h * S, W = w * S;
  const float* src = gy + pl * (size_t)H * W;
  // HR rows/cols that can contribute to LR index t: LR source cells t-2 .. t+1 (cell c uses taps c-1..c+2)
  const int Y0 = (y0 - 2) * S, X0 = (x0 - 2) * S;
  for (int i = threadIdx.x; i < PH * PW; i += 256) {
    const int r = i / PW, c = i - r * PW;
    const int Y = Y0 + r, X = X0 + c;
    patch[r][c] = (Y >= 0 && Y < H && X >= 0 && X < W) ? __ldg(src + (size_t)Y * W + X) : 0.f;
  }
  __syncthreads();
  // x pass: rowred[r][tx] = sum over patch columns of patch[r][c] * wx(X -> x0+tx)
  for (int i = threadIdx.x; i < PH * TX; i += 256) {
    const int r = i / TX, tx = i - r * TX;
    const int xo = x0 + tx;
    float acc = 0.f;
    if (xo < w) {
#pragma unroll
      for (int cell = -2; cell <= 1; ++cell) {       // LR cell xc = xo + cell, its HR columns xc*S + d
        const int xc = xo + cell;
        if (xc < 0 || xc >= w) continue;
#pragma unroll
        for (int d = 0; d < S; ++d) {
          float k[4];
          tg_up_taps(up_mode, d, S, k);
          float wsum = 0.f;
#pragma unroll
          for (int t = 0; t < 4; ++t)
            if (tg_clampi(xc - 1 + t, 0, w - 1) == xo) wsum += k[t];
          acc += wsum * patch[r][(xc - (x0 - 2)) * S + d];
        }
      }
    }
    rowred[r][tx] = acc;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < TY * TX; i += 256) {
    const int ty = i / TX, tx = i - ty * TX;
    const int yo = y0 + ty, xo = x0 + tx;
    if (yo >= h || xo >= w) continue;
    float acc = 0.f;
#pragma unroll
    for (int cell = -2; cell <= 1; ++cell) {
      const int yc = yo + cell;
      if (yc < 0 || yc >= h) continue;
#pragma unroll
      for (int d = 0; d < S; ++d) {
        float k[4];
        tg_up_taps(up_mode, d, S, k);
        float wsum = 0.f;
#pragma unroll
        for (int t = 0; t < 4; ++t)
          if (tg_clampi(yc - 1 + t, 0, h - 1) == yo) wsum += k[t];
        acc += wsum * rowred[(yc - (y0 - 2)) * S + d][tx];
      }
    }
    float* o = gx + pl * (size_t)h * w + (size_t)yo * w + xo;
    *o = accumulate ? *o + mul * acc : mul * acc;
  }
}

// ------------------------------------------------------------------ FNet helpers, backward (NHWC fp16)
// slope of LeakyReLU(0.2) / ReLU / identity from the STORED forward output v (sign(v) == sign(pre-act))
__device__ __forceinline__ float dact_from_out(float v, int act) {
  return act == TG_ACT_NONE ? 1.f : (v > 0.f ? 1.f : (act == TG_ACT_RELU ? 0.f : 0.2f));
}

// maxpool 2x2 backward fused with the activation derivative of the pooled layer's own output x:
// gx[2y+a][2x+b] = (first position of the window, row-major, where x == y) ? gy[y][x] * act'(x) : 0;
// rows / columns beyond 2*(h/2) (odd sizes) receive 0.  One thread = one output window, 8 channels.
__global__ void maxpool2x2_bwd_kernel(const uint4* __restrict__ x, const uint4* __restrict__ gy,
                                      uint4* __restrict__ gx, int n, int h, int w, int c8, int act) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int ho = (h + 1) / 2, wo = (w + 1) / 2;            // windows incl. the ragged last row / column
  const int hp = h / 2, wp = w / 2;
  const size_t total = (size_t)n * ho * wo * c8;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % c8);
    size_t p = i / c8;
    const int xo = (int)(p % wo); p /= wo;
    const int yo = (int)(p % ho);
    const int nn = (int)(p / ho);
    const bool pooled = yo < hp && xo < wp;
    uint4 g = make_uint4(0u, 0u, 0u, 0u);
    if (pooled) g = __ldg(gy + (((size_t)nn * hp + yo) * wp + xo) * c8 + cv);
    const __half* gh = reinterpret_cast<const __half*>(&g);
    uint4 v[4];
    bool valid[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int yy = 2 * yo + (q >> 1), xx = 2 * xo + (q & 1);
      valid[q] = yy < h && xx < w;
      v[q] = valid[q] ? __ldg(x + (((size_t)nn * h + yy) * w + xx) * c8 + cv) : make_uint4(0u, 0u, 0u, 0u);
    }
    uint4 o[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) o[q] = make_uint4(0u, 0u, 0u, 0u);
    if (pooled) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        float xv[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) xv[q] = __half2float(reinterpret_cast<const __half*>(&v[q])[k]);
        const float m = fmaxf(fmaxf(xv[0], xv[1]), fmaxf(xv[2], xv[3]));
        int arg = 3;
#pragma unroll
        for (int q = 3; q >= 0; --q) if (xv[q] == m) arg = q;      // first maximum in row-major order
        const float gval = __half2float(gh[k]) * dact_from_out(xv[arg], act);
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (q == arg) reinterpret_cast<__half*>(&o[q])[k] = __float2half(gval);
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int yy = 2 * yo + (q >> 1), xx = 2 * xo + (q & 1);
      if (valid[q]) gx[(((size_t)nn * h + yy) * w + xx) * c8 + cv] = o[q];
    }
  }
}

// x2 bilinear (align_corners=False) backward fused with the activation derivative of the layer that
// produced the upsampled map (its stored output m):  forward out[2i] = .25*in[max(i-1,0)] + .75*in[i],
// out[2i+1] = .75*in[i] + .25*in[min(i+1,L-1)]  ->  din[i] = .75*(g[2i] + g[2i+1]) + .25*g[2i+2]
// (i+1 <= L-1) + .25*g[2i-1] (i >= 1) + .25*g[0] (i == 0) + .25*g[2L-1] (i == L-1); separable.
__device__ __forceinline__ void up2_bwd_taps(int i, int L, int idx[4], float wgt[4]) {
  idx[0] = 2 * i - 1; wgt[0] = i >= 1 ? 0.25f : 0.f;
  idx[1] = 2 * i;     wgt[1] = i == 0 ? 1.0f : 0.75f;        // .75 + the clamped .25 of out[0]
  idx[2] = 2 * i + 1; wgt[2] = i == L - 1 ? 1.0f : 0.75f;    // .75 + the clamped .25 of out[2L-1]
  idx[3] = 2 * i + 2; wgt[3] = i + 1 <= L - 1 ? 0.25f : 0.f;
  if (idx[0] < 0) idx[0] = 0;
  if (idx[3] > 2 * L - 1) idx[3] = 2 * L - 1;
}
__global__ void __launch_bounds__(256)
upsample2x_bwd_kernel(const uint4* __restrict__ gy, const uint4* __restrict__ m, uint4* __restrict__ gx, int n,
                      int h, int w, int c8, int act) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const size_t total = (size_t)n * h * w * c8;
  const int wo = 2 * w, hh = 2 * h;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int cv = (int)(i % c8);
    size_t p = i / c8;
    const int xi = (int)(p % w); p /= w;
    const int yi = (int)(p % h);
    const int nn = (int)(p / h);
    int iy[4], ix[4];
    float wy[4], wx[4];
    up2_bwd_taps(yi, h, iy, wy);
    up2_bwd_taps(xi, w, ix, wx);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      if (wy[a] == 0.f) continue;
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        if (wx[b] == 0.f) continue;
        const uint4 g = __ldg(gy + (((size_t)nn * hh + iy[a]) * wo + ix[b]) * c8 + cv);
        const __half2* gh = reinterpret_cast<const __half2*>(&g);
        const float ww = wy[a] * wx[b];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = __half22float2(gh[k]);
          acc[2 * k] += ww * f.x; acc[2 * k + 1] += ww * f.y;
        }
      }
    }
    const uint4 mv = __ldg(m + i);
    const __half* mh = reinterpret_cast<const __half*>(&mv);
    __align__(16) __half o[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = __float2half(acc[k] * dact_from_out(__half2float(mh[k]), act));
    gx[i] = *reinterpret_cast<const uint4*>(o);
  }
}

// flow head: flow = 24*tanh(z)  ->  dz = dflow * (24 - flow^2/24) * scale ; NCHW fp32 [n,2,h,w] ->
// NHWC fp16 [n,h,w,cpad] (channels >= 2 zero)
__global__ void flow_head_bwd_kernel(const float* __restrict__ gflow, const float* __restrict__ gflow2,
                                     const float* __restrict__ flow, const float* __restrict__ scale,
                                     uint4* __restrict__ dz, int n, int hw, int c8) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const float s = scale ? __ldg(scale) : 1.f;
  const size_t total = (size_t)n * hw;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int nn = (int)(i / hw);
    const size_t sp = i % hw;
    __align__(16) __half vals[8] = {};
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const size_t off = ((size_t)nn * 2 + k) * hw + sp;
      const float f = __ldg(flow + off);
      float g = __ldg(gflow + off);
      if (gflow2 != nullptr) g += __ldg(gflow2 + off);
      vals[k] = __float2half(g * (24.f - f * f * (1.f / 24.f)) * s);
    }
    dz[i * c8] = *reinterpret_cast<const uint4*>(vals);
    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
    for (int q = 1; q < c8; ++q) dz[i * c8 + q] = z;
  }
}

// amax of the flow-head gradient AFTER the tanh derivative (what actually enters the fp16 path)
__global__ void flow_head_amax_kernel(const float* __restrict__ gflow, const float* __restrict__ gflow2,
                                      const float* __restrict__ flow, size_t total, unsigned int* __restrict__ amax_bits) {
  tg_pdl_wait();
  unsigned int m = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const float f = __ldg(flow + i);
    float g = __ldg(gflow + i);
    if (gflow2 != nullptr) g += __ldg(gflow2 + i);
    m = max(m, __float_as_uint(g * (24.f - f * f * (1.f / 24.f))) & 0x7FFFFFFFu);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
  if ((threadIdx.x & 31) == 0 && m != 0) atomicMax(amax_bits, m);
}

// space_to_depth backward = depth_to_space: gy [n,c*s*s,oh,ow] -> gx [n,c,oh*s,ow*s]
__global__ void depth_to_space_kernel(const float* __restrict__ gy, float* __restrict__ gx, int n, int c, int h,
                                      int w, int s) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int oh = h / s, ow = w / s;
  const size_t total = (size_t)n * c * h * w;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    size_t p = i;
    const int xx = (int)(p % w); p /= w;
    const int yy = (int)(p % h); p /= h;
    const int k = (int)(p % c);
    const int nn = (int)(p / c);
    const int yo = yy / s, sy = yy - yo * s, xo = xx / s, sx = xx - xo * s;
    const bool in = yo < oh && xo < ow;
    gx[i] = in ? __ldg(gy + (((size_t)nn * c * s * s + (sy * s + sx) * c + k) * oh + yo) * ow + xo) : 0.f;
  }
}

}  // namespace

// =====================================================================================
// C ABI
// =====================================================================================
extern "C" {

size_t tg_grad_scale_workspace_bytes(void) { return 16; }   // [0,8) scale, 1/scale (fp32); [8,12) amax bits

int tg_grad_scale_from_amax(const float* a, size_t na, const float* b, size_t nb, float target, void* ws,
                            void* stream) {
  TG_REQUIRE(a && ws && na > 0, TG_E_INVALID, "grad_scale: null pointer / empty tensor");
  TG_REQUIRE(target > 0.f, TG_E_INVALID, "grad_scale: target must be positive");
  TG_REQUIRE(((uintptr_t)ws & 15) == 0, TG_E_INVALID, "grad_scale: workspace must be 16-byte aligned");
  float* scale = reinterpret_cast<float*>(ws);
  unsigned int* bits = reinterpret_cast<unsigned int*>(ws) + 2;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t tot = na > nb ? na : nb;
  tg_launch(amax_kernel, dim3(bgrid(tot, 256)), dim3(256), 0, st, a, na, b, (size_t)(b ? nb : 0), bits);
  TG_CUDA_LAUNCH_CHECK("grad_amax");
  tg_launch(scale_from_amax_kernel, dim3(1), dim3(1), 0, st, bits, target, scale);
  TG_CUDA_LAUNCH_CHECK("grad_scale");
  return TG_OK;
}

int tg_grad_pack_nhwc_f16(const float* a, const float* b, const float* scale, void* y, int n, int c, int h, int w,
                          int cpad, void* stream) {
  TG_REQUIRE(a && y, TG_E_INVALID, "grad_pack: null pointer");
  TG_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0 && cpad % 8 == 0 && c <= cpad, TG_E_INVALID, "grad_pack: bad shape");
  const size_t total = (size_t)n * h * w * (cpad / 8);
  tg_launch(grad_pack_kernel, dim3(bgrid(total, 256)), dim3(256), 0, (cudaStream_t)stream, a, b, scale, (uint4*)y, n,
            c, h * w, cpad / 8);
  TG_CUDA_LAUNCH_CHECK("grad_pack");
  return TG_OK;
}

int tg_grad_unpack_nchw_f32(const void* x, const float* scale, float* y, int n, int c, int h, int w, int cpad,
                            int c_offset, int accumulate, void* stream) {
  TG_REQUIRE(x && y, TG_E_INVALID, "grad_unpack: null pointer");
  TG_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0 && c_offset >= 0 && c_offset + c <= cpad, TG_E_INVALID,
             "grad_unpack: bad shape");
  const size_t total = (size_t)n * c * h * w;
  tg_launch(grad_unpack_kernel, dim3(bgrid(total, 256)), dim3(256), 0, (cudaStream_t)stream, (const __half*)x, scale, y,
            n, c, h * w, cpad, c_offset, accumulate);
  TG_CUDA_LAUNCH_CHECK("grad_unpack");
  return TG_OK;
}

int tg_bias_grad_nhwc_f16(const void* dz, size_t npix, int c, int c_real, const float* scale, float* db,
                          void* stream) {
  TG_REQUIRE(dz && db && npix > 0, TG_E_INVALID, "bias_grad: null pointer");
  TG_REQUIRE(c > 0 && c % 8 == 0 && c <= 256 && c_real > 0 && c_real <= c, TG_E_UNSUPPORTED, "bias_grad: c=%d", c);
  const int c8 = c / 8, rows = 256 / c8;
  size_t blocks = (npix + (size_t)rows * 16 - 1) / ((size_t)rows * 16);
  if (blocks > (size_t)tg_sms() * 4) blocks = (size_t)tg_sms() * 4;
  if (blocks < 1) blocks = 1;
  tg_launch(bias_grad_kernel, dim3((unsigned)blocks), dim3(256), (size_t)rows * c * sizeof(float),
            (cudaStream_t)stream, (const uint4*)dz, npix, c8, c_real, scale, db);
  TG_CUDA_LAUNCH_CHECK("bias_grad");
  return TG_OK;
}

int tg_backward_warp_bwd_nchw_f32(const float* x, const float* flow, const float* gy, float* gx, float* gflow,
                                  int n, int c, int h, int w, void* stream) {
  TG_REQUIRE(x && flow && gy && (gx || gflow), TG_E_INVALID, "backward_warp_bwd: null pointer");
  TG_REQUIRE(n > 0 && c > 0 && h >= 2 && w >= 2, TG_E_INVALID, "backward_warp_bwd: bad shape");
  const size_t total = (size_t)n * h * w;
  tg_launch(backward_warp_bwd_kernel, dim3(bgrid(total, 256)), dim3(256), 0, (cudaStream_t)stream, x, flow, gy, gx,
            gflow, n, c, h, w);
  TG_CUDA_LAUNCH_CHECK("backward_warp_bwd");
  return TG_OK;
}

int tg_warp_s2d_concat_bwd(const void* gx, const float* hr_prev, const float* hr_flow, const float* scale,
                           float* d_hr_prev, float* d_hr_flow, int n, int c, int h, int w, int s, int cpad,
                           void* stream) {
  TG_REQUIRE(gx && hr_prev && hr_flow && (d_hr_prev || d_hr_flow), TG_E_INVALID, "warp_s2d_concat_bwd: null pointer");
  TG_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0, TG_E_INVALID, "warp_s2d_concat_bwd: bad size");
  TG_REQUIRE(s == 2 || s == 4, TG_E_UNSUPPORTED, "warp_s2d_concat_bwd: scale %d (2 or 4)", s);
  TG_REQUIRE(cpad % 8 == 0 && (s * s + 1) * c <= cpad, TG_E_UNSUPPORTED, "warp_s2d_concat_bwd: channels do not fit");
  const size_t total = (size_t)n * h * s * w * s;
  cudaStream_t st = (cudaStream_t)stream;
  if (s == 4)
    tg_launch(warp_s2d_concat_bwd_kernel<4>, dim3(bgrid(total, 256)), dim3(256), 0, st, (const __half*)gx, hr_prev,
              hr_flow, scale, d_hr_prev, d_hr_flow, n, c, h, w, cpad);
  else
    tg_launch(warp_s2d_concat_bwd_kernel<2>, dim3(bgrid(total, 256)), dim3(256), 0, st, (const __half*)gx, hr_prev,
              hr_flow, scale, d_hr_prev, d_hr_flow, n, c, h, w, cpad);
  TG_CUDA_LAUNCH_CHECK("warp_s2d_concat_bwd");
  return TG_OK;
}

int tg_upsample_bwd_nchw_f32(const float* gy, float* gx, int n, int c, int h, int w, int s, int up_mode, float mul,
                             int accumulate, void* stream) {
  TG_REQUIRE(gy && gx, TG_E_INVALID, "upsample_bwd: null pointer");
  TG_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0, TG_E_INVALID, "upsample_bwd: bad shape");
  TG_REQUIRE(up_mode == TG_UP_BICUBIC || up_mode == TG_UP_BILINEAR, TG_E_INVALID, "upsample_bwd: up_mode");
  TG_REQUIRE(s == 2 || s == 4, TG_E_UNSUPPORTED, "upsample_bwd: scale %d (2 or 4)", s);
  TG_REQUIRE((size_t)n * c <= 65535 && tg_ceil_div(h, 8) <= 65535, TG_E_UNSUPPORTED, "upsample_bwd: grid too large");
  dim3 grid(tg_ceil_div(w, 32), tg_ceil_div(h, 8), n * c);
  cudaStream_t st = (cudaStream_t)stream;
  if (s == 4) tg_launch(upsample_bwd_kernel<4>, grid, dim3(256), 0, st, gy, gx, h, w, up_mode, mul, accumulate);
  else        tg_launch(upsample_bwd_kernel<2>, grid, dim3(256), 0, st, gy, gx, h, w, up_mode, mul, accumulate);
  TG_CUDA_LAUNCH_CHECK("upsample_bwd");
  return TG_OK;
}

int tg_maxpool2x2_bwd_nhwc_f16(const void* x, const void* gy, void* gx, int n, int h, int w, int c, int act,
                               void* stream) {
  TG_REQUIRE(x && gy && gx, TG_E_INVALID, "maxpool2x2_bwd: null pointer");
  TG_REQUIRE(n > 0 && h >= 2 && w >= 2 && c > 0 && c % 8 == 0, TG_E_INVALID, "maxpool2x2_bwd: bad shape");
  TG_REQUIRE(act >= TG_ACT_NONE && act <= TG_ACT_LRELU02, TG_E_INVALID, "maxpool2x2_bwd: act");
  const size_t total = (size_t)n * ((h + 1) / 2) * ((w + 1) / 2) * (c / 8);
  tg_launch(maxpool2x2_bwd_kernel, dim3(bgrid(total, 256)), dim3(256), 0, (cudaStream_t)stream, (const uint4*)x,
            (const uint4*)gy, (uint4*)gx, n, h, w, c / 8, act);
  TG_CUDA_LAUNCH_CHECK("maxpool2x2_bwd");
  return TG_OK;
}

int tg_upsample2x_bilinear_bwd_nhwc_f16(const void* gy, const void* m, void* gx, int n, int h, int w, int c,
                                        int act, void* stream) {
  TG_REQUIRE(gy && m && gx, TG_E_INVALID, "upsample2x_bwd: null pointer");
  TG_REQUIRE(n > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0, TG_E_INVALID, "upsample2x_bwd: bad shape");
  TG_REQUIRE(act >= TG_ACT_NONE && act <= TG_ACT_LRELU02, TG_E_INVALID, "upsample2x_bwd: act");
  const size_t total = (size_t)n * h * w * (c / 8);
  tg_launch(upsample2x_bwd_kernel, dim3(bgrid(total, 256)), dim3(256), 0, (cudaStream_t)stream, (const uint4*)gy,
            (const uint4*)m, (uint4*)gx, n, h, w, c / 8, act);
  TG_CUDA_LAUNCH_CHECK("upsample2x_bwd");
  return TG_OK;
}

int tg_flow_head_bwd(const float* gflow, const float* gflow2, const float* flow, void* scale_ws, float target,
                     void* dz, int n, int h, int w, int cpad, void* stream) {
  TG_REQUIRE(gflow && flow && scale_ws && dz, TG_E_INVALID, "flow_head_bwd: null pointer");
  TG_REQUIRE(n > 0 && h > 0 && w > 0 && cpad % 8 == 0 && cpad >= 8, TG_E_INVALID, "flow_head_bwd: bad shape");
  float* scale = reinterpret_cast<float*>(scale_ws);
  unsigned int* bits = reinterpret_cast<unsigned int*>(scale_ws) + 2;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t total = (size_t)n * 2 * h * w;
  tg_launch(flow_head_amax_kernel, dim3(bgrid(total, 256)), dim3(256), 0, st, gflow, gflow2, flow, total, bits);
  TG_CUDA_LAUNCH_CHECK("flow_head_amax");
  tg_launch(scale_from_amax_kernel, dim3(1), dim3(1), 0, st, bits, target, scale);
  TG_CUDA_LAUNCH_CHECK("flow_head_scale");
  tg_launch(flow_head_bwd_kernel, dim3(bgrid((size_t)n * h * w, 256)), dim3(256), 0, st, gflow, gflow2, flow,
            (const float*)scale, (uint4*)dz, n, h * w, cpad / 8);
  TG_CUDA_LAUNCH_CHECK("flow_head_bwd");
  return TG_OK;
}

int tg_depth_to_space_nchw_f32(const float* gy, float* gx, int n, int c, int h, int w, int s, void* stream) {
  TG_REQUIRE(gy && gx, TG_E_INVALID, "depth_to_space: null pointer");
  TG_REQUIRE(n > 0 && c > 0 && s > 0 && h >= s && w >= s, TG_E_INVALID, "depth_to_space: bad shape");
  const size_t total = (size_t)n * c * h * w;
  tg_launch(depth_to_space_kernel, dim3(bgrid(total, 256)), dim3(256), 0, (cudaStream_t)stream, gy, gx, n, c, h, w, s);
  TG_CUDA_LAUNCH_CHECK("depth_to_space");
  return TG_OK;
}

}  // extern "C"
