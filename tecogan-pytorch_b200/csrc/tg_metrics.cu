// Video quality metrics on the device: the frame input of PSNR / tOF scoring (gray planes and per-frame integer
// SSE in one read of the uint8 frames) and Farneback dense optical flow (cv2.calcOpticalFlowFarneback, flags=0),
// batched over many frame pairs per launch, and the per-pair sum of the end-point error between two flow sets over
// a window.  For the official metric script: the unrounded Y's squared-difference sum and the predicted Y's range
// over a window, and SSIM (skimage compare_ssim) of the Y over that window.
// Specification: oracle/farneback.py, oracle/metrics_oracle.py and oracle/official_metrics.py.
// Contract: include/tecogan_b200.h.
#include <math.h>

#include "tg_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxBlurTaps = 63;           // Gaussian kernel of the coarsest level (19 at levels=3, pyr_scale=0.5)
constexpr int kMaxPolyN = 7;
constexpr int kMinLevelSize = 32;
constexpr int kMaxWin = 63;                // box window of the flow update
constexpr int kTileW = 32, kTileH = 16;    // flow-update tile (outputs)

// ---- frame input ---------------------------------------------------------------------------------------------------

// BT.601 studio-swing Y before rounding: float64 r*T0 + g*T1 + b*T2 + 16, left to right, no FMA.  This is the
// official metric script's _rgb2ycbcr Y (maxVal=255), which it never rounds.
__device__ __forceinline__ double y_f64(int r, int g, int b) {
  double s = __dmul_rn((double)r, 0.256788235294118);
  s = __dadd_rn(s, __dmul_rn((double)g, 0.504129411764706));
  s = __dadd_rn(s, __dmul_rn((double)b, 0.097905882352941));
  return __dadd_rn(s, 16.0);
}

// Y of data_utils.rgb_to_ycbcr: y_f64 rounded half to even.  For three colours numpy's matmul rounds its sum to the
// other side of a .5 tie; the reference's Y of those is one lower (the rule is checked over all 2^24 colours in
// tests/test_metrics_cpu.py).
__device__ __forceinline__ int y_of(int r, int g, int b) {
  const double s = y_f64(r, g, b);
  int y = (int)rint(fmin(fmax(s, 0.0), 255.0));
  const int c = (r << 16) | (g << 8) | b;
  if (c == 0x01ade1 || c == 0x0caebf || c == 0x182e49) y -= 1;   // (1,173,225) (12,174,191) (24,46,73)
  return y;
}

// cv2 COLOR_RGB2GRAY on uint8, bit-exact
__device__ __forceinline__ int gray_of(int r, int g, int b) { return (9798 * r + 19235 * g + 3735 * b + 16384) >> 15; }

__global__ void __launch_bounds__(kThreads)
frames_in_kernel(const uint8_t* __restrict__ tru, int ht, int wt, const uint8_t* __restrict__ pred, int hp, int wp,
                 int h, int w, int psnr, uint8_t* __restrict__ gray, unsigned long long* __restrict__ sse, int t) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int f = blockIdx.y;
  const size_t hw = (size_t)h * w;
  const uint8_t* a = tru + (size_t)f * ht * wt * 3;
  const uint8_t* b = pred ? pred + (size_t)f * hp * wp * 3 : nullptr;
  unsigned long long acc = 0;
  for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < hw; i += (size_t)gridDim.x * kThreads) {
    const int y = (int)(i / w), x = (int)(i - (size_t)y * w);
    const uint8_t* pa = a + ((size_t)y * wt + x) * 3;
    const int ar = pa[0], ag = pa[1], ab = pa[2];
    if (gray) gray[(size_t)f * hw + i] = (uint8_t)gray_of(ar, ag, ab);
    if (!b) continue;
    const uint8_t* pb = b + ((size_t)y * wp + x) * 3;
    const int br = pb[0], bg = pb[1], bb = pb[2];
    if (gray) gray[((size_t)t + f) * hw + i] = (uint8_t)gray_of(br, bg, bb);
    if (psnr == TG_PSNR_RGB) {
      acc += (unsigned)((ar - br) * (ar - br) + (ag - bg) * (ag - bg) + (ab - bb) * (ab - bb));
    } else if (psnr == TG_PSNR_Y) {
      const int d = y_of(ar, ag, ab) - y_of(br, bg, bb);
      acc += (unsigned)(d * d);
    }
  }
  if (psnr == TG_PSNR_NONE || !sse) return;
  __shared__ unsigned long long warp_sum[kThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x != 0) return;
  unsigned long long s = 0;
#pragma unroll
  for (int k = 0; k < kThreads / 32; ++k) s += warp_sum[k];
  atomicAdd(sse + f, s);
}

// ---- official metric script: Y statistics and SSIM over a window ---------------------------------------------------
// Every sum is reduced in a fixed order (per-CTA partials in the caller's workspace, then one CTA per frame), so the
// same inputs give the same bits on every run and for every chunking of the frames.

constexpr int kStatsMaxBlocks = 128;       // per frame
constexpr int kSsimTW = 32, kSsimTH = 16;  // SSIM outputs per CTA
constexpr int kSsimR = 3;                  // 7x7 window

// sum, min and max of a CTA, in a fixed order; the result is valid in thread 0
__device__ __forceinline__ void block_sum_min_max(double& s, double& mn, double& mx) {
  __shared__ double red[3][kThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s = __dadd_rn(s, __shfl_down_sync(0xffffffffu, s, o));
    mn = fmin(mn, __shfl_down_sync(0xffffffffu, mn, o));
    mx = fmax(mx, __shfl_down_sync(0xffffffffu, mx, o));
  }
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    red[0][warp] = s;
    red[1][warp] = mn;
    red[2][warp] = mx;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    s = red[0][0];
    mn = red[1][0];
    mx = red[2][0];
#pragma unroll
    for (int k = 1; k < kThreads / 32; ++k) {
      s = __dadd_rn(s, red[0][k]);
      mn = fmin(mn, red[1][k]);
      mx = fmax(mx, red[2][k]);
    }
  }
}

// part [t, gridDim.x, 3]: per CTA {sum (Yt - Yp)^2, min Yp, max Yp} over its rows of the window
__global__ void __launch_bounds__(kThreads)
official_stats_kernel(const uint8_t* __restrict__ tru, int ht, int wt, const uint8_t* __restrict__ pred, int hp,
                      int wp, int y0, int x0, int hc, int wc, double* __restrict__ part) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int f = blockIdx.y;
  const uint8_t* a = tru + (size_t)f * ht * wt * 3;
  const uint8_t* b = pred + (size_t)f * hp * wp * 3;
  double s = 0.0, mn = INFINITY, mx = -INFINITY;
  for (int r = blockIdx.x; r < hc; r += gridDim.x) {          // CTA k: rows k, k + gridDim.x, ...
    const uint8_t* ra = a + ((size_t)(y0 + r) * wt + x0) * 3;
    const uint8_t* rb = b + ((size_t)(y0 + r) * wp + x0) * 3;
    for (int c = threadIdx.x; c < wc; c += kThreads) {
      const double yp = y_f64(rb[3 * c], rb[3 * c + 1], rb[3 * c + 2]);
      const double d = __dadd_rn(y_f64(ra[3 * c], ra[3 * c + 1], ra[3 * c + 2]), -yp);
      s = __dadd_rn(s, __dmul_rn(d, d));
      mn = fmin(mn, yp);
      mx = fmax(mx, yp);
    }
  }
  block_sum_min_max(s, mn, mx);
  if (threadIdx.x == 0) {
    double* o = part + ((size_t)f * gridDim.x + blockIdx.x) * 3;
    o[0] = s;
    o[1] = mn;
    o[2] = mx;
  }
}

// stats [t, 3] from part [t, nb, 3]: one CTA per frame
__global__ void __launch_bounds__(kThreads)
official_stats_final_kernel(const double* __restrict__ part, int nb, double* __restrict__ stats) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int f = blockIdx.x;
  const double* p = part + (size_t)f * nb * 3;
  double s = 0.0, mn = INFINITY, mx = -INFINITY;
  for (int k = threadIdx.x; k < nb; k += kThreads) {
    s = __dadd_rn(s, p[3 * k]);
    mn = fmin(mn, p[3 * k + 1]);
    mx = fmax(mx, p[3 * k + 2]);
  }
  block_sum_min_max(s, mn, mx);
  if (threadIdx.x == 0) {
    stats[3 * f] = s;
    stats[3 * f + 1] = mn;
    stats[3 * f + 2] = mx;
  }
}

// SSIM map of skimage's compare_ssim (7x7 uniform window, sample covariance) on a kSsimTW x kSsimTH tile of the
// window's interior, with data_range = max Yp - min Yp from stats [t, 3].  Interior pixel (i, j) of the window
// (3 <= i < hc - 3, 3 <= j < wc - 3) is tile output (i - 3, j - 3).  part [t, tiles]: the tile's sum of S.
__global__ void __launch_bounds__(kThreads)
ssim_tile_kernel(const uint8_t* __restrict__ tru, int ht, int wt, const uint8_t* __restrict__ pred, int hp, int wp,
                 int y0, int x0, int hc, int wc, const double* __restrict__ stats, double* __restrict__ part) {
  constexpr int LW = kSsimTW + 2 * kSsimR, LH = kSsimTH + 2 * kSsimR;
  __shared__ double ys[2][LH][LW];            // Yt, Yp with a 3-pixel halo
  __shared__ double hs[5][LH][kSsimTW];       // 7-tap row sums of x, y, x x, y y, x y
  tg_pdl_wait();
  tg_pdl_trigger();
  const int f = blockIdx.z;
  const int oy = blockIdx.y * kSsimTH, ox = blockIdx.x * kSsimTW;   // tile origin in window coordinates
  const uint8_t* a = tru + (size_t)f * ht * wt * 3;
  const uint8_t* b = pred + (size_t)f * hp * wp * 3;
  for (int i = threadIdx.x; i < LH * LW; i += kThreads) {
    const int r = i / LW, c = i % LW;
    // rows / columns past the window only feed outputs past the interior, which are not kept
    const int y = y0 + min(oy + r, hc - 1), x = x0 + min(ox + c, wc - 1);
    const uint8_t* pa = a + ((size_t)y * wt + x) * 3;
    const uint8_t* pb = b + ((size_t)y * wp + x) * 3;
    ys[0][r][c] = y_f64(pa[0], pa[1], pa[2]);
    ys[1][r][c] = y_f64(pb[0], pb[1], pb[2]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < LH * kSsimTW; i += kThreads) {
    const int r = i / kSsimTW, c = i % kSsimTW;
    double sx = 0.0, sy = 0.0, sxx = 0.0, syy = 0.0, sxy = 0.0;
#pragma unroll
    for (int k = 0; k <= 2 * kSsimR; ++k) {
      const double x = ys[0][r][c + k], y = ys[1][r][c + k];
      sx = __dadd_rn(sx, x);
      sy = __dadd_rn(sy, y);
      sxx = __dadd_rn(sxx, __dmul_rn(x, x));
      syy = __dadd_rn(syy, __dmul_rn(y, y));
      sxy = __dadd_rn(sxy, __dmul_rn(x, y));
    }
    hs[0][r][c] = sx;
    hs[1][r][c] = sy;
    hs[2][r][c] = sxx;
    hs[3][r][c] = syy;
    hs[4][r][c] = sxy;
  }
  __syncthreads();
  const double R = __dadd_rn(stats[3 * f + 2], -stats[3 * f + 1]);
  const double k1r = __dmul_rn(0.01, R), k2r = __dmul_rn(0.03, R);
  const double C1 = __dmul_rn(k1r, k1r), C2 = __dmul_rn(k2r, k2r);
  const double cov_norm = 49.0 / 48.0;
  double acc = 0.0;
  for (int i = threadIdx.x; i < kSsimTW * kSsimTH; i += kThreads) {
    const int r = i / kSsimTW, c = i % kSsimTW;
    if (oy + r >= hc - 2 * kSsimR || ox + c >= wc - 2 * kSsimR) continue;
    double m[5];
#pragma unroll
    for (int q = 0; q < 5; ++q) {
      double v = 0.0;
#pragma unroll
      for (int k = 0; k <= 2 * kSsimR; ++k) v = __dadd_rn(v, hs[q][r + k][c]);
      m[q] = v / 49.0;
    }
    const double ux = m[0], uy = m[1];
    const double vx = __dmul_rn(cov_norm, __dadd_rn(m[2], -__dmul_rn(ux, ux)));
    const double vy = __dmul_rn(cov_norm, __dadd_rn(m[3], -__dmul_rn(uy, uy)));
    const double vxy = __dmul_rn(cov_norm, __dadd_rn(m[4], -__dmul_rn(ux, uy)));
    const double A1 = __dadd_rn(__dmul_rn(__dmul_rn(2.0, ux), uy), C1);
    const double A2 = __dadd_rn(__dmul_rn(2.0, vxy), C2);
    const double B1 = __dadd_rn(__dadd_rn(__dmul_rn(ux, ux), __dmul_rn(uy, uy)), C1);
    const double B2 = __dadd_rn(__dadd_rn(vx, vy), C2);
    acc = __dadd_rn(acc, __dmul_rn(A1, A2) / __dmul_rn(B1, B2));
  }
  double mn = 0.0, mx = 0.0;
  block_sum_min_max(acc, mn, mx);
  if (threadIdx.x == 0) part[((size_t)f * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = acc;
}

// ssim[f] = sum of part[f, 0..nb) / count: one CTA per frame
__global__ void __launch_bounds__(kThreads)
ssim_final_kernel(const double* __restrict__ part, int nb, double count, double* __restrict__ ssim) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int f = blockIdx.x;
  double s = 0.0, mn = 0.0, mx = 0.0;
  for (int k = threadIdx.x; k < nb; k += kThreads) s = __dadd_rn(s, part[(size_t)f * nb + k]);
  block_sum_min_max(s, mn, mx);
  if (threadIdx.x == 0) ssim[f] = s / count;
}

// ---- pyramid level: Gaussian blur at full size + INTER_LINEAR resize, both separable -------------------------------

struct BlurTaps {
  float g[kMaxBlurTaps];
  int ksize;
};

// cv2 INTER_LINEAR source index / weight along one axis: fx = float((d + 0.5) * scale - 0.5), clamped at the ends
__device__ __forceinline__ void linear_src(int d, int src, double scale, int& s0, int& s1, float& f) {
  float fx = (float)((d + 0.5) * scale - 0.5);
  int s = (int)floorf(fx);
  fx -= (float)s;
  if (s < 0) { fx = 0.f; s = 0; }
  if (s >= src - 1) { fx = 0.f; s = src - 1; }
  s0 = s;
  s1 = min(s + 1, src - 1);
  f = fx;
}

__device__ __forceinline__ int reflect101(int i, int n) {
  const int period = 2 * (n - 1);
  i = abs(i) % period;
  return i >= n ? period - i : i;
}

// gray u8 [img, H, W] -> tmp f32 [img, h, W]: blur along rows of the source, resample to the level's rows
__global__ void __launch_bounds__(kThreads)
blur_resize_v_kernel(const uint8_t* __restrict__ src, float* __restrict__ dst, int H, int W, int h, double scale,
                     BlurTaps taps) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int img = blockIdx.z, y = blockIdx.y;
  int s0, s1;
  float fy;
  linear_src(y, H, scale, s0, s1, fy);
  const uint8_t* in = src + (size_t)img * H * W;
  const int r = taps.ksize / 2;
  for (int x = blockIdx.x * kThreads + threadIdx.x; x < W; x += gridDim.x * kThreads) {
    float a = 0.f, b = 0.f;
    for (int k = 0; k < taps.ksize; ++k) {
      a = fmaf(taps.g[k], (float)__ldg(in + (size_t)reflect101(s0 - r + k, H) * W + x), a);
      b = fmaf(taps.g[k], (float)__ldg(in + (size_t)reflect101(s1 - r + k, H) * W + x), b);
    }
    dst[((size_t)img * h + y) * W + x] = a * (1.f - fy) + b * fy;
  }
}

// tmp f32 [img, h, W] -> I f32 [img, h, w]
__global__ void __launch_bounds__(kThreads)
blur_resize_h_kernel(const float* __restrict__ src, float* __restrict__ dst, int W, int h, int w, double scale,
                     BlurTaps taps) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int img = blockIdx.z, y = blockIdx.y;
  const float* in = src + ((size_t)img * h + y) * W;
  const int r = taps.ksize / 2;
  for (int x = blockIdx.x * kThreads + threadIdx.x; x < w; x += gridDim.x * kThreads) {
    int s0, s1;
    float fx;
    linear_src(x, W, scale, s0, s1, fx);
    float a = 0.f, b = 0.f;
    for (int k = 0; k < taps.ksize; ++k) {
      a = fmaf(taps.g[k], __ldg(in + reflect101(s0 - r + k, W)), a);
      b = fmaf(taps.g[k], __ldg(in + reflect101(s1 - r + k, W)), b);
    }
    dst[((size_t)img * h + y) * w + x] = a * (1.f - fx) + b * fx;
  }
}

// ---- polynomial expansion ------------------------------------------------------------------------------------------

struct PolyTaps {
  float g[kMaxPolyN + 1], xg[kMaxPolyN + 1], xxg[kMaxPolyN + 1];   // offsets 0..n
  double ig11, ig03, ig33, ig55;
  int n;
};

// I [img, h, w] -> t [img, 3, h, w]: sums of g, x g, x^2 g down the columns, rows clamped
__global__ void __launch_bounds__(kThreads)
poly_v_kernel(const float* __restrict__ src, float* __restrict__ dst, int h, int w, PolyTaps p) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int img = blockIdx.z, y = blockIdx.y;
  const float* in = src + (size_t)img * h * w;
  const size_t hw = (size_t)h * w;
  for (int x = blockIdx.x * kThreads + threadIdx.x; x < w; x += gridDim.x * kThreads) {
    const float c = __ldg(in + (size_t)y * w + x);
    float t0 = c * p.g[0], t1 = 0.f, t2 = c * p.xxg[0];
    for (int k = 1; k <= p.n; ++k) {
      const float a = __ldg(in + (size_t)max(y - k, 0) * w + x);
      const float b = __ldg(in + (size_t)min(y + k, h - 1) * w + x);
      const float s = a + b;
      t0 += p.g[k] * s;
      t1 += p.xg[k] * (b - a);
      t2 += p.xxg[k] * s;
    }
    float* o = dst + (size_t)img * 3 * hw + (size_t)y * w + x;
    o[0] = t0;
    o[hw] = t1;
    o[2 * hw] = t2;
  }
}

// t [img, 3, h, w] -> R [img, 5, h, w]: the row sums in float64, columns clamped
__global__ void __launch_bounds__(kThreads)
poly_h_kernel(const float* __restrict__ src, float* __restrict__ dst, int h, int w, PolyTaps p) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int img = blockIdx.z, y = blockIdx.y;
  const size_t hw = (size_t)h * w;
  const float* r0 = src + (size_t)img * 3 * hw + (size_t)y * w;
  const float* r1 = r0 + hw;
  const float* r2 = r1 + hw;
  for (int x = blockIdx.x * kThreads + threadIdx.x; x < w; x += gridDim.x * kThreads) {
    double b1 = (double)__ldg(r0 + x) * p.g[0], b3 = (double)__ldg(r1 + x) * p.g[0];
    double b5 = (double)__ldg(r2 + x) * p.g[0], b2 = 0, b4 = 0, b6 = 0;
    for (int k = 1; k <= p.n; ++k) {
      const int lo = max(x - k, 0), hi = min(x + k, w - 1);
      const float a0 = __ldg(r0 + lo), c0 = __ldg(r0 + hi);
      const float a1 = __ldg(r1 + lo), c1 = __ldg(r1 + hi);
      const double s0 = (double)c0 + a0;
      b1 += s0 * p.g[k];
      b4 += s0 * p.xxg[k];
      b2 += ((double)c0 - a0) * p.xg[k];
      b3 += ((double)c1 + a1) * p.g[k];
      b6 += ((double)c1 - a1) * p.xg[k];
      b5 += ((double)__ldg(r2 + hi) + __ldg(r2 + lo)) * p.g[k];
    }
    float* o = dst + (size_t)img * 5 * hw + (size_t)y * w + x;
    o[0] = (float)(b3 * p.ig11);
    o[hw] = (float)(b2 * p.ig11);
    o[2 * hw] = (float)(b1 * p.ig03 + b5 * p.ig33);
    o[3 * hw] = (float)(b1 * p.ig03 + b4 * p.ig33);
    o[4 * hw] = (float)(b6 * p.ig55);
  }
}

// ---- flow ----------------------------------------------------------------------------------------------------------

// pair q of a batch of groups of t frames: (prev, next) = (g t + j, g t + j + 1), j = q mod (t - 1)
__device__ __forceinline__ int prev_image(int q, int t) { return (q / (t - 1)) * t + q % (t - 1); }

__device__ __forceinline__ float edge_weight(int i, int n) {
  const float kBorder[5] = {0.14f, 0.14f, 0.4472f, 0.4472f, 0.4472f};
  float s = 1.f;
  if (i < 5) s *= kBorder[i];
  if (i >= n - 5) s *= kBorder[n - 1 - i];
  return s;
}

// UpdateMatrices at (x, y) of pair q with flow (dx, dy): M [pair, 5, h, w]
__device__ __forceinline__ void update_matrices_at(const float* __restrict__ R, float* __restrict__ M, int q, int t,
                                                   int x, int y, int h, int w, float dx, float dy) {
  const size_t hw = (size_t)h * w;
  const int i0 = prev_image(q, t);
  const float* R0 = R + (size_t)i0 * 5 * hw + (size_t)y * w + x;
  const float* R1 = R + (size_t)(i0 + 1) * 5 * hw;
  float fx = (float)x + dx, fy = (float)y + dy;
  const float flx = floorf(fx), fly = floorf(fy);
  fx -= flx;
  fy -= fly;
  float r[5];
  float r2, r3, r4, r5, r6;
  if (flx >= 0.f && flx < (float)(w - 1) && fly >= 0.f && fly < (float)(h - 1)) {
    const int x1 = (int)flx, y1 = (int)fly;
    const float a00 = (1.f - fx) * (1.f - fy), a01 = fx * (1.f - fy), a10 = (1.f - fx) * fy, a11 = fx * fy;
    const float* p = R1 + (size_t)y1 * w + x1;
#pragma unroll
    for (int c = 0; c < 5; ++c) {
      const float* pc = p + c * hw;
      r[c] = a00 * __ldg(pc) + a01 * __ldg(pc + 1) + a10 * __ldg(pc + w) + a11 * __ldg(pc + w + 1);
    }
    r4 = (R0[2 * hw] + r[2]) * 0.5f;
    r5 = (R0[3 * hw] + r[3]) * 0.5f;
    r6 = (R0[4 * hw] + r[4]) * 0.25f;
  } else {
    r[0] = r[1] = 0.f;
    r4 = R0[2 * hw];
    r5 = R0[3 * hw];
    r6 = R0[4 * hw] * 0.5f;
  }
  r2 = (R0[0] - r[0]) * 0.5f;
  r3 = (R0[hw] - r[1]) * 0.5f;
  r2 += r4 * dy + r6 * dx;
  r3 += r6 * dy + r5 * dx;
  const float s = edge_weight(x, w) * edge_weight(y, h);
  r2 *= s; r3 *= s; r4 *= s; r5 *= s; r6 *= s;
  float* m = M + (size_t)q * 5 * hw + (size_t)y * w + x;
  m[0] = r4 * r4 + r6 * r6;
  m[hw] = (r4 + r5) * r6;
  m[2 * hw] = r5 * r5 + r6 * r6;
  m[3 * hw] = r4 * r2 + r6 * r3;
  m[4 * hw] = r6 * r2 + r5 * r3;
}

// the level's starting flow (0 on the coarsest level, else the previous level's flow resized INTER_LINEAR and scaled
// by 1/pyr_scale) and the first UpdateMatrices.  prev_flow [pair, hp, wp, 2] or null; flow [pair, h, w, 2]
__global__ void __launch_bounds__(kThreads)
flow_init_kernel(const float* __restrict__ prev_flow, int hp, int wp, double sx, double sy, float inv_scale,
                 const float* __restrict__ R, float* __restrict__ flow, float* __restrict__ M, int t, int h, int w) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int q = blockIdx.z, y = blockIdx.y;
  for (int x = blockIdx.x * kThreads + threadIdx.x; x < w; x += gridDim.x * kThreads) {
    float dx = 0.f, dy = 0.f;
    if (prev_flow) {
      int x0, x1, y0, y1;
      float fx, fy;
      linear_src(x, wp, sx, x0, x1, fx);
      linear_src(y, hp, sy, y0, y1, fy);
      const float2* pf = reinterpret_cast<const float2*>(prev_flow) + (size_t)q * hp * wp;
      const float2 v00 = pf[(size_t)y0 * wp + x0], v01 = pf[(size_t)y0 * wp + x1];
      const float2 v10 = pf[(size_t)y1 * wp + x0], v11 = pf[(size_t)y1 * wp + x1];
      const float ax = (v00.x * (1.f - fx) + v01.x * fx), bx = (v10.x * (1.f - fx) + v11.x * fx);
      const float ay = (v00.y * (1.f - fx) + v01.y * fx), by = (v10.y * (1.f - fx) + v11.y * fx);
      dx = (ax * (1.f - fy) + bx * fy) * inv_scale;
      dy = (ay * (1.f - fy) + by * fy) * inv_scale;
    }
    reinterpret_cast<float2*>(flow)[((size_t)q * h + y) * w + x] = make_float2(dx, dy);
    update_matrices_at(R, M, q, t, x, y, h, w, dx, dy);
  }
}

// One iteration on a kTileW x kTileH tile: S = box mean of M_in (borders replicated), the flow from the 2x2 solve,
// and (M_out non-null) UpdateMatrices with the new flow into M_out
__global__ void __launch_bounds__(kThreads)
flow_iter_kernel(const float* __restrict__ M_in, const float* __restrict__ R, float* __restrict__ flow,
                 float* __restrict__ M_out, int t, int h, int w, int m, float inv_area) {
  extern __shared__ float smem[];
  tg_pdl_wait();
  tg_pdl_trigger();
  const int q = blockIdx.z;
  const int x0 = blockIdx.x * kTileW, y0 = blockIdx.y * kTileH;
  const int lw = kTileW + 2 * m, lh = kTileH + 2 * m;
  const size_t hw = (size_t)h * w;
  float* tile = smem;                          // [5][lh][lw]
  float* vs = smem + 5 * lh * lw;              // [5][kTileH][lw]
  const float* Mq = M_in + (size_t)q * 5 * hw;
  for (int i = threadIdx.x; i < 5 * lh * lw; i += kThreads) {
    const int c = i / (lh * lw), r = (i / lw) % lh, col = i % lw;
    const int yy = min(max(y0 - m + r, 0), h - 1), xx = min(max(x0 - m + col, 0), w - 1);
    tile[i] = __ldg(Mq + c * hw + (size_t)yy * w + xx);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 5 * kTileH * lw; i += kThreads) {
    const int c = i / (kTileH * lw), r = (i / lw) % kTileH, col = i % lw;
    const float* p = tile + (c * lh + r) * lw + col;
    float s = 0.f;
    for (int k = 0; k <= 2 * m; ++k) s += p[k * lw];
    vs[i] = s;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kTileW * kTileH; i += kThreads) {
    const int r = i / kTileW, col = i % kTileW;
    const int x = x0 + col, y = y0 + r;
    if (x >= w || y >= h) continue;
    double S[5];
#pragma unroll
    for (int c = 0; c < 5; ++c) {
      const float* p = vs + (c * kTileH + r) * lw + col;
      float s = 0.f;
      for (int k = 0; k <= 2 * m; ++k) s += p[k];
      S[c] = (double)s * inv_area;
    }
    const double idet = 1.0 / (S[0] * S[2] - S[1] * S[1] + 1e-3);
    const float dx = (float)((S[0] * S[4] - S[1] * S[3]) * idet);
    const float dy = (float)((S[2] * S[3] - S[1] * S[4]) * idet);
    reinterpret_cast<float2*>(flow)[((size_t)q * h + y) * w + x] = make_float2(dx, dy);
    if (M_out) update_matrices_at(R, M_out, q, t, x, y, h, w, dx, dy);
  }
}

constexpr int kEpeMaxBlocks = 512;        // CTAs per pair

// The sum over the window (y0, x0, hc, wc) of |a[q] - b[q]| (Euclidean, per pixel), in float64.  With part, CTA k of
// pair q takes rows k, k + gridDim.x, ... and writes its sum to part[q, k] (epe_final_kernel adds them in a fixed
// order: the same bits on every run).  Without, the window is the whole frame, read as one grid-strided range, and
// each CTA adds its sum to sums[q] with a float64 atomic.
__global__ void __launch_bounds__(kThreads)
epe_kernel(const float2* __restrict__ a, const float2* __restrict__ b, int h, int w, int y0, int x0, int hc, int wc,
           double* __restrict__ sums, double* __restrict__ part) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int q = blockIdx.y;
  const size_t base = (size_t)q * h * w + (size_t)y0 * w + x0;
  const float2* pa = a + base;
  const float2* pb = b + base;
  double acc = 0.0;
  if (!part) {                                 // the whole frame (tg_flow_epe_sum): one flat range
    const size_t n = (size_t)hc * wc;
    for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads) {
      const float2 u = __ldg(pa + i), v = __ldg(pb + i);
      const float ex = u.x - v.x, ey = u.y - v.y;
      acc += (double)sqrtf(ex * ex + ey * ey);
    }
  } else {
    for (int r = blockIdx.x; r < hc; r += gridDim.x) {
      for (int c = threadIdx.x; c < wc; c += kThreads) {
        const float2 u = __ldg(pa + (size_t)r * w + c), v = __ldg(pb + (size_t)r * w + c);
        const float ex = u.x - v.x, ey = u.y - v.y;
        acc += (double)sqrtf(ex * ex + ey * ey);
      }
    }
  }
  double mn = 0.0, mx = 0.0;
  block_sum_min_max(acc, mn, mx);
  if (threadIdx.x != 0) return;
  if (part)
    part[(size_t)q * gridDim.x + blockIdx.x] = acc;
  else
    atomicAdd(sums + q, acc);
}

// sums[q] = the sum of part[q, 0..nb) in a fixed order: one CTA per pair
__global__ void __launch_bounds__(kThreads)
epe_final_kernel(const double* __restrict__ part, int nb, double* __restrict__ sums) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int q = blockIdx.x;
  double s = 0.0, mn = 0.0, mx = 0.0;
  for (int k = threadIdx.x; k < nb; k += kThreads) s = __dadd_rn(s, part[(size_t)q * nb + k]);
  block_sum_min_max(s, mn, mx);
  if (threadIdx.x == 0) sums[q] = s;
}

// ---- host side ------------------------------------------------------------------------------------------------------

struct Level {
  int h, w, ksize;
  double sigma, scale;
};

int level_count(int h, int w, const tg_farneback_params* p) {
  double scale = 1.0;
  int k = 0;
  for (; k < p->levels; ++k) {
    scale *= p->pyr_scale;
    if (w * scale < kMinLevelSize || h * scale < kMinLevelSize) break;
  }
  return k;
}

Level level_of(int h, int w, const tg_farneback_params* p, int k) {
  Level L;
  double scale = 1.0;
  for (int i = 0; i < k; ++i) scale *= p->pyr_scale;
  L.scale = scale;
  L.sigma = (1.0 / scale - 1.0) * 0.5;
  L.ksize = ((int)nearbyint(L.sigma * 5)) | 1;
  if (L.ksize < 3) L.ksize = 3;
  L.h = (int)nearbyint(h * scale);
  L.w = (int)nearbyint(w * scale);
  return L;
}

BlurTaps blur_taps(int ksize, double sigma) {
  BlurTaps b = {};
  b.ksize = ksize;
  if (sigma <= 0 && ksize == 3) {           // cv2's fixed small kernel
    b.g[0] = 0.25f; b.g[1] = 0.5f; b.g[2] = 0.25f;
    return b;
  }
  if (sigma <= 0) sigma = 0.3 * ((ksize - 1) * 0.5 - 1) + 0.8;
  double t[kMaxBlurTaps], s = 0;
  for (int i = 0; i < ksize; ++i) {
    const double x = i - (ksize - 1) * 0.5;
    t[i] = exp(-0.5 / (sigma * sigma) * x * x);
    s += t[i];
  }
  for (int i = 0; i < ksize; ++i) b.g[i] = (float)(t[i] / s);
  return b;
}

// FarnebackPrepareGaussian: float32 taps, moments in float64 from float32 products, inverse by Gaussian elimination
PolyTaps poly_taps(int n, double sigma) {
  PolyTaps p = {};
  p.n = n;
  float g[2 * kMaxPolyN + 1];
  double s = 0;
  for (int x = -n; x <= n; ++x) {
    g[x + n] = (float)exp(-x * x / (2 * sigma * sigma));
    s += g[x + n];
  }
  s = 1.0 / s;
  for (int x = -n; x <= n; ++x) g[x + n] = (float)(g[x + n] * s);
  for (int x = 0; x <= n; ++x) {
    p.g[x] = g[x + n];
    p.xg[x] = (float)(x * g[x + n]);
    p.xxg[x] = (float)(x * x * g[x + n]);
  }
  double G[6][6] = {};
  for (int y = -n; y <= n; ++y)
    for (int x = -n; x <= n; ++x) {
      const float gg = g[y + n] * g[x + n], fx = (float)x, fy = (float)y;
      G[0][0] += gg;
      G[1][1] += gg * fx * fx;
      G[3][3] += gg * fx * fx * fx * fx;
      G[5][5] += gg * fx * fx * fy * fy;
    }
  G[2][2] = G[0][3] = G[0][4] = G[3][0] = G[4][0] = G[1][1];
  G[4][4] = G[3][3];
  G[3][4] = G[4][3] = G[5][5];
  double A[6][12] = {};
  for (int i = 0; i < 6; ++i) {
    for (int j = 0; j < 6; ++j) A[i][j] = G[i][j];
    A[i][6 + i] = 1.0;
  }
  for (int c = 0; c < 6; ++c) {             // symmetric positive definite: no pivoting needed
    const double d = A[c][c];
    for (int j = 0; j < 12; ++j) A[c][j] /= d;
    for (int i = 0; i < 6; ++i) {
      if (i == c) continue;
      const double f = A[i][c];
      for (int j = 0; j < 12; ++j) A[i][j] -= f * A[c][j];
    }
  }
  p.ig11 = A[1][7];
  p.ig03 = A[0][9];
  p.ig33 = A[3][9];
  p.ig55 = A[5][11];
  return p;
}

const char* check_params(const tg_farneback_params* p) {
  if (!p) return "null params";
  if (!(p->pyr_scale > 0.0 && p->pyr_scale < 1.0)) return "pyr_scale outside (0, 1)";
  if (p->levels < 0) return "negative levels";
  if (p->winsize < 1 || p->winsize > kMaxWin) return "winsize outside [1, 63]";
  if (p->iterations < 1) return "iterations < 1";
  if (p->poly_n != 5 && p->poly_n != 7) return "poly_n not 5 or 7";
  if (!(p->poly_sigma > 0.0 && isfinite(p->poly_sigma))) return "poly_sigma not positive";
  if (p->flags != 0) return "flags other than 0";
  return nullptr;
}

struct Layout {                              // float offsets into the workspace
  size_t scratch, R, M0, M1, flow_prev, total;
};

Layout layout_of(int n_img, int pairs, int h, int w) {
  const size_t hw = (size_t)h * w;
  auto up = [](size_t v) { return (v + 63) & ~(size_t)63; };   // 256-byte aligned regions
  Layout L;
  L.scratch = 0;
  L.R = up(L.scratch + 3 * (size_t)n_img * hw);   // >= tmp [img, h, W] of every level (level 0 is the largest)
  L.M0 = up(L.R + 5 * (size_t)n_img * hw);
  L.M1 = up(L.M0 + 5 * (size_t)pairs * hw);
  L.flow_prev = up(L.M1 + 5 * (size_t)pairs * hw);
  L.total = up(L.flow_prev + 2 * (size_t)pairs * hw);
  return L;
}

inline dim3 row_grid(int w, int rows, int z) {
  const int bx = (w + kThreads - 1) / kThreads;
  return dim3((unsigned)(bx < 8 ? bx : 8), (unsigned)rows, (unsigned)z);
}

bool window_inside(int y0, int x0, int hc, int wc, int h, int w) {
  return y0 >= 0 && x0 >= 0 && hc > 0 && wc > 0 && (long long)y0 + hc <= h && (long long)x0 + wc <= w;
}

int stats_blocks(int hc, int wc) {
  (void)wc;
  return hc < kStatsMaxBlocks ? hc : kStatsMaxBlocks;
}

// CTAs of ssim_tile_kernel over the (hc - 6) x (wc - 6) interior of the window
dim3 ssim_tiles(int hc, int wc) {
  return dim3((unsigned)((wc - 2 * kSsimR + kSsimTW - 1) / kSsimTW),
              (unsigned)((hc - 2 * kSsimR + kSsimTH - 1) / kSsimTH));
}

// the frame and window arguments of tg_official_frames_stats / tg_ssim_y; the window lies in the common size
const char* check_official_args(const uint8_t* tru, int ht, int wt, const uint8_t* pred, int hp, int wp, int t,
                                int y0, int x0, int hc, int wc, int min_side) {
  if (!tru || !pred) return "null frames";
  if (t <= 0 || ht <= 0 || wt <= 0 || hp <= 0 || wp <= 0) return "non-positive size";
  if (!window_inside(y0, x0, hc, wc, ht < hp ? ht : hp, wt < wp ? wt : wp)) return "window outside the common size";
  if (hc < min_side || wc < min_side) return "window smaller than the 7x7 SSIM window";
  return nullptr;
}

}  // namespace

extern "C" int tg_metrics_frames_in(const uint8_t* true_u8, int ht, int wt, const uint8_t* pred_u8, int hp, int wp,
                                    int t, int psnr, uint8_t* gray, unsigned long long* sse, void* stream) {
  const char* name = "metrics_frames_in";
  TG_REQUIRE(true_u8 != nullptr, TG_E_INVALID, "%s: null true frames", name);
  TG_REQUIRE(t > 0 && ht > 0 && wt > 0, TG_E_INVALID, "%s: bad size t=%d h=%d w=%d", name, t, ht, wt);
  TG_REQUIRE(psnr == TG_PSNR_NONE || psnr == TG_PSNR_RGB || psnr == TG_PSNR_Y, TG_E_INVALID, "%s: bad psnr mode %d",
             name, psnr);
  TG_REQUIRE(pred_u8 != nullptr || psnr == TG_PSNR_NONE, TG_E_INVALID, "%s: PSNR needs predicted frames", name);
  TG_REQUIRE(pred_u8 == nullptr || (hp > 0 && wp > 0), TG_E_INVALID, "%s: bad predicted size %dx%d", name, hp, wp);
  TG_REQUIRE((psnr == TG_PSNR_NONE) == (sse == nullptr), TG_E_INVALID, "%s: sse must be given exactly with PSNR",
             name);
  TG_REQUIRE(gray != nullptr || sse != nullptr, TG_E_INVALID, "%s: neither gray nor sse requested", name);
  TG_REQUIRE((((uintptr_t)sse) & 7u) == 0, TG_E_INVALID, "%s: sse must be 8-byte aligned", name);
  const int h = pred_u8 ? (ht < hp ? ht : hp) : ht, w = pred_u8 ? (wt < wp ? wt : wp) : wt;
  TG_REQUIRE(t <= 65535, TG_E_UNSUPPORTED, "%s: %d frames per launch (at most 65535)", name, t);
  cudaStream_t s = (cudaStream_t)stream;
  if (sse) {
    cudaError_t e = cudaMemsetAsync(sse, 0, (size_t)t * sizeof(unsigned long long), s);
    TG_REQUIRE(e == cudaSuccess, (int)e, "%s: memset: %s", name, cudaGetErrorString(e));
  }
  const size_t hw = (size_t)h * w;
  size_t bx = (hw + kThreads * 4 - 1) / (kThreads * 4);
  if (bx > 1024) bx = 1024;
  tg_launch(frames_in_kernel, dim3((unsigned)bx, (unsigned)t), dim3(kThreads), 0, s, true_u8, ht, wt, pred_u8, hp,
            wp, h, w, psnr, gray, sse, t);
  TG_CUDA_LAUNCH_CHECK(name);
  return TG_OK;
}

extern "C" size_t tg_farneback_workspace_bytes(int groups, int t, int h, int w) {
  if (groups <= 0 || t < 2 || h <= 0 || w <= 0) return 0;
  return layout_of(groups * t, groups * (t - 1), h, w).total * sizeof(float);
}

extern "C" int tg_farneback(const uint8_t* gray, int groups, int t, int h, int w, const tg_farneback_params* params,
                            float* flow, void* work, size_t work_bytes, void* stream) {
  const char* name = "farneback";
  TG_REQUIRE(gray && flow && work, TG_E_INVALID, "%s: null pointer (gray / flow / work)", name);
  TG_REQUIRE(groups > 0 && t >= 2 && h > 0 && w > 0, TG_E_INVALID, "%s: bad size groups=%d t=%d h=%d w=%d", name,
             groups, t, h, w);
  const char* bad = check_params(params);
  TG_REQUIRE(bad == nullptr, TG_E_INVALID, "%s: %s", name, bad);
  TG_REQUIRE(((((uintptr_t)flow) | ((uintptr_t)work)) & 15u) == 0, TG_E_INVALID,
             "%s: flow and work must be 16-byte aligned", name);
  TG_REQUIRE(h >= 2 && w >= 2, TG_E_UNSUPPORTED, "%s: frames of %dx%d (at least 2x2)", name, h, w);
  TG_REQUIRE((long long)groups * t <= 65535, TG_E_UNSUPPORTED, "%s: %d frames per launch (at most 65535)", name,
             groups * t);
  const int n_img = groups * t, pairs = groups * (t - 1);
  const Layout lay = layout_of(n_img, pairs, h, w);
  TG_REQUIRE(work_bytes >= lay.total * sizeof(float), TG_E_INVALID, "%s: workspace of %zu bytes, %zu needed", name,
             work_bytes, lay.total * sizeof(float));
  const int L = level_count(h, w, params);
  const Level top = level_of(h, w, params, L);
  TG_REQUIRE(top.ksize <= kMaxBlurTaps, TG_E_UNSUPPORTED, "%s: coarsest blur of %d taps (at most %d)", name,
             top.ksize, kMaxBlurTaps);
  float* ws = static_cast<float*>(work);
  float* scratch = ws + lay.scratch;
  float* R = ws + lay.R;
  float* M[2] = {ws + lay.M0, ws + lay.M1};
  float* flow_prev = ws + lay.flow_prev;
  const PolyTaps pt = poly_taps(params->poly_n, params->poly_sigma);
  const int m = params->winsize / 2;
  const size_t iter_smem = (size_t)5 * ((kTileH + 2 * m) + kTileH) * (kTileW + 2 * m) * sizeof(float);
  if (iter_smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(flow_iter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)iter_smem);
    TG_REQUIRE(e == cudaSuccess, (int)e, "%s: shared memory attribute: %s", name, cudaGetErrorString(e));
  }
  cudaStream_t s = (cudaStream_t)stream;
  int ph = 0, pw = 0;
  for (int k = L; k >= 0; --k) {
    const Level lv = level_of(h, w, params, k);
    const BlurTaps bt = blur_taps(lv.ksize, k == 0 ? 0.0 : lv.sigma);
    // the previous level's flow moves to flow_prev; the level's flow is built in `flow` (as big as level 0)
    float* cur = flow;
    const float* prev = nullptr;
    if (k < L) {
      cudaError_t e = cudaMemcpyAsync(flow_prev, flow, (size_t)pairs * ph * pw * 2 * sizeof(float),
                                      cudaMemcpyDeviceToDevice, s);
      TG_REQUIRE(e == cudaSuccess, (int)e, "%s: copy: %s", name, cudaGetErrorString(e));
      prev = flow_prev;
    }
    // gray -> tmp [img, lv.h, w] (scratch) -> level image [img, lv.h, lv.w] (R's region, free until poly_h) ->
    // t [img, 3, lv.h, lv.w] (scratch) -> R
    float* tmp = scratch;
    float* img = R;
    tg_launch(blur_resize_v_kernel, row_grid(w, lv.h, n_img), dim3(kThreads), 0, s, gray, tmp, h, w, lv.h,
              1.0 / ((double)lv.h / h), bt);
    TG_CUDA_LAUNCH_CHECK(name);
    tg_launch(blur_resize_h_kernel, row_grid(lv.w, lv.h, n_img), dim3(kThreads), 0, s, (const float*)tmp, img, w,
              lv.h, lv.w, 1.0 / ((double)lv.w / w), bt);
    TG_CUDA_LAUNCH_CHECK(name);
    tg_launch(poly_v_kernel, row_grid(lv.w, lv.h, n_img), dim3(kThreads), 0, s, (const float*)img, scratch, lv.h,
              lv.w, pt);
    TG_CUDA_LAUNCH_CHECK(name);
    tg_launch(poly_h_kernel, row_grid(lv.w, lv.h, n_img), dim3(kThreads), 0, s, (const float*)scratch, R, lv.h, lv.w,
              pt);
    TG_CUDA_LAUNCH_CHECK(name);
    tg_launch(flow_init_kernel, row_grid(lv.w, lv.h, pairs), dim3(kThreads), 0, s, prev, ph, pw,
              1.0 / ((double)lv.w / pw), 1.0 / ((double)lv.h / ph), (float)(1.0 / params->pyr_scale),
              (const float*)R, cur, M[0], t, lv.h, lv.w);
    TG_CUDA_LAUNCH_CHECK(name);
    const dim3 tiles((unsigned)((lv.w + kTileW - 1) / kTileW), (unsigned)((lv.h + kTileH - 1) / kTileH),
                     (unsigned)pairs);
    for (int i = 0; i < params->iterations; ++i) {
      const bool last = i == params->iterations - 1;
      tg_launch(flow_iter_kernel, tiles, dim3(kThreads), iter_smem, s, (const float*)M[i & 1], (const float*)R, cur,
                last ? nullptr : M[(i + 1) & 1], t, lv.h, lv.w, m,
                (float)(1.0 / ((double)params->winsize * params->winsize)));
      TG_CUDA_LAUNCH_CHECK(name);
    }
    ph = lv.h;
    pw = lv.w;
  }
  return TG_OK;
}

namespace {

int epe_blocks(int hc) { return hc < kEpeMaxBlocks ? hc : kEpeMaxBlocks; }

// work == nullptr: per-CTA float64 atomics into sums (zeroed first); else the fixed-order two-pass sum
int epe_sum(const char* name, const float* a, const float* b, int n, int h, int w, int y0, int x0, int hc, int wc,
            double* sums, void* work, size_t work_bytes, void* stream) {
  TG_REQUIRE(a && b && sums, TG_E_INVALID, "%s: null pointer (a / b / sums)", name);
  TG_REQUIRE(n > 0 && h > 0 && w > 0, TG_E_INVALID, "%s: bad size n=%d h=%d w=%d", name, n, h, w);
  TG_REQUIRE(window_inside(y0, x0, hc, wc, h, w), TG_E_INVALID, "%s: window (%d, %d, %d, %d) outside %dx%d", name,
             y0, x0, hc, wc, h, w);
  TG_REQUIRE(((((uintptr_t)a) | ((uintptr_t)b) | ((uintptr_t)sums) | ((uintptr_t)work)) & 7u) == 0, TG_E_INVALID,
             "%s: a / b / sums / work must be 8-byte aligned", name);
  TG_REQUIRE(n <= 65535, TG_E_UNSUPPORTED, "%s: %d pairs per launch (at most 65535)", name, n);
  double* part = static_cast<double*>(work);
  size_t flat = ((size_t)hc * wc + kThreads * 8 - 1) / (kThreads * 8);
  const int nb = part ? epe_blocks(hc) : (int)(flat < kEpeMaxBlocks ? flat : kEpeMaxBlocks);
  cudaStream_t s = (cudaStream_t)stream;
  if (part) {
    const size_t need = (size_t)n * nb * sizeof(double);
    TG_REQUIRE(work_bytes >= need, TG_E_INVALID, "%s: workspace of %zu bytes, %zu needed", name, work_bytes, need);
  } else {
    cudaError_t e = cudaMemsetAsync(sums, 0, (size_t)n * sizeof(double), s);
    TG_REQUIRE(e == cudaSuccess, (int)e, "%s: memset: %s", name, cudaGetErrorString(e));
  }
  tg_launch(epe_kernel, dim3((unsigned)nb, (unsigned)n), dim3(kThreads), 0, s, reinterpret_cast<const float2*>(a),
            reinterpret_cast<const float2*>(b), h, w, y0, x0, hc, wc, sums, part);
  TG_CUDA_LAUNCH_CHECK(name);
  if (part) {
    tg_launch(epe_final_kernel, dim3((unsigned)n), dim3(kThreads), 0, s, (const double*)part, nb, sums);
    TG_CUDA_LAUNCH_CHECK(name);
  }
  return TG_OK;
}

}  // namespace

extern "C" size_t tg_flow_epe_sum_window_workspace_bytes(int n, int hc) {
  if (n <= 0 || hc <= 0) return 0;
  return (size_t)n * epe_blocks(hc) * sizeof(double);
}

extern "C" int tg_flow_epe_sum_window(const float* a, const float* b, int n, int h, int w, int y0, int x0, int hc,
                                      int wc, double* sums, void* work, size_t work_bytes, void* stream) {
  TG_REQUIRE(work != nullptr, TG_E_INVALID, "flow_epe_sum_window: null workspace");
  return epe_sum("flow_epe_sum_window", a, b, n, h, w, y0, x0, hc, wc, sums, work, work_bytes, stream);
}

extern "C" int tg_flow_epe_sum(const float* a, const float* b, int n, int h, int w, double* sums, void* stream) {
  return epe_sum("flow_epe_sum", a, b, n, h, w, 0, 0, h, w, sums, nullptr, 0, stream);
}

extern "C" size_t tg_official_frames_stats_workspace_bytes(int t, int hc, int wc) {
  if (t <= 0 || hc <= 0 || wc <= 0) return 0;
  return (size_t)t * stats_blocks(hc, wc) * 3 * sizeof(double);
}

extern "C" int tg_official_frames_stats(const uint8_t* true_u8, int ht, int wt, const uint8_t* pred_u8, int hp,
                                        int wp, int t, int y0, int x0, int hc, int wc, double* stats, void* work,
                                        size_t work_bytes, void* stream) {
  const char* name = "official_frames_stats";
  const char* bad = check_official_args(true_u8, ht, wt, pred_u8, hp, wp, t, y0, x0, hc, wc, 1);
  TG_REQUIRE(bad == nullptr, TG_E_INVALID, "%s: %s", name, bad);
  TG_REQUIRE(stats && work, TG_E_INVALID, "%s: null pointer (stats / work)", name);
  TG_REQUIRE(((((uintptr_t)stats) | ((uintptr_t)work)) & 7u) == 0, TG_E_INVALID,
             "%s: stats and work must be 8-byte aligned", name);
  const size_t need = tg_official_frames_stats_workspace_bytes(t, hc, wc);
  TG_REQUIRE(work_bytes >= need, TG_E_INVALID, "%s: workspace of %zu bytes, %zu needed", name, work_bytes, need);
  TG_REQUIRE(t <= 65535, TG_E_UNSUPPORTED, "%s: %d frames per launch (at most 65535)", name, t);
  cudaStream_t s = (cudaStream_t)stream;
  const int nb = stats_blocks(hc, wc);
  double* part = static_cast<double*>(work);
  tg_launch(official_stats_kernel, dim3((unsigned)nb, (unsigned)t), dim3(kThreads), 0, s, true_u8, ht, wt, pred_u8,
            hp, wp, y0, x0, hc, wc, part);
  TG_CUDA_LAUNCH_CHECK(name);
  tg_launch(official_stats_final_kernel, dim3((unsigned)t), dim3(kThreads), 0, s, (const double*)part, nb, stats);
  TG_CUDA_LAUNCH_CHECK(name);
  return TG_OK;
}

extern "C" size_t tg_ssim_y_workspace_bytes(int t, int hc, int wc) {
  if (t <= 0 || hc < 2 * kSsimR + 1 || wc < 2 * kSsimR + 1) return 0;
  return (size_t)t * ssim_tiles(hc, wc).x * ssim_tiles(hc, wc).y * sizeof(double);
}

extern "C" int tg_ssim_y(const uint8_t* true_u8, int ht, int wt, const uint8_t* pred_u8, int hp, int wp, int t,
                         int y0, int x0, int hc, int wc, const double* stats, double* ssim, void* work,
                         size_t work_bytes, void* stream) {
  const char* name = "ssim_y";
  const char* bad = check_official_args(true_u8, ht, wt, pred_u8, hp, wp, t, y0, x0, hc, wc, 2 * kSsimR + 1);
  TG_REQUIRE(bad == nullptr, TG_E_INVALID, "%s: %s", name, bad);
  TG_REQUIRE(stats && ssim && work, TG_E_INVALID, "%s: null pointer (stats / ssim / work)", name);
  TG_REQUIRE(((((uintptr_t)stats) | ((uintptr_t)ssim) | ((uintptr_t)work)) & 7u) == 0, TG_E_INVALID,
             "%s: stats, ssim and work must be 8-byte aligned", name);
  const size_t need = tg_ssim_y_workspace_bytes(t, hc, wc);
  TG_REQUIRE(work_bytes >= need, TG_E_INVALID, "%s: workspace of %zu bytes, %zu needed", name, work_bytes, need);
  TG_REQUIRE(t <= 65535, TG_E_UNSUPPORTED, "%s: %d frames per launch (at most 65535)", name, t);
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 tiles = ssim_tiles(hc, wc);
  double* part = static_cast<double*>(work);
  tg_launch(ssim_tile_kernel, dim3(tiles.x, tiles.y, (unsigned)t), dim3(kThreads), 0, s, true_u8, ht, wt, pred_u8,
            hp, wp, y0, x0, hc, wc, stats, part);
  TG_CUDA_LAUNCH_CHECK(name);
  tg_launch(ssim_final_kernel, dim3((unsigned)t), dim3(kThreads), 0, s, (const double*)part, (int)(tiles.x * tiles.y),
            (double)(hc - 2 * kSsimR) * (wc - 2 * kSsimR), ssim);
  TG_CUDA_LAUNCH_CHECK(name);
  return TG_OK;
}
