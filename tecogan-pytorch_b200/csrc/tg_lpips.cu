// LPIPS (net-lin, AlexNet, v0.1) around the conv kernels: the frame prologue in conv1's space-to-depth layout,
// the 3x3 / stride-2 max pools (plain, or into conv2's four-shift layout) and the per-layer heads.
// oracle/lpips.py specifies every layout; include/tecogan_b200.h states the contracts.
#include "tg_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kHeadWarps = kThreads / 32;
constexpr int kHeadMaxChunks = 2;          // 16-byte chunks per lane: 2 x 32 x 8 = 512 channels
constexpr int kHeadMaxBlocks = 64;         // per-pair CTAs of tg_lpips_head (its workspace: one double each)

// ScalingLayer of PNetLin (float32 constants, as torch.Tensor([...]) holds them)
__constant__ float kShift[3] = {-.030f, -.088f, -.188f};
__constant__ float kScale[3] = {.458f, .448f, .450f};

// out[f][Y][X][ch] fp16, ch = (py*4 + px)*3 + c < 48: the scaled value of picture pixel (4Y+py-2, 4X+px-2), zero
// outside the picture and in channels 48..63.  One thread per 8 channels of a pixel (one 16-byte store).
__global__ void lpips_frames_in_kernel(const uint8_t* __restrict__ in, tg_frame_window win, int t, int h, int w,
                                       int hs, int ws, int norm, __half* __restrict__ out) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const size_t total = (size_t)t * hs * ws * 8;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int g = (int)(i & 7);
    size_t p = i >> 3;
    const int X = (int)(p % ws); p /= ws;
    const int Y = (int)(p % hs);
    const int f = (int)(p / hs);
    const uint8_t* frame = in + (size_t)f * win.frame_h * win.frame_w * 3;
    __align__(16) __half v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int ch = g * 8 + j;
      float val = 0.f;
      if (ch < 48) {
        const int q = ch / 3, c = ch - 3 * q;
        const int r = 4 * Y + (q >> 2) - 2, col = 4 * X + (q & 3) - 2;
        if (r >= 0 && r < h && col >= 0 && col < w) {
          const uint8_t u = __ldg(frame + ((size_t)(win.top + r) * win.frame_w + (win.left + col)) * 3 + c);
          // MetricCalculator: float32 x * 2 / 255 - 1; official script (util.im2tensor): float64 x / 127.5 - 1
          const float x = norm == TG_LPIPS_NORM_CALC ? (float)u * 2.f / 255.f - 1.f
                                                     : (float)((double)u / 127.5 - 1.0);
          val = (x - kShift[c]) / kScale[c];
        }
      }
      v[j] = __float2half_rn(val);
    }
    reinterpret_cast<uint4*>(out)[i] = *reinterpret_cast<const uint4*>(v);
  }
}

// Floor 3x3 / stride-2 max pool of the h x w interior at (y0, x0) of x [n][xh][xw][c].  shifts == 0: y [n][ph][pw][c];
// shifts != 0: y [n][ph+2][pw+2][4c], channel block b = by*2+bx of pixel (i, j) = pooled (i + 3by - 2, j + 3bx - 2),
// zero outside the pooled map.  One thread per 8 output channels.
__global__ void maxpool3x3s2_kernel(const __half* __restrict__ x, int n, int xh, int xw, int c, int y0, int x0,
                                    int ph, int pw, int shifts, __half* __restrict__ y) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int oh = shifts ? ph + 2 : ph, ow = shifts ? pw + 2 : pw, oc = shifts ? 4 * c : c;
  const int groups = oc / 8, cg = c / 8;
  const size_t total = (size_t)n * oh * ow * groups;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % groups);
    size_t p = i / groups;
    const int j = (int)(p % ow); p /= ow;
    const int r = (int)(p % oh);
    const int img = (int)(p / oh);
    int pi = r, pj = j, gc = g;
    if (shifts) {
      const int b = g / cg;
      gc = g - b * cg;
      pi = r + 3 * (b >> 1) - 2;
      pj = j + 3 * (b & 1) - 2;
    }
    uint4 m = make_uint4(0u, 0u, 0u, 0u);
    if (pi >= 0 && pi < ph && pj >= 0 && pj < pw) {
      const uint4* src = reinterpret_cast<const uint4*>(x) + gc;
      const size_t row = (size_t)xw * cg;
      const size_t base = ((size_t)img * xh + y0 + 2 * pi) * row + (size_t)(x0 + 2 * pj) * cg;
      m = __ldg(src + base);
#pragma unroll
      for (int dy = 0; dy < 3; ++dy)
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
          if (dy == 0 && dx == 0) continue;
          const uint4 v = __ldg(src + base + (size_t)dy * row + (size_t)dx * cg);
          __half2* a = reinterpret_cast<__half2*>(&m);
          const __half2* b = reinterpret_cast<const __half2*>(&v);
#pragma unroll
          for (int k = 0; k < 4; ++k) a[k] = __hmax2(a[k], b[k]);
        }
    }
    reinterpret_cast<uint4*>(y)[i] = m;
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
  return v;
}

// One warp per pixel of the interior: both channel norms and sum_c w_c (f0 / (|f0| + eps) - f1 / (|f1| + eps))^2 in
// fp32 (xor-tree sums, a fixed order), then the CTA's float64 sum of its pixels, in warp order, to work[pair][cta].
__global__ void __launch_bounds__(kThreads, 3) lpips_head_kernel(const __half* __restrict__ f, int n, int xh, int xw, int c, int y0, int x0, int h, int w,
                                  const int32_t* __restrict__ pairs, const float* __restrict__ wts,
                                  double* __restrict__ work) {
  tg_pdl_wait();
  tg_pdl_trigger();
  __shared__ double part[kHeadWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pair = blockIdx.y;
  const int i0 = __ldg(pairs + 2 * pair), i1 = __ldg(pairs + 2 * pair + 1);
  if (i0 < 0 || i0 >= n || i1 < 0 || i1 >= n) {   // an index outside the batch scores NaN; nothing is read
    if (threadIdx.x == 0) work[(size_t)pair * gridDim.x + blockIdx.x] = __longlong_as_double(0x7FF8000000000000LL);
    return;
  }
  const int chunks = c / 8;
  float wl[kHeadMaxChunks][8];
#pragma unroll
  for (int k = 0; k < kHeadMaxChunks; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int ch = (lane + 32 * k) * 8 + j;
      wl[k][j] = ch < c ? __ldg(wts + ch) : 0.f;
    }
  double acc = 0.0;
  const int hw = h * w;
  for (int p = blockIdx.x * kHeadWarps + warp; p < hw; p += gridDim.x * kHeadWarps) {
    const int py = p / w, px = p - py * w;
    const size_t pix = ((size_t)(y0 + py) * xw + (x0 + px)) * chunks;
    const uint4* a = reinterpret_cast<const uint4*>(f) + (size_t)i0 * xh * xw * chunks + pix;
    const uint4* b = reinterpret_cast<const uint4*>(f) + (size_t)i1 * xh * xw * chunks + pix;
    float va[kHeadMaxChunks][8], vb[kHeadMaxChunks][8];
    float sa = 0.f, sb = 0.f;
#pragma unroll
    for (int k = 0; k < kHeadMaxChunks; ++k) {
      if (k > 0 && chunks <= 32) break;    // warp-uniform: 256 channels or fewer fit in one chunk per lane
      const int q = lane + 32 * k;
      uint4 ua = make_uint4(0u, 0u, 0u, 0u), ub = ua;
      if (q < chunks) { ua = __ldg(a + q); ub = __ldg(b + q); }
      const __half2* ha = reinterpret_cast<const __half2*>(&ua);
      const __half2* hb = reinterpret_cast<const __half2*>(&ub);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 fa = __half22float2(ha[j]), fb = __half22float2(hb[j]);
        va[k][2 * j] = fa.x; va[k][2 * j + 1] = fa.y;
        vb[k][2 * j] = fb.x; vb[k][2 * j + 1] = fb.y;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) { sa += va[k][j] * va[k][j]; sb += vb[k][j] * vb[k][j]; }
    }
    sa = warp_sum(sa);
    sb = warp_sum(sb);
    const float ra = 1.f / (sqrtf(sa) + 1e-10f), rb = 1.f / (sqrtf(sb) + 1e-10f);
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < kHeadMaxChunks; ++k) {
      if (k > 0 && chunks <= 32) break;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float dlt = __fmul_rn(va[k][j], ra) - __fmul_rn(vb[k][j], rb);   // no FMA: d(a, b) = d(b, a), d(a, a) = 0
        s += wl[k][j] * dlt * dlt;
      }
    }
    acc += (double)warp_sum(s);
  }
  if (lane == 0) part[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int k = 0; k < kHeadWarps; ++k) t += part[k];
    work[(size_t)pair * gridDim.x + blockIdx.x] = t;
  }
}

// out[pair] (+)= the sum of the pair's CTA partials in CTA order / (h w)
__global__ void lpips_head_finish_kernel(const double* __restrict__ work, int npairs, int blocks, double hw,
                                         int accumulate, double* __restrict__ out) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int pair = blockIdx.x * blockDim.x + threadIdx.x;
  if (pair >= npairs) return;
  double t = 0.0;
  for (int k = 0; k < blocks; ++k) t += work[(size_t)pair * blocks + k];
  t /= hw;
  out[pair] = accumulate ? out[pair] + t : t;
}

int head_blocks(int h, int w) {
  const long long px = (long long)h * w;
  long long b = (px + 8LL * kHeadWarps - 1) / (8LL * kHeadWarps);     // about 8 pixels per warp
  if (b > kHeadMaxBlocks) b = kHeadMaxBlocks;
  return b < 1 ? 1 : (int)b;
}

int grid_for(size_t total) {
  size_t g = (total + kThreads - 1) / kThreads;
  const size_t cap = (size_t)tg_sms() * 16;
  if (g > cap) g = cap;
  return g < 1 ? 1 : (int)g;
}

}  // namespace

extern "C" {

int tg_lpips_frames_in(const uint8_t* frames, const tg_frame_window* win, int t, int h, int w, int norm, void* out,
                       void* stream) {
  TG_REQUIRE(frames && win && out, TG_E_INVALID, "lpips_frames_in: null pointer");
  TG_REQUIRE(t > 0 && h > 0 && w > 0, TG_E_INVALID, "lpips_frames_in: bad size t=%d h=%d w=%d", t, h, w);
  TG_REQUIRE(norm == TG_LPIPS_NORM_CALC || norm == TG_LPIPS_NORM_OFFICIAL, TG_E_INVALID,
             "lpips_frames_in: norm %d", norm);
  TG_REQUIRE(win->frame_h > 0 && win->frame_w > 0 && win->top >= 0 && win->left >= 0 &&
                 win->top + h <= win->frame_h && win->left + w <= win->frame_w,
             TG_E_INVALID, "lpips_frames_in: the %dx%d picture at (%d, %d) lies outside the %dx%d frame", h, w, win->top,
             win->left, win->frame_h, win->frame_w);
  TG_REQUIRE(h >= TG_LPIPS_MIN_SIDE && w >= TG_LPIPS_MIN_SIDE, TG_E_UNSUPPORTED,
             "lpips_frames_in: %dx%d is below %dx%d", h, w, TG_LPIPS_MIN_SIDE, TG_LPIPS_MIN_SIDE);
  TG_REQUIRE(((uintptr_t)out & 15) == 0, TG_E_INVALID, "lpips_frames_in: out must be 16-byte aligned");
  const int hs = (h - 7) / 4 + 3, ws = (w - 7) / 4 + 3;
  tg_launch(lpips_frames_in_kernel, dim3(grid_for((size_t)t * hs * ws * 8)), dim3(kThreads), 0, (cudaStream_t)stream,
            frames, *win, t, h, w, hs, ws, norm, (__half*)out);
  TG_CUDA_LAUNCH_CHECK("lpips_frames_in");
  return TG_OK;
}

int tg_maxpool3x3s2_nhwc_f16(const void* x, int n, int xh, int xw, int c, int y0, int x0, int h, int w, void* y,
                             int shifts, void* stream) {
  TG_REQUIRE(x && y, TG_E_INVALID, "maxpool3x3s2: null pointer");
  TG_REQUIRE(n > 0 && xh > 0 && xw > 0 && c > 0 && c % 8 == 0, TG_E_INVALID,
             "maxpool3x3s2: bad size n=%d %dx%d c=%d (a multiple of 8)", n, xh, xw, c);
  TG_REQUIRE(h >= 3 && w >= 3 && y0 >= 0 && x0 >= 0 && y0 + h <= xh && x0 + w <= xw, TG_E_INVALID,
             "maxpool3x3s2: the %dx%d interior at (%d, %d) of %dx%d (at least 3x3 inside)", h, w, y0, x0, xh, xw);
  TG_REQUIRE((((uintptr_t)x | (uintptr_t)y) & 15) == 0, TG_E_INVALID, "maxpool3x3s2: pointers must be 16-byte aligned");
  const int ph = (h - 3) / 2 + 1, pw = (w - 3) / 2 + 1;
  const size_t out_px = shifts ? (size_t)(ph + 2) * (pw + 2) * 4 : (size_t)ph * pw;
  tg_launch(maxpool3x3s2_kernel, dim3(grid_for((size_t)n * out_px * (c / 8))), dim3(kThreads), 0,
            (cudaStream_t)stream, (const __half*)x, n, xh, xw, c, y0, x0, ph, pw, shifts ? 1 : 0, (__half*)y);
  TG_CUDA_LAUNCH_CHECK("maxpool3x3s2");
  return TG_OK;
}

size_t tg_lpips_head_workspace_bytes(int npairs, int h, int w) {
  if (npairs <= 0 || h <= 0 || w <= 0) return 0;
  return (size_t)npairs * head_blocks(h, w) * sizeof(double);
}

int tg_lpips_head(const void* feat, int n, int xh, int xw, int c, int y0, int x0, int h, int w, const int32_t* pairs,
                  int npairs, const float* weights, int accumulate, double* out, void* work, size_t work_bytes,
                  void* stream) {
  TG_REQUIRE(feat && pairs && weights && out && work, TG_E_INVALID, "lpips_head: null pointer");
  TG_REQUIRE(n > 0 && npairs > 0 && xh > 0 && xw > 0, TG_E_INVALID, "lpips_head: bad size n=%d pairs=%d %dx%d", n,
             npairs, xh, xw);
  TG_REQUIRE(c > 0 && c % 8 == 0 && c <= kHeadMaxChunks * 32 * 8, TG_E_UNSUPPORTED,
             "lpips_head: c=%d (a multiple of 8, at most %d)", c, kHeadMaxChunks * 32 * 8);
  TG_REQUIRE(h > 0 && w > 0 && y0 >= 0 && x0 >= 0 && y0 + h <= xh && x0 + w <= xw, TG_E_INVALID,
             "lpips_head: the %dx%d interior at (%d, %d) lies outside %dx%d", h, w, y0, x0, xh, xw);
  TG_REQUIRE(npairs <= 65535, TG_E_UNSUPPORTED, "lpips_head: %d pairs (at most 65535)", npairs);
  TG_REQUIRE(((uintptr_t)feat & 15) == 0 && ((uintptr_t)pairs & 3) == 0 && ((uintptr_t)weights & 3) == 0 &&
                 ((uintptr_t)out & 7) == 0 && ((uintptr_t)work & 7) == 0,
             TG_E_INVALID, "lpips_head: misaligned pointer");
  TG_REQUIRE(work_bytes >= tg_lpips_head_workspace_bytes(npairs, h, w), TG_E_INVALID,
             "lpips_head: workspace of %zu bytes, %zu needed", work_bytes, tg_lpips_head_workspace_bytes(npairs, h, w));
  const int blocks = head_blocks(h, w);
  cudaStream_t st = (cudaStream_t)stream;
  tg_launch(lpips_head_kernel, dim3(blocks, npairs), dim3(kThreads), 0, st, (const __half*)feat, n, xh, xw, c, y0, x0, h,
            w, pairs, weights, (double*)work);
  TG_CUDA_LAUNCH_CHECK("lpips_head");
  tg_launch(lpips_head_finish_kernel, dim3(tg_ceil_div(npairs, 128)), dim3(128), 0, st, (const double*)work, npairs,
            blocks, (double)h * w, accumulate ? 1 : 0, out);
  TG_CUDA_LAUNCH_CHECK("lpips_head_finish");
  return TG_OK;
}

}  // extern "C"
