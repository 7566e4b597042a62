// Antialiased bicubic / Lanczos-3 resize of the streamed HR frame (fp32 NCHW) to the output size, written as uint8
// NHWC (quantised like float32_to_uint8) or fp32 NCHW (the source of the 10-bit encodes), and the host-side builder
// of its per-axis tables.  The filters are Pillow's (Image.resize on 'F' images); oracle/resample.py specifies them.
// Contract: include/tecogan_b200.h (tg_resample_taps, tg_resample_table, tg_resample_nchw_f32).
#include <math.h>

#include "tg_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kTY = 16, kTX = 64;            // output tile of one CTA: kTY rows x kTX columns, every channel
constexpr int kMaxTaps = 25;                 // lanczos at a 1/4 downscale: 2 * ceil(3 * 4) + 1
constexpr int kMaxC = 4;
constexpr int kOutRow = kTX * kMaxC + 16;    // staged uint8 row: the destination's 16-byte lead, then the pixels
// the vertical pass's columns of one tile: first[last] - first[0] + taps <= ceil((kTX - 1) * in / out) + 1 + taps
constexpr int kMaxSpan = (kTX - 1) * 4 + 2 + kMaxTaps;
constexpr int kMaxMidBytes = kMaxC * kTY * kMaxSpan * (int)sizeof(float);

int span_cap(int in, int out, int taps) { return (int)(((long long)(kTX - 1) * in + out - 1) / out) + 2 + taps; }

// One CTA: output rows [oy0, oy0 + kTY) x columns [ox0, ox0 + kTX) of image `img`, all c channels.
//  1. vertical pass: for every input column the tile's horizontal windows cover ([base, base + span)), every channel
//     and every output row, mid = sum_q row_w[q] * x[row_first + q][col] -- coalesced row reads (L1 / L2 serve the
//     rows neighbouring outputs share), fp32 results in shared memory;
//  2. horizontal pass: y = sum_q col_w[q] * mid[col_first + q - base] from shared memory.
// Both sums run in tap order with fmaf, so an output's value does not depend on the grid.  Every row and column
// index is clamped into the image (padding taps have weight 0) and into the staged span.
template <bool kU8>
__global__ void __launch_bounds__(kThreads)
resample_kernel(const float* __restrict__ x, int c, int H, int W, const int32_t* __restrict__ row_first,
                const float* __restrict__ row_w, int row_taps, const int32_t* __restrict__ col_first,
                const float* __restrict__ col_w, int col_taps, int Ho, int Wo, int tiles_x, int tiles_y, int cap,
                uint8_t* __restrict__ y_u8, float* __restrict__ y_f32) {
  __shared__ float s_rw[kTY * kMaxTaps];
  __shared__ float s_cw[kTX * kMaxTaps];
  __shared__ int s_rf[kTY], s_cf[kTX];
  __shared__ __align__(16) uint8_t s_out[kU8 ? kTY : 1][kU8 ? kOutRow : 16];
  extern __shared__ float s_mid[];           // [c][kTY][cap]
  const int t = threadIdx.x;
  const int tx = blockIdx.x % tiles_x, rest = blockIdx.x / tiles_x;
  const int ty = rest % tiles_y, img = rest / tiles_y;
  const int ox0 = tx * kTX, oy0 = ty * kTY;
  const int nx = min(kTX, Wo - ox0), ny = min(kTY, Ho - oy0);
  // the tables stay the same for the whole stream: staged before waiting on the previous kernel
  for (int i = t; i < ny * row_taps; i += kThreads) s_rw[i] = __ldg(row_w + (size_t)oy0 * row_taps + i);
  for (int i = t; i < nx * col_taps; i += kThreads) s_cw[i] = __ldg(col_w + (size_t)ox0 * col_taps + i);
  if (t < ny) s_rf[t] = __ldg(row_first + oy0 + t);
  if (t < nx) s_cf[t] = __ldg(col_first + ox0 + t);
  // x is the previous kernel's output; y may still be read by the copy of an earlier step
  tg_pdl_wait();
  tg_pdl_trigger();
  __syncthreads();
  const int base = min(max(s_cf[0], 0), W - 1);
  const int span = max(min(s_cf[nx - 1] - base + col_taps, cap), 1);

  const size_t plane = (size_t)H * W;
  const float* src = x + (size_t)img * c * plane;
  // items (channel, output row, column), columns fastest: consecutive threads read consecutive addresses.  Two
  // items per thread and iteration, so that both windows' loads are in flight together.
  const int items = c * ny * span;
  for (int i0 = t; i0 < items; i0 += 2 * kThreads) {
    const int i1 = min(i0 + kThreads, items - 1);
    const float *p[2], *w[2];
    int f[2], dst[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int i = u ? i1 : i0;
      const int kr = i / span, j = i - kr * span;
      const int k = kr / ny, r = kr - k * ny;
      p[u] = src + k * plane + min(base + j, W - 1);
      w[u] = s_rw + r * row_taps;
      f[u] = s_rf[r];
      dst[u] = (k * kTY + r) * cap + j;
    }
    float acc0 = 0.f, acc1 = 0.f;
#pragma unroll 4
    for (int q = 0; q < row_taps; ++q) {
      const float x0 = __ldg(p[0] + (size_t)min(max(f[0] + q, 0), H - 1) * W);
      const float x1 = __ldg(p[1] + (size_t)min(max(f[1] + q, 0), H - 1) * W);
      acc0 = fmaf(w[0][q], x0, acc0);
      acc1 = fmaf(w[1][q], x1, acc1);
    }
    s_mid[dst[0]] = acc0;
    if (i0 + kThreads < items) s_mid[dst[1]] = acc1;
  }
  __syncthreads();

  for (int i = t; i < ny * nx; i += kThreads) {
    const int r = i / nx, xo = i - r * nx;
    const int off = s_cf[xo] - base;
    const float* w = s_cw + xo * col_taps;
    for (int k = 0; k < c; ++k) {
      const float* mid = s_mid + (k * kTY + r) * cap;
      float acc = 0.f;
      for (int q = 0; q < col_taps; ++q) acc = fmaf(w[q], mid[min(max(off + q, 0), span - 1)], acc);
      if constexpr (kU8) {
        const int lead = (int)((uintptr_t)(y_u8 + (((size_t)img * Ho + oy0 + r) * Wo + ox0) * c) & 15u);
        s_out[r][lead + xo * c + k] = (uint8_t)fminf(fmaxf(rintf(acc * 255.f), 0.f), 255.f);
      } else {
        y_f32[(((size_t)img * c + k) * Ho + oy0 + r) * Wo + ox0 + xo] = acc;
      }
    }
  }
  if constexpr (kU8) {
    // each row of the tile is one contiguous run of nx * c bytes: 16-byte stores over its aligned interior, single
    // bytes at the ends, nothing outside the run; a warp per row
    __syncthreads();
    const int warp = t >> 5, lane = t & 31;
    const int bytes = nx * c;
    for (int r = warp; r < ny; r += kThreads / 32) {
      uint8_t* dst = y_u8 + (((size_t)img * Ho + oy0 + r) * Wo + ox0) * c;
      const int lead = (int)((uintptr_t)dst & 15u);
      const int a0 = min(lead ? 16 - lead : 0, bytes);
      const int nv = (bytes - a0) / 16;
      const int tail0 = a0 + 16 * nv;
      const uint8_t* sb = s_out[r] + lead;
      for (int v = lane; v < nv; v += 32)
        reinterpret_cast<uint4*>(dst + a0)[v] = *reinterpret_cast<const uint4*>(sb + a0 + 16 * v);
      if (lane < a0) dst[lane] = sb[lane];
      if (tail0 + lane < bytes) dst[tail0 + lane] = sb[tail0 + lane];
    }
  }
}

// ---------------------------------------------------------------- host: Pillow's filters and window placement
double filter_support(int filter) { return filter == TG_RESAMPLE_BICUBIC ? 2.0 : 3.0; }

double k_bicubic(double x) {
  const double a = -0.5;
  x = fabs(x);
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1.0;
  if (x < 2.0) return (((x - 5.0) * x + 8.0) * x - 4.0) * a;
  return 0.0;
}

double k_sinc(double x) {
  if (x == 0.0) return 1.0;
  x = x * M_PI;
  return sin(x) / x;
}

double k_lanczos(double x) { return (-3.0 <= x && x < 3.0) ? k_sinc(x) * k_sinc(x / 3.0) : 0.0; }

int check_axis(const char* name, int in, int out, int filter) {
  TG_REQUIRE(in > 0 && out > 0, TG_E_INVALID, "%s: bad size %d -> %d", name, in, out);
  TG_REQUIRE(filter == TG_RESAMPLE_BICUBIC || filter == TG_RESAMPLE_LANCZOS3, TG_E_UNSUPPORTED,
             "%s: unknown filter %d", name, filter);
  TG_REQUIRE(4ll * out >= in && out <= 2ll * in, TG_E_UNSUPPORTED,
             "%s: %d -> %d is outside the supported ratios (in/4 <= out <= 2*in)", name, in, out);
  return TG_OK;
}

int taps_of(int in, int out, int filter) {
  const double scale = (double)in / out;
  return 2 * (int)ceil(filter_support(filter) * (scale > 1.0 ? scale : 1.0)) + 1;
}

}  // namespace

extern "C" int tg_resample_taps(int in, int out, int filter, int* taps) {
  TG_REQUIRE(taps, TG_E_INVALID, "resample_taps: null pointer (taps)");
  const int rc = check_axis("resample_taps", in, out, filter);
  if (rc != TG_OK) return rc;
  *taps = taps_of(in, out, filter);
  return TG_OK;
}

extern "C" int tg_resample_table(int in, int out, int filter, int taps, int32_t* first, float* weights) {
  const char* name = "resample_table";
  TG_REQUIRE(first && weights, TG_E_INVALID, "%s: null pointer (first / weights)", name);
  const int rc = check_axis(name, in, out, filter);
  if (rc != TG_OK) return rc;
  const int need = taps_of(in, out, filter);
  TG_REQUIRE(taps == need, TG_E_INVALID, "%s: taps %d, %d -> %d needs %d", name, taps, in, out, need);
  const double scale = (double)in / out;
  const double fs = scale > 1.0 ? scale : 1.0;
  const double support = filter_support(filter) * fs;
  const double ss = 1.0 / fs;
  double w[kMaxTaps + 1];
  for (int o = 0; o < out; ++o) {
    const double center = (o + 0.5) * scale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in) xmax = in;
    const int len = xmax - xmin;
    TG_REQUIRE(len >= 1 && len <= taps, TG_E_INVALID, "%s: window of %d taps at %d (internal)", name, len, o);
    double tot = 0.0;
    for (int i = 0; i < len; ++i) {
      const double v = (double)(xmin + i) - center + 0.5;
      w[i] = filter == TG_RESAMPLE_BICUBIC ? k_bicubic(v * ss) : k_lanczos(v * ss);
      tot += w[i];
    }
    if (tot != 0.0)
      for (int i = 0; i < len; ++i) w[i] /= tot;
    // the window ends inside the axis where it fits, so the zero-weight padding taps index the image
    int f = xmin < in - taps ? xmin : in - taps;
    if (f < 0) f = 0;
    first[o] = f;
    float* row = weights + (size_t)o * taps;
    for (int i = 0; i < taps; ++i) row[i] = 0.f;
    for (int i = 0; i < len; ++i) row[xmin - f + i] = (float)w[i];
  }
  return TG_OK;
}

extern "C" int tg_resample_nchw_f32(const float* x, int n, int c, int H, int W, const int32_t* row_first,
                                    const float* row_w, int row_taps, const int32_t* col_first, const float* col_w,
                                    int col_taps, int Ho, int Wo, uint8_t* y_u8, float* y_f32, void* stream) {
  const char* name = "resample_nchw_f32";
  TG_REQUIRE(x && row_first && row_w && col_first && col_w, TG_E_INVALID,
             "%s: null pointer (x / row_first / row_w / col_first / col_w)", name);
  TG_REQUIRE((y_u8 != nullptr) != (y_f32 != nullptr), TG_E_INVALID, "%s: exactly one of y_u8 / y_f32 is written",
             name);
  TG_REQUIRE(n > 0 && c > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0, TG_E_INVALID,
             "%s: bad size n=%d c=%d %dx%d -> %dx%d", name, n, c, H, W, Ho, Wo);
  TG_REQUIRE(c <= kMaxC, TG_E_INVALID, "%s: %d channels (at most %d)", name, c, kMaxC);
  TG_REQUIRE(row_taps > 0 && col_taps > 0, TG_E_INVALID, "%s: bad taps %d / %d", name, row_taps, col_taps);
  TG_REQUIRE((((uintptr_t)x | (uintptr_t)row_first | (uintptr_t)row_w | (uintptr_t)col_first | (uintptr_t)col_w |
               (uintptr_t)y_f32) & 3u) == 0,
             TG_E_INVALID, "%s: x, the tables and y_f32 must be 4-byte aligned", name);
  TG_REQUIRE(4ll * Ho >= H && Ho <= 2ll * H && 4ll * Wo >= W && Wo <= 2ll * W, TG_E_UNSUPPORTED,
             "%s: %dx%d -> %dx%d is outside the supported ratios (in/4 <= out <= 2*in per axis)", name, H, W, Ho, Wo);
  TG_REQUIRE(row_taps <= kMaxTaps && col_taps <= kMaxTaps, TG_E_UNSUPPORTED, "%s: taps %d / %d (at most %d)", name,
             row_taps, col_taps, kMaxTaps);
  const int tiles_x = tg_ceil_div(Wo, kTX), tiles_y = tg_ceil_div(Ho, kTY);
  const size_t ctas = (size_t)tiles_x * tiles_y * n;
  TG_REQUIRE(ctas <= 0x7fffffff, TG_E_UNSUPPORTED, "%s: grid too large", name);
  const int cap = span_cap(W, Wo, col_taps);
  const size_t smem = (size_t)c * kTY * cap * sizeof(float);
  const cudaStream_t st = (cudaStream_t)stream;
  if (y_u8) {
    static TgPerDeviceOnce attr_once;
    const cudaError_t e = attr_once.run([] {
      return cudaFuncSetAttribute(resample_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxMidBytes);
    });
    TG_REQUIRE(e == cudaSuccess, (int)e, "%s: cudaFuncSetAttribute: %s", name, cudaGetErrorString(e));
    tg_launch(resample_kernel<true>, dim3((unsigned)ctas), dim3(kThreads), smem, st, x, c, H, W, row_first, row_w,
              row_taps, col_first, col_w, col_taps, Ho, Wo, tiles_x, tiles_y, cap, y_u8, (float*)nullptr);
  } else {
    static TgPerDeviceOnce attr_once;
    const cudaError_t e = attr_once.run([] {
      return cudaFuncSetAttribute(resample_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxMidBytes);
    });
    TG_REQUIRE(e == cudaSuccess, (int)e, "%s: cudaFuncSetAttribute: %s", name, cudaGetErrorString(e));
    tg_launch(resample_kernel<false>, dim3((unsigned)ctas), dim3(kThreads), smem, st, x, c, H, W, row_first, row_w,
              row_taps, col_first, col_w, col_taps, Ho, Wo, tiles_x, tiles_y, cap, (uint8_t*)nullptr, y_f32);
  }
  TG_CUDA_LAUNCH_CHECK(name);
  return TG_OK;
}
