// Antialiased bicubic / Lanczos-3 resize of the streamed HR frame (fp32 NCHW) to the output size, written as uint8
// NHWC (quantised like float32_to_uint8) or fp32 NCHW (the source of the 10-bit encodes), and the host-side builder
// of its per-axis tables.  The filters are Pillow's (Image.resize on 'F' images); oracle/resample.py specifies them.
// The uint8 output can be a picture window of larger frames (tg_frame_window).  The same tiles resize the streamed
// input: the frame-input launch's decode of the source picture (tg_frame_decode.cuh) read in place of the fp32 frame,
// fp32 LR frame out, with the per-slot reset of tg_stream_frame_in in the same launch.
// Contract: include/tecogan_b200.h (tg_resample_taps, tg_resample_table, tg_resample_nchw_f32[_window],
// tg_stream_frame_in_resample).
#include <math.h>

#include "tg_common.cuh"
#include "tg_frame_decode.cuh"     // also kThreads (256) and kMaxC (4)

namespace {

constexpr int kTY = 16, kTX = 64;            // output tile of one CTA: kTY rows x kTX columns, every channel
constexpr int kMaxTaps = 25;                 // lanczos at a 1/4 downscale: 2 * ceil(3 * 4) + 1
constexpr int kOutRow = kTX * kMaxC + 16;    // staged uint8 row: the destination's 16-byte lead, then the pixels
// the vertical pass's columns of one tile: first[last] - first[0] + taps <= ceil((kTX - 1) * in / out) + 1 + taps
constexpr int kMaxSpan = (kTX - 1) * 4 + 2 + kMaxTaps;
constexpr int kMaxMidBytes = kMaxC * kTY * kMaxSpan * (int)sizeof(float);

int span_cap(int in, int out, int taps) { return (int)(((long long)(kTX - 1) * in + out - 1) / out) + 2 + taps; }

// Sources of the vertical pass.  An item of the pass is one column of one output row for kC channels: col() names
// the column (channel group k, source column xc, already clamped), read() gives its kC values at source row y.
// fp32 NCHW x [n,c,H,W] (the streamed HR frame): one channel per item.
struct NchwSource {
  // kC channels per item, kItems items per thread and iteration, the vertical pass's taps unrolled kUnroll times
  static constexpr int kC = 1, kItems = 2, kUnroll = 4;
  using Col = const float*;
  const float* x;
  int c, H, W;
  __device__ __forceinline__ Col col(int img, int k, int xc) const { return x + ((size_t)img * c + k) * H * W + xc; }
  __device__ __forceinline__ void read(Col p, int y, float* v) const { v[0] = __ldg(p + (size_t)y * W); }
};

// The H x W picture at `win` of stored frames of layout kFmt, decoded as the frame input decodes it (decode_pixel):
// every channel of a pixel per item, so a source pixel is decoded once per tap, not once per channel.
template <int kFmt>
struct FrameSource {
  static constexpr int kC = kMaxC, kItems = 1, kUnroll = 1;   // no spills around the decode's divisions
  struct Col {
    int img, x;
  };
  const uint8_t* in;
  tg_frame_window win;
  int c, bgr, color;
  __device__ __forceinline__ Col col(int img, int, int xc) const { return Col{img, xc}; }
  __device__ __forceinline__ void read(Col p, int y, float* v) const {
    decode_pixel<kFmt>(in, win, c, bgr, color, p.img, y, p.x, v);
  }
};

// One CTA (b of the resize's CTAs): output rows [oy0, oy0 + kTY) x columns [ox0, ox0 + kTX) of image `img`, all c
// channels.
//  1. vertical pass: for every input column the tile's horizontal windows cover ([base, base + span)), every channel
//     and every output row, mid = sum_q row_w[q] * x[row_first + q][col] -- coalesced row reads (L1 / L2 serve the
//     rows neighbouring outputs share), fp32 results in shared memory;
//  2. horizontal pass: y = sum_q col_w[q] * mid[col_first + q - base] from shared memory.
// Both sums run in tap order with fmaf, so an output's value does not depend on the grid or on the source (an fp32
// frame, or the decode that would have written it).  Every row and column index is clamped into the image (padding
// taps have weight 0) and into the staged span.
template <bool kU8, class Src>
__device__ __forceinline__ void resample_tile(const Src& src, int b, int c, int H, int W,
                                              const int32_t* __restrict__ row_first, const float* __restrict__ row_w,
                                              int row_taps, const int32_t* __restrict__ col_first,
                                              const float* __restrict__ col_w, int col_taps, int Ho, int Wo,
                                              int tiles_x, int tiles_y, int cap, uint8_t* __restrict__ y_u8,
                                              tg_frame_window win, float* __restrict__ y_f32) {
  constexpr int kC = Src::kC;
  __shared__ float s_rw[kTY * kMaxTaps];
  __shared__ float s_cw[kTX * kMaxTaps];
  __shared__ int s_rf[kTY], s_cf[kTX];
  __shared__ __align__(16) uint8_t s_out[kU8 ? kTY : 1][kU8 ? kOutRow : 16];
  extern __shared__ float s_mid[];           // [c][kTY][cap]
  const int t = threadIdx.x;
  const int tx = b % tiles_x, rest = b / tiles_x;
  const int ty = rest % tiles_y, img = rest / tiles_y;
  const int ox0 = tx * kTX, oy0 = ty * kTY;
  const int nx = min(kTX, Wo - ox0), ny = min(kTY, Ho - oy0);
  // uint8 output: pixel (y, x) of the picture is pixel (top + y, left + x) of its frame
  const auto out_px = [&](int im, int y, int x) {
    return ((size_t)im * win.frame_h + win.top + y) * win.frame_w + win.left + x;
  };
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

  // items (channel group, output row, column), columns fastest: consecutive threads read consecutive addresses.
  // kI items per thread and iteration, so that their windows' loads are in flight together.
  constexpr int kI = Src::kItems;
  const int items = (kC == 1 ? c : 1) * ny * span;
  for (int i0 = t; i0 < items; i0 += kI * kThreads) {
    typename Src::Col p[kI];
    const float* w[kI];
    int f[kI], dst[kI];
#pragma unroll
    for (int u = 0; u < kI; ++u) {
      const int i = u ? min(i0 + u * kThreads, items - 1) : i0;
      const int kr = i / span, j = i - kr * span;
      const int k = kr / ny, r = kr - k * ny;
      p[u] = src.col(img, k, min(base + j, W - 1));
      w[u] = s_rw + r * row_taps;
      f[u] = s_rf[r];
      dst[u] = (k * kTY + r) * cap + j;
    }
    float acc[kI][kC];
#pragma unroll
    for (int u = 0; u < kI; ++u)
#pragma unroll
      for (int k = 0; k < kC; ++k) acc[u][k] = 0.f;
#pragma unroll Src::kUnroll
    for (int q = 0; q < row_taps; ++q) {
      float x[kI][kC] = {};
#pragma unroll
      for (int u = 0; u < kI; ++u) src.read(p[u], min(max(f[u] + q, 0), H - 1), x[u]);
#pragma unroll
      for (int u = 0; u < kI; ++u)
#pragma unroll
        for (int k = 0; k < kC; ++k) acc[u][k] = fmaf(w[u][q], x[u][k], acc[u][k]);
    }
#pragma unroll
    for (int k = 0; k < kC; ++k) {
      if (k >= c) break;
#pragma unroll
      for (int u = 0; u < kI; ++u)
        if (u == 0 || i0 + u * kThreads < items) s_mid[dst[u] + k * kTY * cap] = acc[u][k];
    }
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
        const int lead = (int)((uintptr_t)(y_u8 + out_px(img, oy0 + r, ox0) * c) & 15u);
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
      uint8_t* dst = y_u8 + out_px(img, oy0 + r, ox0) * c;
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

// the output resize: one CTA per tile of the fp32 NCHW frame x
template <bool kU8>
__global__ void __launch_bounds__(kThreads)
resample_kernel(const float* __restrict__ x, int c, int H, int W, const int32_t* __restrict__ row_first,
                const float* __restrict__ row_w, int row_taps, const int32_t* __restrict__ col_first,
                const float* __restrict__ col_w, int col_taps, int Ho, int Wo, int tiles_x, int tiles_y, int cap,
                uint8_t* __restrict__ y_u8, tg_frame_window win, float* __restrict__ y_f32) {
  resample_tile<kU8>(NchwSource{x, c, H, W}, blockIdx.x, c, H, W, row_first, row_w, row_taps, col_first, col_w,
                     col_taps, Ho, Wo, tiles_x, tiles_y, cap, y_u8, win, y_f32);
}

// The resizing frame input.  blockIdx.x < resize_ctas: a tile of lr_curr [n,c,Ho,Wo] resized from the decoded source
// picture; the rest: zpc CTAs per slot, each zeroing a strided share of that slot's lr_prev and hr_prev when flagged
// (stream_frame_in_kernel's reset).
template <int kFmt>
__global__ void __launch_bounds__(kThreads)
frame_in_resample_kernel(FrameSource<kFmt> src, int H, int W, const int32_t* __restrict__ row_first,
                         const float* __restrict__ row_w, int row_taps, const int32_t* __restrict__ col_first,
                         const float* __restrict__ col_w, int col_taps, int Ho, int Wo, int tiles_x, int tiles_y,
                         int cap, float* __restrict__ lr_curr, const int32_t* __restrict__ reset,
                         float* __restrict__ lr_prev, float* __restrict__ hr_prev, int s, int resize_ctas, int zpc) {
  const int b = blockIdx.x, c = src.c;
  if (b < resize_ctas) {
    resample_tile<false>(src, b, c, H, W, row_first, row_w, row_taps, col_first, col_w, col_taps, Ho, Wo, tiles_x,
                         tiles_y, cap, nullptr, tg_frame_window{Ho, Wo, 0, 0}, lr_curr);
    return;
  }
  // lr_prev and hr_prev belong to the previous step until it has finished
  tg_pdl_wait();
  tg_pdl_trigger();
  const int rb = b - resize_ctas;
  const int slot = rb / zpc, part = rb - slot * zpc;
  if (__ldg(reset + slot) == 0) return;
  const size_t nlr = (size_t)c * Ho * Wo, nhr = nlr * s * s;
  const size_t worker = (size_t)part * kThreads + threadIdx.x, workers = (size_t)zpc * kThreads;
  zero_range(lr_prev + slot * nlr, nlr, worker, workers);
  zero_range(hr_prev + slot * nhr, nhr, worker, workers);
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

namespace {

int resample(const char* name, const float* x, int n, int c, int H, int W, const int32_t* row_first,
             const float* row_w, int row_taps, const int32_t* col_first, const float* col_w, int col_taps, int Ho,
             int Wo, uint8_t* y_u8, const tg_frame_window* win, float* y_f32, void* stream) {
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
  const tg_frame_window whole = {Ho, Wo, 0, 0};
  if (!win) win = &whole;
  TG_REQUIRE(win->frame_h > 0 && win->frame_w > 0 && win->top >= 0 && win->left >= 0 &&
                 (long long)win->top + Ho <= win->frame_h && (long long)win->left + Wo <= win->frame_w,
             TG_E_INVALID, "%s: a %dx%d picture at (%d, %d) does not fit a %dx%d frame", name, Ho, Wo, win->top,
             win->left, win->frame_h, win->frame_w);
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
              row_taps, col_first, col_w, col_taps, Ho, Wo, tiles_x, tiles_y, cap, y_u8, *win, (float*)nullptr);
  } else {
    static TgPerDeviceOnce attr_once;
    const cudaError_t e = attr_once.run([] {
      return cudaFuncSetAttribute(resample_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxMidBytes);
    });
    TG_REQUIRE(e == cudaSuccess, (int)e, "%s: cudaFuncSetAttribute: %s", name, cudaGetErrorString(e));
    tg_launch(resample_kernel<false>, dim3((unsigned)ctas), dim3(kThreads), smem, st, x, c, H, W, row_first, row_w,
              row_taps, col_first, col_w, col_taps, Ho, Wo, tiles_x, tiles_y, cap, (uint8_t*)nullptr, *win, y_f32);
  }
  TG_CUDA_LAUNCH_CHECK(name);
  return TG_OK;
}

// one axis of the input resize: `in` -> `out` within the ratios, `taps` the bicubic or the Lanczos table's width
int check_input_axis(const char* name, const char* axis, int in, int out, int taps) {
  TG_REQUIRE(4ll * out >= in && out <= 2ll * in, TG_E_UNSUPPORTED,
             "%s: %s %d -> %d is outside the supported ratios (in/4 <= out <= 2*in)", name, axis, in, out);
  const int bicubic = taps_of(in, out, TG_RESAMPLE_BICUBIC), lanczos = taps_of(in, out, TG_RESAMPLE_LANCZOS3);
  TG_REQUIRE(taps == bicubic || taps == lanczos, TG_E_INVALID,
             "%s: %s table of %d taps, %d -> %d takes %d (bicubic) or %d (lanczos)", name, axis, taps, in, out,
             bicubic, lanczos);
  return TG_OK;
}

template <int kFmt>
int launch_frame_in_resample(const char* name, const void* in, const tg_frame_window* win, int bgr, int color, int h,
                             int w, const int32_t* row_first, const float* row_w, int row_taps,
                             const int32_t* col_first, const float* col_w, int col_taps, const int32_t* reset,
                             float* lr_curr, float* lr_prev, float* hr_prev, int n, int c, int hn, int wn, int s,
                             cudaStream_t stream) {
  TG_REQUIRE(in, TG_E_INVALID, "%s: null pointer (in)", name);
  TG_REQUIRE(lr_curr && lr_prev && hr_prev, TG_E_INVALID, "%s: null pointer (lr_curr / lr_prev / hr_prev)", name);
  TG_REQUIRE(row_first && row_w && col_first && col_w, TG_E_INVALID,
             "%s: null pointer (row_first / row_w / col_first / col_w)", name);
  TG_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0 && hn > 0 && wn > 0, TG_E_INVALID,
             "%s: bad size n=%d c=%d %dx%d -> %dx%d", name, n, c, h, w, hn, wn);
  TG_REQUIRE(c <= kMaxC, TG_E_UNSUPPORTED, "%s: %d channels (at most %d)", name, c, kMaxC);
  TG_REQUIRE(s == 2 || s == 4, TG_E_UNSUPPORTED, "%s: scale %d (2 or 4)", name, s);
  TG_REQUIRE((((uintptr_t)lr_curr | (uintptr_t)lr_prev | (uintptr_t)hr_prev | (uintptr_t)row_first |
               (uintptr_t)row_w | (uintptr_t)col_first | (uintptr_t)col_w) & 3u) == 0,
             TG_E_INVALID, "%s: fp32 buffers and the tables must be 4-byte aligned", name);
  int rc = check_frames<kFmt>(name, in, h, w, win, Yuv<kFmt>::kAlign);
  const tg_frame_window whole = {h, w, 0, 0};
  if (!win) win = &whole;
  if (rc == TG_OK) rc = check_input_axis(name, "rows", h, hn, row_taps);
  if (rc == TG_OK) rc = check_input_axis(name, "columns", w, wn, col_taps);
  if (rc != TG_OK) return rc;
  const int tiles_x = tg_ceil_div(wn, kTX), tiles_y = tg_ceil_div(hn, kTY);
  const size_t resize = (size_t)tiles_x * tiles_y * n;
  const size_t hr4 = (size_t)c * s * hn * s * wn / 4;
  const int zpc = reset ? (int)(hr4 / (kThreads * 8) + 1 < 64 ? hr4 / (kThreads * 8) + 1 : 64) : 0;
  const size_t ctas = resize + (size_t)zpc * n;
  TG_REQUIRE(ctas <= 0x7fffffff, TG_E_UNSUPPORTED, "%s: grid too large", name);
  const int cap = span_cap(w, wn, col_taps);
  const size_t smem = (size_t)c * kTY * cap * sizeof(float);
  static TgPerDeviceOnce attr_once;
  const cudaError_t e = attr_once.run([] {
    return cudaFuncSetAttribute(frame_in_resample_kernel<kFmt>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                kMaxMidBytes);
  });
  TG_REQUIRE(e == cudaSuccess, (int)e, "%s: cudaFuncSetAttribute: %s", name, cudaGetErrorString(e));
  const FrameSource<kFmt> src{static_cast<const uint8_t*>(in), *win, c, bgr, color};
  tg_launch(frame_in_resample_kernel<kFmt>, dim3((unsigned)ctas), dim3(kThreads), smem, stream, src, h, w, row_first,
            row_w, row_taps, col_first, col_w, col_taps, hn, wn, tiles_x, tiles_y, cap, lr_curr, reset, lr_prev,
            hr_prev, s, (int)resize, zpc);
  TG_CUDA_LAUNCH_CHECK(name);
  return TG_OK;
}

}  // namespace

extern "C" int tg_stream_frame_in_resample(const void* in, const tg_yuv_format* fmt, int bgr,
                                           const tg_frame_window* win, int h, int w, const int32_t* row_first,
                                           const float* row_w, int row_taps, const int32_t* col_first,
                                           const float* col_w, int col_taps, const int32_t* reset, float* lr_curr,
                                           float* lr_prev, float* hr_prev, int n, int c, int hn, int wn, int s,
                                           void* stream) {
  const char* name = "stream_frame_in_resample";
  int f = kHWC, color = 0;
  if (fmt) {
    const int rc = parse_yuv_format(name, fmt, &f, &color);
    if (rc != TG_OK) return rc;
    TG_REQUIRE(c == 3, TG_E_INVALID, "%s: YUV frames decode to 3 channels, got c=%d", name, c);
    TG_REQUIRE(bgr == 0, TG_E_INVALID, "%s: bgr applies to uint8 HWC frames only", name);
  }
  return dispatch_format(f, [&](auto k) {
    return launch_frame_in_resample<decltype(k)::value>(name, in, win, bgr, color, h, w, row_first, row_w, row_taps,
                                                        col_first, col_w, col_taps, reset, lr_curr, lr_prev, hr_prev,
                                                        n, c, hn, wn, s, (cudaStream_t)stream);
  });
}

extern "C" int tg_resample_nchw_f32(const float* x, int n, int c, int H, int W, const int32_t* row_first,
                                    const float* row_w, int row_taps, const int32_t* col_first, const float* col_w,
                                    int col_taps, int Ho, int Wo, uint8_t* y_u8, float* y_f32, void* stream) {
  return resample("resample_nchw_f32", x, n, c, H, W, row_first, row_w, row_taps, col_first, col_w, col_taps, Ho, Wo,
                  y_u8, nullptr, y_f32, stream);
}

extern "C" int tg_resample_nchw_f32_window(const float* x, int n, int c, int H, int W, const int32_t* row_first,
                                           const float* row_w, int row_taps, const int32_t* col_first,
                                           const float* col_w, int col_taps, int Ho, int Wo, uint8_t* y_u8,
                                           const tg_frame_window* win, void* stream) {
  TG_REQUIRE(win, TG_E_INVALID, "resample_nchw_f32_window: null window");
  TG_REQUIRE(y_u8, TG_E_INVALID, "resample_nchw_f32_window: null pointer (y_u8)");
  return resample("resample_nchw_f32_window", x, n, c, H, W, row_first, row_w, row_taps, col_first, col_w, col_taps,
                  Ho, Wo, y_u8, win, nullptr, stream);
}
