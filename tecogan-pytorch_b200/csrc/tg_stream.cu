// Frame I/O of one streamed inference step: uint8 HWC or YUV (4:2:0: NV12 / I420, 8 bit; P010 / I420_10, 10 bit;
// packed 4:2:2: YUY2 / UYVY, 8 bit; planar 4:4:4: I444, 8 bit, I444_10; 10-bit 4:2:2: P210, I422_10, v210) frames decoded on the device into the
// step's fp32 NCHW lr_curr, the per-slot reset of the recurrent state, and the encode of the step's RGB output
// (uint8 NHWC, or the fp32 NCHW HR frame for 10-bit output) into any of those YUV layouts; each of them reads or
// writes a picture window of larger stored frames (tg_frame_window).  Also the fill of padded frames with a format's
// black and the per-row / per-column luma sums of letterbox detection.
// Contract: include/tecogan_b200.h (tg_stream_frame_in[_window], tg_stream_frame_in_yuv420, tg_rgb_u8_to_yuv420,
// tg_stream_frame_in_yuv[_window], tg_rgb_to_yuv[_window], tg_yuv_coefficients, tg_fill_black, tg_luma_line_sums).
#include <type_traits>

#include "tg_common.cuh"
#include "tg_frame_decode.cuh"

namespace {

// Encode rows of 4:2:2: Y per pixel, U and V from the sum of the pair's two pixels,
//   Y = clip((kY . rgb + 2^(sy-1) + (yoff << sy)) >> sy)
//   C = clip((kC . (rgb0 + rgb1) + 2^(sc-1) + (coff << sc)) >> sc)
// i.e. the chroma of the pair's mean, rounded half up.  [depth 8 / 10][colour][kRY kGY kBY kRU kGU kBU kRV kGV kBV
// sy sc].  The 8-bit bt601 row is cv2's COLOR_RGB2YUV_YUY2 / _UYVY (14-bit constants of its own, luma included,
// with the chroma constants halved for the sum); the other rows are the table's encode rows with sy its shift (20
// at 8 bits, 18 at 10) and sc = sy + 1.  oracle/yuv_422_444.py and oracle/yuv_422_10.py specify the same rule.
struct Yuv422Enc {
  int v[2][4][11];
};

constexpr Yuv422Enc make_yuv422_enc() {
  Yuv422Enc e{};
  const int cv2[11] = {4211, 8258, 1606, -1212, -2384, 3596, 3596, -3015, -582, 14, 14};
  for (int di = 0; di < 2; ++di) {
    for (int ci = 0; ci < 4; ++ci) {
      int* r = e.v[di][ci];
      if (di == 0 && ci == 0) {
        for (int k = 0; k < 11; ++k) r[k] = cv2[k];
        continue;
      }
      for (int k = 0; k < 9; ++k) r[k] = kYuvTable.v[di][ci][k];
      r[9] = kYuvTable.v[di][ci][14];
      r[10] = kYuvTable.v[di][ci][14] + 1;
    }
  }
  return e;
}

__constant__ Yuv422Enc c_yuv422 = make_yuv422_enc();

// The encode of RGB codes into the samples of layout kFmt, colour row `color`:
//   Y = clip((kY . rgb + 2^(sy-1) + (yoff << sy)) >> sy),  C = clip((kC . rgb + 2^(sc-1) + (coff << sc)) >> sc)
// 4:2:0 and 4:4:4 with the table row (sy = sc = its shift), U and V of one pixel (4:2:0: a block's top-left, as cv2
// COLOR_RGB2YUV_I420); 4:2:2 with the c_yuv422 row, U and V of the sums of a pair's two pixels.
template <int kFmt>
struct YuvEncode {
  using F = Yuv<kFmt>;
  static constexpr bool kPairSum = F::k422;
  const int* k;
  int sy, sc, yo, co;
  __device__ __forceinline__ explicit YuvEncode(int color) {
    k = kPairSum ? c_yuv422.v[F::k10][color] : c_yuv.v[F::k10][color];
    sy = kPairSum ? k[9] : F::kShift;
    sc = kPairSum ? k[10] : F::kShift;
    yo = (c_yuv.v[F::k10][color][15] << sy) + (1 << (sy - 1));
    co = (F::kCoff << sc) + (1 << (sc - 1));
  }
  static __device__ __forceinline__ int q(int a, int s) { return min(max(a >> s, 0), F::kTop); }
  __device__ __forceinline__ int y(int R, int G, int B) const { return q(k[0] * R + k[1] * G + k[2] * B + yo, sy); }
  __device__ __forceinline__ int u(int R, int G, int B) const { return q(k[3] * R + k[4] * G + k[5] * B + co, sc); }
  __device__ __forceinline__ int v(int R, int G, int B) const { return q(k[6] * R + k[7] * G + k[8] * B + co, sc); }
};

// The RGB codes of a row's pixels [x0, x0 + npx) of the encode's source: the step's uint8 NHWC RGB (8-bit output),
// staged into sb with 16-byte loads (the caller synchronises before reading), or its fp32 NCHW HR frame (kF32,
// 10-bit output), read per pixel with coalesced row reads of the three planes, q = clip(rint(x * 1023), 0, 1023).
template <bool kF32>
struct RgbRow {
  const void* rgb;
  const uint8_t* sb;
  int H, W, img, y, x0, lead = 0;
  __device__ __forceinline__ RgbRow(const void* rgb_, const uint8_t* sb_, int H_, int W_, int img_, int y_, int x0_)
      : rgb(rgb_), sb(sb_), H(H_), W(W_), img(img_), y(y_), x0(x0_) {}
  // stages the uint8 row's npx pixels into sb (thread t of kThreads; the caller synchronises before reading)
  __device__ __forceinline__ RgbRow(const void* rgb_, uint8_t* sb_, int H_, int W_, int img_, int y_, int x0_, int npx,
                                    int t)
      : RgbRow(rgb_, sb_, H_, W_, img_, y_, x0_) {
    if constexpr (!kF32)
      lead = stage_bytes(sb_, static_cast<const uint8_t*>(rgb) + (((size_t)img * H + y) * W + x0) * 3, npx * 3, t);
  }
  // R, G, B of pixel x0 + j (recomputed per call: cheaper than keeping a row pointer live)
  __device__ __forceinline__ void operator()(int j, int& R, int& G, int& B) const {
    if constexpr (kF32) {
      const size_t plane = (size_t)H * W;
      const float* f = static_cast<const float*>(rgb) + (size_t)img * 3 * plane + (size_t)y * W + x0 + j;
      auto q10 = [](float x) { return (int)fminf(fmaxf(rintf(x * 1023.f), 0.f), 1023.f); };
      R = q10(__ldg(f)), G = q10(__ldg(f + plane)), B = q10(__ldg(f + 2 * plane));
    } else {
      const uint8_t* b = sb + lead + 3 * j;
      R = b[0], G = b[1], B = b[2];
    }
  }
};

// the store counterpart: dst[j] = sb[lead + j] for j < bytes with lead = dst % 16 (the caller placed the bytes
// there); 16-byte stores over the aligned interior, single bytes at the ends, nothing outside [dst, dst + bytes)
__device__ __forceinline__ void flush_bytes(uint8_t* __restrict__ dst, const uint8_t* sb, int bytes, int t) {
  const int lead = (int)((uintptr_t)dst & 15u);
  const int a0 = min(lead ? 16 - lead : 0, bytes);
  const int nv = (bytes - a0) / 16;
  const int tail0 = a0 + 16 * nv;
  for (int i = t; i < nv; i += kThreads)
    reinterpret_cast<uint4*>(dst + a0)[i] = *reinterpret_cast<const uint4*>(sb + lead + a0 + 16 * i);
  if (t < a0) dst[t] = sb[lead + t];
  if (tail0 + t < bytes) dst[tail0 + t] = sb[lead + tail0 + t];
}

// blockIdx.x < decode_ctas: decode CTA, row-major over x tiles (kHWC, 4:2:2, 4:4:4: one image row; 4:2:0: a pair
// of rows);
// the rest: zpc CTAs per slot, each zeroing a strided share of that slot's lr_prev and hr_prev when flagged.
template <int kFmt>
__global__ void __launch_bounds__(kThreads)
stream_frame_in_kernel(const uint8_t* __restrict__ in, const int32_t* __restrict__ reset,
                       float* __restrict__ lr_curr, float* __restrict__ lr_prev, float* __restrict__ hr_prev,
                       int c, int h, int w, tg_frame_window win, int s, int bgr, int x_tiles, int decode_ctas,
                       int zpc, int color) {
  // lr_curr, lr_prev and hr_prev belong to the previous step until it has finished
  tg_pdl_wait();
  tg_pdl_trigger();
  const int t = threadIdx.x;
  const int b = blockIdx.x;
  if (b < decode_ctas) {
    if constexpr (kFmt == kHWC)
      decode_hwc(in, lr_curr, b, t, c, h, w, win, bgr, x_tiles);
    else if constexpr (Yuv<kFmt>::k420)
      decode_yuv420<kFmt>(in, lr_curr, b, t, h, w, win, x_tiles, color);
    else
      decode_units<kFmt>(in, lr_curr, b, t, h, w, win, x_tiles, color);
    return;
  }
  const int rb = b - decode_ctas;
  const int slot = rb / zpc, part = rb - slot * zpc;
  if (__ldg(reset + slot) == 0) return;
  const size_t nlr = (size_t)c * h * w, nhr = nlr * s * s;
  const size_t worker = (size_t)part * kThreads + t, workers = (size_t)zpc * kThreads;
  zero_range(lr_prev + slot * nlr, nlr, worker, workers);
  zero_range(hr_prev + slot * nhr, nhr, worker, workers);
}


template <int kFmt>
int launch_frame_in(const char* name, const void* in, const int32_t* reset, float* lr_curr, float* lr_prev,
                    float* hr_prev, int n, int c, int h, int w, const tg_frame_window* win, int s, int bgr, int color,
                    cudaStream_t stream) {
  using F = Yuv<kFmt>;
  TG_REQUIRE(in || reset, TG_E_INVALID, "%s: in_u8 and reset are both NULL", name);
  TG_REQUIRE(lr_curr && lr_prev && hr_prev, TG_E_INVALID, "%s: null pointer (lr_curr / lr_prev / hr_prev)", name);
  TG_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0, TG_E_INVALID, "%s: bad size n=%d c=%d h=%d w=%d", name, n, c, h, w);
  TG_REQUIRE(c <= kMaxC, TG_E_UNSUPPORTED, "%s: %d channels (at most %d)", name, c, kMaxC);
  TG_REQUIRE(s == 2 || s == 4, TG_E_UNSUPPORTED, "%s: scale %d (2 or 4)", name, s);
  TG_REQUIRE((((uintptr_t)lr_curr | (uintptr_t)lr_prev | (uintptr_t)hr_prev) & 3u) == 0, TG_E_INVALID,
             "%s: fp32 buffers must be 4-byte aligned", name);
  const int rc = check_frames<kFmt>(name, in, h, w, win, F::kAlign);
  if (rc != TG_OK) return rc;
  const tg_frame_window whole = {h, w, 0, 0};
  if (!win) win = &whole;
  const int x_tiles = tg_ceil_div(tg_ceil_div(w, F::kUnitPx), kTilePx);
  const size_t decode = in ? (size_t)x_tiles * (h / F::kGy) * n : 0;
  const size_t hr4 = (size_t)c * s * h * s * w / 4;
  const int zpc = reset ? (int)(hr4 / (kThreads * 8) + 1 < 64 ? hr4 / (kThreads * 8) + 1 : 64) : 0;
  const size_t ctas = decode + (size_t)zpc * n;
  TG_REQUIRE(ctas <= 0x7fffffff, TG_E_UNSUPPORTED, "%s: grid too large", name);
  tg_launch(stream_frame_in_kernel<kFmt>, dim3((unsigned)ctas), dim3(kThreads), 0, stream,
            static_cast<const uint8_t*>(in), reset, lr_curr, lr_prev, hr_prev, c, h, w, *win, s, bgr, x_tiles,
            (int)decode, zpc, color);
  TG_CUDA_LAUNCH_CHECK(name);
  return TG_OK;
}

// one CTA: kTilePx pixels of the RGB rows 2*yp and 2*yp + 1 -> their Y words and the chroma words of the pair
// (U and V of a 2x2 block from its top-left pixel), staged in shared memory and written with 16-byte stores.
template <int kFmt>
__global__ void __launch_bounds__(kThreads)
rgb_to_yuv420_kernel(const void* __restrict__ rgb, uint8_t* __restrict__ out, int H, int W, tg_frame_window win,
                     int x_tiles, int color) {
  using F = Yuv<kFmt>;
  using Wd = typename F::Word;
  constexpr bool kF32 = F::k10;                              // 8-bit output reads uint8 RGB, 10-bit the fp32 frame
  constexpr int kB = (int)sizeof(Wd);
  __shared__ __align__(16) uint8_t sin[2][kF32 ? 16 : kTilePx * 3 + 16];
  __shared__ __align__(16) uint8_t sy[2][kTilePx * kB + 16];
  __shared__ __align__(16) uint8_t sc[2][kTilePx * kB + 16];   // NV12 layout: sc[0] = U V U V ...; I420: U, V
  // rgb is the previous kernel's output; out may still be read by the copy of an earlier step
  tg_pdl_wait();
  tg_pdl_trigger();
  const int t = threadIdx.x;
  const int xt = blockIdx.x % x_tiles, r = blockIdx.x / x_tiles;
  const int hp = H >> 1, yp = r % hp, img = r / hp;
  const int x0 = xt * kTilePx;
  const int npx = min(kTilePx, W - x0);                      // even
  const RgbRow<kF32> src0(rgb, sin[0], H, W, img, 2 * yp, x0, npx, t), src1(rgb, sin[1], H, W, img, 2 * yp + 1, x0,
                                                                          npx, t);
  const int fh = win.frame_h, fw = win.frame_w;              // even, as are top and left
  const int fx = win.left + x0, fy = win.top + 2 * yp;       // the tile's column and first row in the frame
  Wd* frame = reinterpret_cast<Wd*>(out) + (size_t)img * F::frame_words(3, fh, fw);
  Wd* yrow = frame + F::y_at(fw, fy, fx);
  Wd* c0 = frame + F::chroma_at(fw, fy, fx) + F::u_plane(fh, fw);
  Wd* c1 = frame + F::chroma_at(fw, fy, fx) + F::v_plane(fh, fw);   // I420 layout
  const int ly0 = lead_of(yrow), ly1 = lead_of(yrow + fw), lc0 = lead_of(c0), lc1 = F::kSemi ? 0 : lead_of(c1);
  auto put = [](uint8_t* sb, int lead, int j, int v) { reinterpret_cast<Wd*>(sb + lead)[j] = F::word(v); };
  if constexpr (!kF32) __syncthreads();
  if (t < npx) {
    const YuvEncode<kFmt> e(color);
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
      int R, G, B;
      if (dy) src1(t, R, G, B);
      else src0(t, R, G, B);
      put(sy[dy], dy ? ly1 : ly0, t, e.y(R, G, B));
      if (dy == 0 && (t & 1) == 0) {
        const int u = e.u(R, G, B), v = e.v(R, G, B);
        if (F::kSemi) {
          put(sc[0], lc0, t, u);
          put(sc[0], lc0, t + 1, v);
        } else {
          put(sc[0], lc0, t >> 1, u);
          put(sc[1], lc1, t >> 1, v);
        }
      }
    }
  }
  __syncthreads();
  auto flush = [&](Wd* dst, const uint8_t* sb, int words) {
    flush_bytes(reinterpret_cast<uint8_t*>(dst), sb, words * kB, t);
  };
  flush(yrow, sy[0], npx);
  flush(yrow + fw, sy[1], npx);
  if (F::kSemi) {
    flush(c0, sc[0], npx);
  } else {
    flush(c0, sc[0], npx >> 1);
    flush(c1, sc[1], npx >> 1);
  }
}

// q into the unit whose first pixel is (y, x) of frame img (fh x fw pixels): one 4-byte (packed 4:2:2) or 16-byte
// (v210) store of its group, or one word of each plane per sample
template <int kFmt>
__device__ __forceinline__ void store_unit(uint8_t* __restrict__ out, int fh, int fw, int img, int y, int x,
                                           const Unit<kFmt>& q) {
  using F = Yuv<kFmt>;
  if constexpr (kFmt == kV210) {
    *reinterpret_cast<uint4*>(out + F::group_at(fh, fw, img, y, x)) = make_uint4(q.w[0], q.w[1], q.w[2], q.w[3]);
  } else if constexpr (F::kGrouped) {
    *reinterpret_cast<uint32_t*>(out + F::group_at(fh, fw, img, y, x)) = q.w[0];
  } else {
    typename F::Word* f = reinterpret_cast<typename F::Word*>(out) + (size_t)img * F::frame_words(3, fh, fw);
#pragma unroll
    for (int j = 0; j < q.kPx; ++j) f[F::y_at(fw, y, x + j)] = F::word(q.y(j));
    typename F::Word* c = f + F::chroma_at(fw, y, x);
    c[F::u_plane(fh, fw)] = F::word(q.u(0));
    c[F::v_plane(fh, fw)] = F::word(q.v(0));
  }
}

// one CTA: kTilePx units of one row of the per-unit layouts (packed 4:2:2, 4:4:4, 10-bit 4:2:2), one per thread:
// Y of each pixel, U and V of each pixel (4:4:4) or of each pair's sum (4:2:2).  Units [0, units) of the picture are
// written; the fields past pixel W - 1 of a partial last v210 group are 0, and a whole-frame v210 encode (units = the
// row's S / 16 groups) also writes the row padding as 0.
template <int kFmt>
__global__ void __launch_bounds__(kThreads)
rgb_to_yuv_kernel(const void* __restrict__ rgb, uint8_t* __restrict__ out, int H, int W, tg_frame_window win,
                  int x_tiles, int units, int color) {
  using U = Unit<kFmt>;
  constexpr bool kF32 = Yuv<kFmt>::k10;                      // 8-bit output reads uint8 RGB, 10-bit the fp32 frame
  __shared__ __align__(16) uint8_t sin[kF32 ? 16 : kTilePx * U::kPx * 3 + 16];
  // rgb is the previous kernel's output; out may still be read by the copy of an earlier step
  tg_pdl_wait();
  tg_pdl_trigger();
  const int t = threadIdx.x;
  const int xt = blockIdx.x % x_tiles, r = blockIdx.x / x_tiles;
  const int y = r % H, img = r / H;
  const int tx0 = xt * kTilePx * U::kPx;                     // the tile's first pixel
  const RgbRow<kF32> src(rgb, sin, H, W, img, y, tx0, min(kTilePx * U::kPx, W - tx0), t);
  if constexpr (!kF32) __syncthreads();
  const int unit = xt * kTilePx + t;
  if (unit >= units) return;
  const YuvEncode<kFmt> e(color);
  U q;
#pragma unroll
  for (int p = 0; p < U::kC; ++p) {
    const int j = t * U::kPx + 2 * p;                        // the pair's (4:4:4: the pixel's) column in the tile
    if (tx0 + j >= W) break;                                 // W is even: a pair is whole or absent
    int R0, G0, B0;
    src(j, R0, G0, B0);
    if constexpr (U::kPx == 1) {
      q.set_y(0, e.y(R0, G0, B0));
      q.set_uv(0, e.u(R0, G0, B0), e.v(R0, G0, B0));
    } else {
      int R1, G1, B1;
      src(j + 1, R1, G1, B1);
      q.set_y(2 * p, e.y(R0, G0, B0));
      q.set_y(2 * p + 1, e.y(R1, G1, B1));
      q.set_uv(p, e.u(R0 + R1, G0 + G1, B0 + B1), e.v(R0 + R1, G0 + G1, B0 + B1));
    }
  }
  store_unit<kFmt>(out, win.frame_h, win.frame_w, img, win.top + y, win.left + unit * U::kPx, q);
}

template <int kFmt>
int launch_to_yuv(const char* name, const void* rgb, void* out, int n, int H, int W, const tg_frame_window* win,
                  int color, cudaStream_t stream) {
  using F = Yuv<kFmt>;
  TG_REQUIRE(n > 0 && H > 0 && W > 0, TG_E_INVALID, "%s: bad size n=%d H=%d W=%d", name, n, H, W);
  const int rc = check_frames<kFmt>(name, out, H, W, win, F::kAlign, "output");
  if (rc != TG_OK) return rc;
  const bool whole_frame = win == nullptr;
  const tg_frame_window whole = {H, W, 0, 0};
  if (!win) win = &whole;
  // the picture's units, or every v210 group of the row up to its stride for a whole-frame encode
  const int units = kFmt == kV210 && whole_frame ? (int)(v210_stride(W) / 16) : tg_ceil_div(W, F::kUnitPx);
  const int x_tiles = tg_ceil_div(units, kTilePx);
  const size_t ctas = (size_t)x_tiles * (H / F::kGy) * n;
  TG_REQUIRE(ctas <= 0x7fffffff, TG_E_UNSUPPORTED, "%s: grid too large", name);
  uint8_t* o = static_cast<uint8_t*>(out);
  if constexpr (F::k420)
    tg_launch(rgb_to_yuv420_kernel<kFmt>, dim3((unsigned)ctas), dim3(kThreads), 0, stream, rgb, o, H, W, *win,
              x_tiles, color);
  else
    tg_launch(rgb_to_yuv_kernel<kFmt>, dim3((unsigned)ctas), dim3(kThreads), 0, stream, rgb, o, H, W, *win, x_tiles,
              units, color);
  TG_CUDA_LAUNCH_CHECK(name);
  return TG_OK;
}

// total words of n frames := the layout's black (Y: the colour's luma offset, U = V: kCoff; HWC: 0).  Grid-stride;
// runs once per stream, when the padded output frames are allocated.  v210 (frame_w fw): the fields of each row's
// ceil(fw / 6) groups that hold a pixel, 0 in the rest of a partial last group and in the row padding.
template <int kFmt>
__global__ void __launch_bounds__(kThreads)
fill_black_kernel(uint8_t* __restrict__ out, size_t frame, size_t luma, size_t total, int color, int fw) {
  using F = Yuv<kFmt>;
  using Wd = typename F::Word;
  tg_pdl_wait();
  tg_pdl_trigger();
  Wd* o = reinterpret_cast<Wd*>(out);
  const int y = kFmt == kHWC ? 0 : c_yuv.v[F::k10][color][15];
  if constexpr (kFmt == kV210) {
    const size_t row_words = v210_stride(fw) / 4;
    uint32_t* o32 = reinterpret_cast<uint32_t*>(out);
    for (size_t i = blockIdx.x * (size_t)kThreads + threadIdx.x; i < total / 4; i += (size_t)gridDim.x * kThreads) {
      const int wi = (int)(i % row_words), x0 = 6 * (wi >> 2);
      uint32_t word = 0;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const int f = 3 * (wi & 3) + k;              // Y of pixel (f - 1) / 2 when f is odd, else chroma of pair f / 4
        const int x = x0 + ((f & 1) ? (f - 1) / 2 : 2 * (f / 4));
        if (x < fw) word |= (uint32_t)((f & 1) ? y : F::kCoff) << (10 * k);
      }
      o32[i] = word;
    }
  } else {
    for (size_t i = blockIdx.x * (size_t)kThreads + threadIdx.x; i < total; i += (size_t)gridDim.x * kThreads) {
      const size_t j = i % frame;
      // packed 4:2:2: Y is every other byte, starting at Y0's; planar: the first fh * fw words
      const bool is_y = F::kGrouped ? (int)(j & 1) == F::y_field(0) : j < luma;
      o[i] = kFmt == kHWC ? (Wd)0 : F::word(is_y ? y : F::kCoff);
    }
  }
}

template <int kFmt>
int launch_fill_black(const char* name, void* out, int n, int c, int fh, int fw, int color, cudaStream_t stream) {
  using F = Yuv<kFmt>;
  TG_REQUIRE(out, TG_E_INVALID, "%s: null pointer (out)", name);
  TG_REQUIRE(n > 0 && c > 0 && fh > 0 && fw > 0, TG_E_INVALID, "%s: bad size n=%d c=%d %dx%d", name, n, c, fh, fw);
  TG_REQUIRE(kFmt == kHWC || c == 3, TG_E_INVALID, "%s: YUV frames carry 3 channels, got %d", name, c);
  // words, one at a time; v210 frames are whole groups
  const int rc =
      check_frames<kFmt>(name, out, fh, fw, nullptr, kFmt == kV210 ? F::kAlign : (int)sizeof(typename F::Word));
  if (rc != TG_OK) return rc;
  const size_t frame = F::frame_words(c, fh, fw), total = frame * n;
  const size_t need = (total + kThreads - 1) / kThreads, ctas = need < 4096 ? need : 4096;
  tg_launch(fill_black_kernel<kFmt>, dim3((unsigned)ctas), dim3(kThreads), 0, stream, static_cast<uint8_t*>(out),
            frame, (size_t)fh * fw, total, color, fw);
  TG_CUDA_LAUNCH_CHECK(name);
  return TG_OK;
}

// One CTA: kTilePx pixels of one row of one frame -> their 8-bit luma (Y, 10-bit >> 2; RGB: cv2's gray) added to
// cols[img][x] and, summed over the CTA, to rows[img][y].  Integer sums: the order does not matter.
template <int kFmt>
__global__ void __launch_bounds__(kThreads)
luma_sums_kernel(const uint8_t* __restrict__ in, int c, int h, int w, int bgr, int x_tiles,
                 unsigned long long* __restrict__ rows, unsigned long long* __restrict__ cols) {
  using F = Yuv<kFmt>;
  __shared__ unsigned warp_sum[kThreads / 32];
  tg_pdl_wait();
  tg_pdl_trigger();
  const int t = threadIdx.x;
  const int xt = blockIdx.x % x_tiles, r = blockIdx.x / x_tiles;
  const int y = r % h, img = r / h;
  const int x = xt * kTilePx + t;
  unsigned v = 0;
  if (x < w) {
    if constexpr (kFmt == kHWC) {
      const uint8_t* p = in + (((size_t)img * h + y) * w + x) * c;
      const unsigned R = __ldg(p + (bgr ? 2 : 0)), G = __ldg(p + 1), B = __ldg(p + (bgr ? 0 : 2));
      v = (9798u * R + 19235u * G + 3735u * B + 16384u) >> 15;
    } else if constexpr (kFmt == kV210) {
      const uint32_t* g = reinterpret_cast<const uint32_t*>(in + F::group_at(h, w, img, y, x));
      const int f = F::y_field(x % 6);
      v = (unsigned)F::field(__ldg(g + f / F::kFieldsPerWord), f) >> 2;
    } else if constexpr (F::kGrouped) {
      v = __ldg(in + F::group_at(h, w, img, y, x) + F::y_field(x & 1));   // a packed field is a byte of the group
    } else {
      const typename F::Word* frame = reinterpret_cast<const typename F::Word*>(in) + img * F::frame_words(3, h, w);
      v = (unsigned)F::sample(__ldg(frame + F::y_at(w, y, x))) >> (F::k10 ? 2 : 0);
    }
    atomicAdd(cols + (size_t)img * w + x, (unsigned long long)v);
  }
  v = __reduce_add_sync(0xffffffffu, v);       // at most 32 * 255
  if ((t & 31) == 0) warp_sum[t >> 5] = v;
  __syncthreads();
  if (t == 0) {
    unsigned long long sum = 0;
    for (int i = 0; i < kThreads / 32; ++i) sum += warp_sum[i];
    atomicAdd(rows + (size_t)img * h + y, sum);
  }
}

template <int kFmt>
int launch_luma_sums(const char* name, const void* in, int bgr, int n, int c, int h, int w, unsigned long long* rows,
                     unsigned long long* cols, cudaStream_t stream) {
  TG_REQUIRE(in && rows && cols, TG_E_INVALID, "%s: null pointer (in / rows / cols)", name);
  TG_REQUIRE(n > 0 && h > 0 && w > 0, TG_E_INVALID, "%s: bad size n=%d %dx%d", name, n, h, w);
  TG_REQUIRE(c == 3, TG_E_INVALID, "%s: luma of 3-channel frames, got %d channels", name, c);
  TG_REQUIRE((((uintptr_t)rows | (uintptr_t)cols) & 7u) == 0, TG_E_INVALID, "%s: rows and cols 8-byte aligned", name);
  // Y alone: a byte of a packed group, a 4-byte word of a v210 group, a planar word
  const int rc = check_frames<kFmt>(name, in, h, w, nullptr, kFmt == kV210 ? 4 : (int)sizeof(typename Yuv<kFmt>::Word));
  if (rc != TG_OK) return rc;
  const int x_tiles = tg_ceil_div(w, kTilePx);
  const size_t ctas = (size_t)x_tiles * h * n;
  TG_REQUIRE(ctas <= 0x7fffffff, TG_E_UNSUPPORTED, "%s: grid too large", name);
  cudaError_t e = cudaMemsetAsync(rows, 0, (size_t)n * h * sizeof(unsigned long long), stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(cols, 0, (size_t)n * w * sizeof(unsigned long long), stream);
  TG_REQUIRE(e == cudaSuccess, (int)e, "%s: cudaMemsetAsync: %s", name, cudaGetErrorString(e));
  tg_launch(luma_sums_kernel<kFmt>, dim3((unsigned)ctas), dim3(kThreads), 0, stream, static_cast<const uint8_t*>(in),
            c, h, w, bgr, x_tiles, rows, cols);
  TG_CUDA_LAUNCH_CHECK(name);
  return TG_OK;
}


}  // namespace

namespace {

int frame_in_yuv(const char* name, const void* in, const tg_yuv_format* fmt, const tg_frame_window* win,
                 const int32_t* reset, float* lr_curr, float* lr_prev, float* hr_prev, int n, int h, int w, int s,
                 cudaStream_t st) {
  int f = 0, color = 0;
  const int rc = parse_yuv_format(name, fmt, &f, &color);
  if (rc != TG_OK) return rc;
  return dispatch_format(f, [&](auto k) {
    constexpr int K = decltype(k)::value;
    if constexpr (K == kHWC) return (int)TG_E_UNSUPPORTED;
    else return launch_frame_in<K>(name, in, reset, lr_curr, lr_prev, hr_prev, n, 3, h, w, win, s, 0, color, st);
  });
}

int rgb_to_yuv(const char* name, const uint8_t* rgb_u8, const float* rgb_f32, void* out, const tg_yuv_format* fmt,
               const tg_frame_window* win, int n, int H, int W, cudaStream_t st) {
  int f = 0, color = 0;
  const int rc = parse_yuv_format(name, fmt, &f, &color);
  if (rc != TG_OK) return rc;
  const bool ten = fmt_10(f);
  TG_REQUIRE(out, TG_E_INVALID, "%s: null pointer (out)", name);
  TG_REQUIRE(ten ? (rgb_f32 && !rgb_u8) : (rgb_u8 && !rgb_f32), TG_E_INVALID,
             "%s: %s output is encoded from %s (and only that source)", name, ten ? "10-bit" : "8-bit",
             ten ? "rgb_f32" : "rgb_u8");
  TG_REQUIRE(!ten || ((((uintptr_t)rgb_f32) & 3u) == 0 && (((uintptr_t)out) & 1u) == 0), TG_E_INVALID,
             "%s: rgb_f32 must be 4-byte and 10-bit output 2-byte aligned", name);
  const void* rgb = ten ? static_cast<const void*>(rgb_f32) : static_cast<const void*>(rgb_u8);
  return dispatch_format(f, [&](auto k) {
    constexpr int K = decltype(k)::value;
    if constexpr (K == kHWC) return (int)TG_E_UNSUPPORTED;
    else return launch_to_yuv<K>(name, rgb, out, n, H, W, win, color, st);
  });
}

// copy floats [0, count) of src to dst (4-byte aligned, not overlapping): 16-byte vectors over the interior when
// both share their alignment mod 16, else one float at a time.  `worker` of `workers` threads.
__device__ __forceinline__ void copy_range(float* __restrict__ dst, const float* __restrict__ src, size_t count,
                                           size_t worker, size_t workers) {
  if ((((uintptr_t)dst ^ (uintptr_t)src) & 15u) != 0) {
    for (size_t i = worker; i < count; i += workers) dst[i] = __ldg(src + i);
    return;
  }
  size_t head = ((16u - ((uintptr_t)dst & 15u)) & 15u) / 4u;
  if (head > count) head = count;
  const size_t n4 = (count - head) / 4;
  const size_t tail0 = head + n4 * 4;
  const float4* s4 = reinterpret_cast<const float4*>(src + head);
  float4* d4 = reinterpret_cast<float4*>(dst + head);
  for (size_t i = worker; i < n4; i += workers) d4[i] = __ldg(s4 + i);
  if (worker < head) dst[worker] = __ldg(src + worker);
  if (worker < count - tail0) dst[tail0 + worker] = __ldg(src + tail0 + worker);
}

// blockIdx.x < n * cpc: cpc CTAs per slot copy a strided share of its current frame out of the ring; the rest: zpc
// CTAs per slot apply its state mode (a keep-slot's CTAs read mode[k] and return)
__global__ void __launch_bounds__(kThreads)
stream_gather_kernel(const float* __restrict__ ring, int depth, const int32_t* __restrict__ table,
                     const float* __restrict__ warm_hr, float* __restrict__ lr_curr, float* __restrict__ lr_prev,
                     float* __restrict__ hr_prev, int n, size_t nlr, size_t nhr, int cpc, int zpc) {
  // the table is written, and lr_curr / lr_prev / hr_prev read, by work ordered before this launch
  tg_pdl_wait();
  tg_pdl_trigger();
  const int t = threadIdx.x, b = blockIdx.x;
  const size_t frame = (size_t)n * nlr;          // one ring position
  if (b < n * cpc) {
    const int slot = b / cpc, part = b - slot * cpc;
    const int cur = __ldg(table + slot);
    if (cur < 0 || cur >= depth) return;
    copy_range(lr_curr + slot * nlr, ring + cur * frame + slot * nlr, nlr, (size_t)part * kThreads + t,
               (size_t)cpc * kThreads);
    return;
  }
  const int rb = b - n * cpc;
  const int slot = rb / zpc, part = rb - slot * zpc;
  const int mode = __ldg(table + n + slot);
  if (mode != TG_GATHER_ZERO && (mode != TG_GATHER_LOAD || warm_hr == nullptr)) return;
  const size_t worker = (size_t)part * kThreads + t, workers = (size_t)zpc * kThreads;
  const int prev = mode == TG_GATHER_LOAD ? __ldg(table + 2 * n + slot) : -1;
  if (prev < 0 || prev >= depth)
    zero_range(lr_prev + slot * nlr, nlr, worker, workers);
  else
    copy_range(lr_prev + slot * nlr, ring + prev * frame + slot * nlr, nlr, worker, workers);
  if (mode == TG_GATHER_ZERO)
    zero_range(hr_prev + slot * nhr, nhr, worker, workers);
  else
    copy_range(hr_prev + slot * nhr, warm_hr + slot * nhr, nhr, worker, workers);
}

// CTAs per slot for `count` floats: one per 8 float4 vectors of each thread, at most 64
inline int ctas_per_slot(size_t count) {
  const size_t v = count / 4 / (kThreads * 8) + 1;
  return (int)(v < 64 ? v : 64);
}

}  // namespace

extern "C" int tg_stream_gather(const float* ring, int depth, const int32_t* table, const float* warm_hr,
                                float* lr_curr, float* lr_prev, float* hr_prev, int n, int c, int h, int w, int s,
                                void* stream) {
  const char* name = "stream_gather";
  TG_REQUIRE(ring && table && lr_curr && lr_prev && hr_prev, TG_E_INVALID,
             "%s: null pointer (ring / table / lr_curr / lr_prev / hr_prev)", name);
  TG_REQUIRE(depth > 0 && n > 0 && c > 0 && h > 0 && w > 0, TG_E_INVALID, "%s: bad size depth=%d n=%d c=%d h=%d w=%d",
             name, depth, n, c, h, w);
  TG_REQUIRE(s == 2 || s == 4, TG_E_UNSUPPORTED, "%s: scale %d (2 or 4)", name, s);
  TG_REQUIRE((((uintptr_t)ring | (uintptr_t)table | (uintptr_t)warm_hr | (uintptr_t)lr_curr | (uintptr_t)lr_prev |
               (uintptr_t)hr_prev) & 3u) == 0,
             TG_E_INVALID, "%s: buffers must be 4-byte aligned", name);
  const size_t nlr = (size_t)c * h * w, nhr = nlr * s * s;
  const int cpc = ctas_per_slot(nlr), zpc = ctas_per_slot(nhr);
  const size_t ctas = (size_t)(cpc + zpc) * n;
  TG_REQUIRE(ctas <= 0x7fffffff, TG_E_UNSUPPORTED, "%s: grid too large", name);
  tg_launch(stream_gather_kernel, dim3((unsigned)ctas), dim3(kThreads), 0, (cudaStream_t)stream, ring, depth, table,
            warm_hr, lr_curr, lr_prev, hr_prev, n, nlr, nhr, cpc, zpc);
  TG_CUDA_LAUNCH_CHECK(name);
  return TG_OK;
}

extern "C" int tg_stream_frame_in(const uint8_t* in_u8, const int32_t* reset, float* lr_curr, float* lr_prev,
                                  float* hr_prev, int n, int c, int h, int w, int s, int bgr, void* stream) {
  return launch_frame_in<kHWC>("stream_frame_in", in_u8, reset, lr_curr, lr_prev, hr_prev, n, c, h, w, nullptr, s,
                               bgr, 0, (cudaStream_t)stream);
}

extern "C" int tg_stream_frame_in_window(const uint8_t* in_u8, const tg_frame_window* win, const int32_t* reset,
                                         float* lr_curr, float* lr_prev, float* hr_prev, int n, int c, int h, int w,
                                         int s, int bgr, void* stream) {
  TG_REQUIRE(win, TG_E_INVALID, "stream_frame_in_window: null window");
  return launch_frame_in<kHWC>("stream_frame_in_window", in_u8, reset, lr_curr, lr_prev, hr_prev, n, c, h, w, win, s,
                               bgr, 0, (cudaStream_t)stream);
}

extern "C" int tg_stream_frame_in_yuv420(const uint8_t* in, int nv12, const int32_t* reset, float* lr_curr,
                                         float* lr_prev, float* hr_prev, int n, int h, int w, int s, void* stream) {
  return nv12 ? launch_frame_in<kNV12>("stream_frame_in_yuv420", in, reset, lr_curr, lr_prev, hr_prev, n, 3, h, w,
                                       nullptr, s, 0, 0, (cudaStream_t)stream)
              : launch_frame_in<kI420>("stream_frame_in_yuv420", in, reset, lr_curr, lr_prev, hr_prev, n, 3, h, w,
                                       nullptr, s, 0, 0, (cudaStream_t)stream);
}

extern "C" int tg_rgb_u8_to_yuv420(const uint8_t* rgb, uint8_t* out, int nv12, int n, int H, int W, void* stream) {
  TG_REQUIRE(rgb && out, TG_E_INVALID, "rgb_u8_to_yuv420: null pointer (rgb / out)");
  return nv12 ? launch_to_yuv<kNV12>("rgb_u8_to_yuv420", rgb, out, n, H, W, nullptr, 0, (cudaStream_t)stream)
              : launch_to_yuv<kI420>("rgb_u8_to_yuv420", rgb, out, n, H, W, nullptr, 0, (cudaStream_t)stream);
}

extern "C" int tg_stream_frame_in_yuv(const void* in, const tg_yuv_format* fmt, const int32_t* reset, float* lr_curr,
                                      float* lr_prev, float* hr_prev, int n, int h, int w, int s, void* stream) {
  return frame_in_yuv("stream_frame_in_yuv", in, fmt, nullptr, reset, lr_curr, lr_prev, hr_prev, n, h, w, s,
                      (cudaStream_t)stream);
}

extern "C" int tg_stream_frame_in_yuv_window(const void* in, const tg_yuv_format* fmt, const tg_frame_window* win,
                                             const int32_t* reset, float* lr_curr, float* lr_prev, float* hr_prev,
                                             int n, int h, int w, int s, void* stream) {
  TG_REQUIRE(win, TG_E_INVALID, "stream_frame_in_yuv_window: null window");
  return frame_in_yuv("stream_frame_in_yuv_window", in, fmt, win, reset, lr_curr, lr_prev, hr_prev, n, h, w, s,
                      (cudaStream_t)stream);
}

extern "C" int tg_rgb_to_yuv(const uint8_t* rgb_u8, const float* rgb_f32, void* out, const tg_yuv_format* fmt, int n,
                             int H, int W, void* stream) {
  return rgb_to_yuv("rgb_to_yuv", rgb_u8, rgb_f32, out, fmt, nullptr, n, H, W, (cudaStream_t)stream);
}

extern "C" int tg_rgb_to_yuv_window(const uint8_t* rgb_u8, const float* rgb_f32, void* out, const tg_yuv_format* fmt,
                                    const tg_frame_window* win, int n, int H, int W, void* stream) {
  TG_REQUIRE(win, TG_E_INVALID, "rgb_to_yuv_window: null window");
  return rgb_to_yuv("rgb_to_yuv_window", rgb_u8, rgb_f32, out, fmt, win, n, H, W, (cudaStream_t)stream);
}

extern "C" int tg_fill_black(void* out, const tg_yuv_format* fmt, int n, int c, int frame_h, int frame_w,
                             void* stream) {
  const char* name = "fill_black";
  int f = kHWC, color = 0;
  if (fmt) {
    const int rc = parse_yuv_format(name, fmt, &f, &color);
    if (rc != TG_OK) return rc;
  }
  return dispatch_format(f, [&](auto k) {
    return launch_fill_black<decltype(k)::value>(name, out, n, c, frame_h, frame_w, color, (cudaStream_t)stream);
  });
}

extern "C" int tg_luma_line_sums(const void* in, const tg_yuv_format* fmt, int bgr, int n, int c, int h, int w,
                                 unsigned long long* rows, unsigned long long* cols, void* stream) {
  const char* name = "luma_line_sums";
  int f = kHWC, color = 0;
  if (fmt) {
    const int rc = parse_yuv_format(name, fmt, &f, &color);
    if (rc != TG_OK) return rc;
  }
  return dispatch_format(f, [&](auto k) {
    return launch_luma_sums<decltype(k)::value>(name, in, bgr, n, c, h, w, rows, cols, (cudaStream_t)stream);
  });
}

extern "C" int tg_yuv_coefficients(const tg_yuv_format* fmt, int32_t* out16) {
  int f = 0, color = 0;
  const int rc = parse_yuv_format("yuv_coefficients", fmt, &f, &color);
  if (rc != TG_OK) return rc;
  TG_REQUIRE(out16, TG_E_INVALID, "yuv_coefficients: null pointer (out16)");
  const int* r = kYuvTable.v[fmt_10(f) ? 1 : 0][color];
  for (int k = 0; k < 16; ++k) out16[k] = r[k];
  return TG_OK;
}
