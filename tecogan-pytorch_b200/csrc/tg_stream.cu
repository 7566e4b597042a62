// Frame I/O of one streamed inference step: uint8 HWC or YUV (4:2:0: NV12 / I420, 8 bit; P010 / I420_10, 10 bit;
// packed 4:2:2: YUY2 / UYVY, 8 bit; planar 4:4:4: I444, 8 bit, I444_10) frames decoded on the device into the
// step's fp32 NCHW lr_curr, the per-slot reset of the recurrent state, and the encode of the step's RGB output
// (uint8 NHWC, or the fp32 NCHW HR frame for 10-bit output) into any of those YUV layouts.
// Contract: include/tecogan_b200.h (tg_stream_frame_in, tg_stream_frame_in_yuv420, tg_rgb_u8_to_yuv420,
// tg_stream_frame_in_yuv, tg_rgb_to_yuv, tg_yuv_coefficients).
#include <type_traits>

#include "tg_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kTilePx = 256;            // decode / encode CTA: kTilePx pixels of a row, one per thread
constexpr int kMaxC = 4;

enum FrameFormat { kHWC = 0, kNV12 = 1, kI420 = 2, kP010 = 3, kI420_10 = 4, kYUY2 = 5, kUYVY = 6, kI444 = 7,
                   kI444_10 = 8 };

constexpr bool fmt_10(int f) { return f == kP010 || f == kI420_10 || f == kI444_10; }
constexpr bool fmt_packed(int f) { return f == kYUY2 || f == kUYVY; }     // 4:2:2, one 4-byte group per pair
constexpr bool fmt_444(int f) { return f == kI444 || f == kI444_10; }     // three full-size planes
constexpr bool fmt_420(int f) { return f != kHWC && !fmt_packed(f) && !fmt_444(f); }
// byte of Y0 (Y1 two bytes later) and of U (V two bytes later) in a packed group: YUY2 is Y0 U Y1 V, UYVY U Y0 V Y1
constexpr int packed_y0(int f) { return f == kUYVY ? 1 : 0; }
constexpr int packed_u(int f) { return f == kUYVY ? 0 : 1; }

template <int kFmt>
struct Yuv {
  static constexpr bool kInterleaved = kFmt == kNV12 || kFmt == kP010;     // NV12 plane layout
  static constexpr bool k10 = fmt_10(kFmt);
  using Word = typename std::conditional<k10, uint16_t, uint8_t>::type;
  static constexpr int kShift = k10 ? 18 : 20;                              // fraction bits of the table row
  static constexpr int kTop = k10 ? 1023 : 255;
  static constexpr int kCoff = k10 ? 512 : 128;
  // the sample of a stored word: P010 keeps it in the high 10 bits, I420_10 / I444_10 in the low 10 (larger
  // words clamp)
  static __device__ __forceinline__ int sample(Word v) {
    return kFmt == kP010 ? (int)(v >> 6) : (kFmt == kI420_10 || kFmt == kI444_10) ? min((int)v, 1023) : (int)v;
  }
  static __device__ __forceinline__ Word word(int v) { return (Word)(kFmt == kP010 ? v << 6 : v); }
};

// The colour table (oracle/yuv_color.py derives the same numbers): [depth 8 / 10][colour][16] with colour
// 0 bt601, 1 bt709, 2 bt601-full, 3 bt709-full and the row
//   cRY cGY cBY cRU cGU cBU cRV cGV cBV   encode, per RGB code value
//   CY CUB CUG CVG CVR                    decode
//   shift yoff                            fraction bits (20 at 8 bits, 18 at 10), luma offset (0: full range)
// Rows are (Kr, Kb) quantised as ITU-T H.273 does for the bit depth, rounded half away from zero.  The 8-bit
// bt601 row is cv2's BT.601 limited-range constants (color_yuv), so the NV12 / I420 bytes stay cv2's; its
// decode also keeps cv2's max(Y - 16, 0) before the multiply, the derived rows clamp only the RGB result.
// Every fixed-point intermediate fits in int32: |sum| < 6e8.
struct YuvTable {
  int v[2][4][16];
};

constexpr int yuv_round(double x) { return x >= 0 ? (int)(x + 0.5) : -(int)(-x + 0.5); }

constexpr YuvTable make_yuv_table() {
  YuvTable t{};
  const int cv2[16] = {269484, 528482, 102760, -155188, -305135, 460324, 460324, -385875, -74448,
                       1220542, 2116026, -409993, -852492, 1673527, 20, 16};
  for (int di = 0; di < 2; ++di) {
    const int depth = di ? 10 : 8, shift = di ? 18 : 20;
    for (int ci = 0; ci < 4; ++ci) {
      int* r = t.v[di][ci];
      if (di == 0 && ci == 0) {
        for (int k = 0; k < 16; ++k) r[k] = cv2[k];
        continue;
      }
      const bool full = ci >= 2;
      const double kr = (ci & 1) ? 0.2126 : 0.299, kb = (ci & 1) ? 0.0722 : 0.114;
      const double kg = 1.0 - kr - kb;
      const double d = (double)((1 << depth) - 1), sc = (double)(1 << (depth - 8));
      const double ky = full ? d : 219.0 * sc, kc = full ? d : 224.0 * sc;
      const double one = (double)(1 << shift);
      const double m[14] = {kr * ky / d, kg * ky / d, kb * ky / d,
                            -kr / (2.0 * (1.0 - kb)) * kc / d, -kg / (2.0 * (1.0 - kb)) * kc / d, 0.5 * kc / d,
                            0.5 * kc / d, -kg / (2.0 * (1.0 - kr)) * kc / d, -kb / (2.0 * (1.0 - kr)) * kc / d,
                            d / ky, d * 2.0 * (1.0 - kb) / kc, -d * 2.0 * (1.0 - kb) * kb / (kg * kc),
                            -d * 2.0 * (1.0 - kr) * kr / (kg * kc), d * 2.0 * (1.0 - kr) / kc};
      for (int k = 0; k < 14; ++k) r[k] = yuv_round(m[k] * one);
      r[14] = shift;
      r[15] = full ? 0 : 16 << (depth - 8);
    }
  }
  return t;
}

constexpr YuvTable kYuvTable = make_yuv_table();
__constant__ YuvTable c_yuv = make_yuv_table();
static_assert(kYuvTable.v[0][0][14] == Yuv<kNV12>::kShift && kYuvTable.v[1][3][14] == Yuv<kP010>::kShift,
              "table shift and kernel shift disagree");
static_assert(kYuvTable.v[0][0][14] == Yuv<kYUY2>::kShift && kYuvTable.v[0][3][14] == Yuv<kUYVY>::kShift &&
                  kYuvTable.v[0][1][14] == Yuv<kI444>::kShift && kYuvTable.v[1][2][14] == Yuv<kI444_10>::kShift,
              "table shift and kernel shift of the 4:2:2 / 4:4:4 layouts disagree");
static_assert(Yuv<kYUY2>::kTop == 255 && Yuv<kUYVY>::kCoff == 128 && Yuv<kI444>::kTop == 255 &&
                  Yuv<kI444_10>::kTop == 1023 && Yuv<kI444_10>::kCoff == 512 && Yuv<kI444_10>::k10,
              "4:2:2 is 8 bit only, I444_10 is the 10-bit table row");
static_assert(!Yuv<kYUY2>::kInterleaved && !Yuv<kUYVY>::kInterleaved && !Yuv<kI444>::kInterleaved &&
                  !Yuv<kI444_10>::kInterleaved, "4:2:2 and 4:4:4 frames have no NV12 chroma plane");

// Encode rows of 4:2:2 (8 bit): Y per pixel, U and V from the sum of the pair's two pixels,
//   Y = clip((kY . rgb + 2^(sy-1) + (yoff << sy)) >> sy)
//   C = clip((kC . (rgb0 + rgb1) + 2^(sc-1) + (128 << sc)) >> sc)
// i.e. the chroma of the pair's mean, rounded half up.  [colour][kRY kGY kBY kRU kGU kBU kRV kGV kBV sy sc].  The
// bt601 row is cv2's COLOR_RGB2YUV_YUY2 / _UYVY (14-bit constants of its own, luma included, with the chroma
// constants halved for the sum); the derived rows are the table's encode rows with sy = 20 and sc = 21.
// oracle/yuv_422_444.py specifies the same rule.
struct Yuv422Enc {
  int v[4][11];
};

constexpr Yuv422Enc make_yuv422_enc() {
  Yuv422Enc e{};
  const int cv2[11] = {4211, 8258, 1606, -1212, -2384, 3596, 3596, -3015, -582, 14, 14};
  for (int k = 0; k < 11; ++k) e.v[0][k] = cv2[k];
  for (int ci = 1; ci < 4; ++ci) {
    for (int k = 0; k < 9; ++k) e.v[ci][k] = kYuvTable.v[0][ci][k];
    e.v[ci][9] = kYuvTable.v[0][ci][14];
    e.v[ci][10] = kYuvTable.v[0][ci][14] + 1;
  }
  return e;
}

__constant__ Yuv422Enc c_yuv422 = make_yuv422_enc();

// zero floats [0, count) of p (4-byte aligned): 16-byte stores over the aligned interior, at most three
// scalar stores at each end.  `worker` of `workers` threads; writes nothing outside the range.
__device__ __forceinline__ void zero_range(float* p, size_t count, size_t worker, size_t workers) {
  size_t head = ((16u - ((uintptr_t)p & 15u)) & 15u) / 4u;
  if (head > count) head = count;
  const size_t n4 = (count - head) / 4;
  const size_t tail0 = head + n4 * 4;
  float4* v = reinterpret_cast<float4*>(p + head);
  for (size_t i = worker; i < n4; i += workers) v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (worker < head) p[worker] = 0.f;
  if (worker < count - tail0) p[tail0 + worker] = 0.f;
}

// sb[lead + j] = src[j] for j < bytes, lead = src % 16: the 16-byte-aligned interior of the source lands on
// 16-byte-aligned shared memory and is read with 16-byte loads, the ragged ends byte by byte.  Thread t of
// kThreads; returns lead.  sb must hold lead + bytes <= bytes + 15.
__device__ __forceinline__ int stage_bytes(uint8_t* sb, const uint8_t* __restrict__ src, int bytes, int t) {
  const int lead = (int)((uintptr_t)src & 15u);
  const int a0 = min(lead ? 16 - lead : 0, bytes);     // bytes before the first aligned 16-byte vector
  const int nv = (bytes - a0) / 16;
  const int tail0 = a0 + 16 * nv;
  for (int i = t; i < nv; i += kThreads)
    *reinterpret_cast<uint4*>(sb + lead + a0 + 16 * i) = __ldg(reinterpret_cast<const uint4*>(src + a0) + i);
  if (t < a0) sb[lead + t] = __ldg(src + t);
  if (tail0 + t < bytes) sb[lead + tail0 + t] = __ldg(src + tail0 + t);
  return lead;
}

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

__device__ __forceinline__ int lead_of(const void* p) { return (int)((uintptr_t)p & 15u); }

// decode CTA of HWC frames: kTilePx pixels of one image row
__device__ __forceinline__ void decode_hwc(const uint8_t* __restrict__ in, float* __restrict__ lr_curr, int b, int t,
                                           int c, int h, int w, int bgr, int x_tiles) {
  __shared__ __align__(16) uint8_t sb[kTilePx * kMaxC + 32];
  const int xt = b % x_tiles, r = b / x_tiles;
  const int y = r % h, img = r / h;
  const int x0 = xt * kTilePx;
  const int npx = min(kTilePx, w - x0);
  const int lead = stage_bytes(sb, in + (((size_t)img * h + y) * w + x0) * c, npx * c, t);
  __syncthreads();
  if (t < npx) {
    float* dst = lr_curr + ((size_t)img * c * h + y) * w + x0 + t;
    const size_t plane = (size_t)h * w;
    for (int k = 0; k < c; ++k) {
      const int ks = bgr ? c - 1 - k : k;
      // IEEE division, == numpy float32(v) / 255.0 (paired_folder_dataset.py:49); v * (1/255) differs
      dst[k * plane] = __fdiv_rn((float)sb[lead + t * c + ks], 255.f);
    }
  }
}

// decode CTA of YUV 4:2:0 frames ([3h/2, w] words each): kTilePx pixels of the luma rows 2*yp and 2*yp + 1 and
// the chroma samples they share (nearest chroma), written as RGB / 255 (8 bit) or RGB / 1023 (10 bit).  Colour
// row `color` of the table; with the 8-bit bt601 row this is cv2 COLOR_YUV2RGB_NV12 / _I420 bit for bit.
template <int kFmt>
__device__ __forceinline__ void decode_yuv420(const uint8_t* __restrict__ in, float* __restrict__ lr_curr, int b,
                                              int t, int h, int w, int x_tiles, int color) {
  using F = Yuv<kFmt>;
  using W = typename F::Word;
  constexpr int kB = (int)sizeof(W);
  __shared__ __align__(16) uint8_t sy[2][kTilePx * kB + 16];
  __shared__ __align__(16) uint8_t sc[2][kTilePx * kB + 16];   // NV12 layout: sc[0] = U V U V ...; I420: U, V
  const int xt = b % x_tiles, r = b / x_tiles;
  const int hp = h >> 1, yp = r % hp, img = r / hp;
  const int x0 = xt * kTilePx;
  const int npx = min(kTilePx, w - x0);                      // even: w and x0 are
  const W* frame = reinterpret_cast<const W*>(in) + (size_t)img * (3 * hp) * w;
  const W* yrow = frame + (size_t)(2 * yp) * w + x0;
  const W* crow = frame + (size_t)h * w;                     // chroma of the frame
  const uint8_t* ysrc = reinterpret_cast<const uint8_t*>(yrow);
  const uint8_t* csrc = reinterpret_cast<const uint8_t*>(crow);
  const uint8_t* c0 = csrc + (F::kInterleaved ? (size_t)yp * w + x0 : (size_t)yp * (w >> 1) + (x0 >> 1)) * kB;
  const uint8_t* c1 = c0 + (size_t)hp * (w >> 1) * kB;        // I420 layout: the V sample of the same block
  stage_bytes(sy[0], ysrc, npx * kB, t);
  stage_bytes(sy[1], ysrc + (size_t)w * kB, npx * kB, t);
  if (F::kInterleaved) {
    stage_bytes(sc[0], c0, npx * kB, t);
  } else {
    stage_bytes(sc[0], c0, (npx >> 1) * kB, t);
    stage_bytes(sc[1], c1, (npx >> 1) * kB, t);
  }
  __syncthreads();
  if (t >= npx) return;
  // the staged words start at the sources' offsets within 16 bytes (cheaper to recompute than to keep live)
  const int ly0 = lead_of(ysrc), ly1 = lead_of(ysrc + (size_t)w * kB), lc0 = lead_of(c0);
  const int lc1 = F::kInterleaved ? 0 : lead_of(c1);
  // the leads are multiples of the word size: sources are word aligned
  const auto at = [](const uint8_t* sb, int lead, int j) { return F::sample(reinterpret_cast<const W*>(sb + lead)[j]); };
  const int j = t >> 1;
  const int u = F::kInterleaved ? at(sc[0], lc0, 2 * j) : at(sc[0], lc0, j);
  const int v = F::kInterleaved ? at(sc[0], lc0, 2 * j + 1) : at(sc[1], lc1, j);
  const int* k = c_yuv.v[F::k10][color];
  constexpr int kHalf = 1 << (F::kShift - 1);
  const int ruv = kHalf + k[13] * (v - F::kCoff);
  const int guv = kHalf + k[12] * (v - F::kCoff) + k[11] * (u - F::kCoff);
  const int buv = kHalf + k[10] * (u - F::kCoff);
  const int cy = k[9], yoff = k[15];
  const bool cv2_clamp = !F::k10 && color == 0;              // cv2: max(Y - 16, 0) before the multiply
  constexpr float kScale = F::k10 ? 1023.f : 255.f;
  auto rgb = [](int a) { return __fdiv_rn((float)min(max(a >> F::kShift, 0), F::kTop), kScale); };
  const size_t plane = (size_t)h * w;
  float* dst = lr_curr + (size_t)img * 3 * plane + (size_t)(2 * yp) * w + x0 + t;
#pragma unroll
  for (int dy = 0; dy < 2; ++dy) {
    int yv = at(sy[dy], dy ? ly1 : ly0, t) - yoff;
    if (cv2_clamp) yv = max(yv, 0);
    const int yy = yv * cy;
    dst[dy * w] = rgb(yy + ruv);
    dst[dy * w + plane] = rgb(yy + guv);
    dst[dy * w + 2 * plane] = rgb(yy + buv);
  }
}

// one pixel's RGB from its Y and the (U, V) it takes, colour row `color`: the per-pixel rule of decode_yuv420
template <int kFmt>
struct YuvDecode {
  using F = Yuv<kFmt>;
  int ruv, guv, buv, cy, yoff;
  bool cv2_clamp;
  __device__ __forceinline__ YuvDecode(int u, int v, int color) {
    const int* k = c_yuv.v[F::k10][color];
    constexpr int kHalf = 1 << (F::kShift - 1);
    ruv = kHalf + k[13] * (v - F::kCoff);
    guv = kHalf + k[12] * (v - F::kCoff) + k[11] * (u - F::kCoff);
    buv = kHalf + k[10] * (u - F::kCoff);
    cy = k[9], yoff = k[15];
    cv2_clamp = !F::k10 && color == 0;                          // cv2: max(Y - 16, 0) before the multiply
  }
  // dst[0], dst[plane], dst[2 * plane] = R, G, B / 255 (8 bit) or / 1023 (10 bit)
  __device__ __forceinline__ void put(float* dst, size_t plane, int y) const {
    constexpr float kScale = F::k10 ? 1023.f : 255.f;
    auto rgb = [](int a) { return __fdiv_rn((float)min(max(a >> F::kShift, 0), F::kTop), kScale); };
    int yv = y - yoff;
    if (cv2_clamp) yv = max(yv, 0);
    const int yy = yv * cy;
    dst[0] = rgb(yy + ruv);
    dst[plane] = rgb(yy + guv);
    dst[2 * plane] = rgb(yy + buv);
  }
};

// decode CTA of packed 4:2:2 frames ([h, 2w] bytes each): kTilePx pixel pairs of one row, one 4-byte group per
// thread; both pixels of a pair take its U and V (nearest chroma).  With the 8-bit bt601 row this is cv2
// COLOR_YUV2RGB_YUY2 / _UYVY bit for bit.  The frames are 4-byte aligned (the launch checks).
template <int kFmt>
__device__ __forceinline__ void decode_yuv422(const uint8_t* __restrict__ in, float* __restrict__ lr_curr, int b,
                                              int t, int h, int w, int x_tiles, int color) {
  using F = Yuv<kFmt>;
  const int xt = b % x_tiles, r = b / x_tiles;
  const int y = r % h, img = r / h;
  const int pair = xt * kTilePx + t;
  if (pair >= (w >> 1)) return;
  const uint32_t g = __ldg(reinterpret_cast<const uint32_t*>(in) + ((size_t)img * h + y) * (w >> 1) + pair);
  const auto byte = [g](int k) { return (int)((g >> (8 * k)) & 255u); };
  const YuvDecode<kFmt> d(byte(packed_u(kFmt)), byte(packed_u(kFmt) + 2), color);
  const size_t plane = (size_t)h * w;
  float* dst = lr_curr + (size_t)img * 3 * plane + (size_t)y * w + 2 * pair;
  d.put(dst, plane, byte(packed_y0(kFmt)));
  d.put(dst + 1, plane, byte(packed_y0(kFmt) + 2));
}

// decode CTA of planar 4:4:4 frames ([3h, w] words each: the Y, U and V planes): kTilePx pixels of one row, one
// sample of each plane per thread (coalesced word loads)
template <int kFmt>
__device__ __forceinline__ void decode_yuv444(const uint8_t* __restrict__ in, float* __restrict__ lr_curr, int b,
                                              int t, int h, int w, int x_tiles, int color) {
  using F = Yuv<kFmt>;
  using W = typename F::Word;
  const int xt = b % x_tiles, r = b / x_tiles;
  const int y = r % h, img = r / h;
  const int x = xt * kTilePx + t;
  if (x >= w) return;
  const size_t plane = (size_t)h * w;
  const W* src = reinterpret_cast<const W*>(in) + (size_t)img * 3 * plane + (size_t)y * w + x;
  const YuvDecode<kFmt> d(F::sample(__ldg(src + plane)), F::sample(__ldg(src + 2 * plane)), color);
  d.put(lr_curr + (size_t)img * 3 * plane + (size_t)y * w + x, plane, F::sample(__ldg(src)));
}

// blockIdx.x < decode_ctas: decode CTA, row-major over x tiles (kHWC, 4:2:2, 4:4:4: one image row; 4:2:0: a pair
// of rows);
// the rest: zpc CTAs per slot, each zeroing a strided share of that slot's lr_prev and hr_prev when flagged.
template <int kFmt>
__global__ void __launch_bounds__(kThreads)
stream_frame_in_kernel(const uint8_t* __restrict__ in, const int32_t* __restrict__ reset,
                       float* __restrict__ lr_curr, float* __restrict__ lr_prev, float* __restrict__ hr_prev,
                       int c, int h, int w, int s, int bgr, int x_tiles, int decode_ctas, int zpc, int color) {
  // lr_curr, lr_prev and hr_prev belong to the previous step until it has finished
  tg_pdl_wait();
  tg_pdl_trigger();
  const int t = threadIdx.x;
  const int b = blockIdx.x;
  if (b < decode_ctas) {
    if constexpr (kFmt == kHWC)
      decode_hwc(in, lr_curr, b, t, c, h, w, bgr, x_tiles);
    else if constexpr (fmt_packed(kFmt))
      decode_yuv422<kFmt>(in, lr_curr, b, t, h, w, x_tiles, color);
    else if constexpr (fmt_444(kFmt))
      decode_yuv444<kFmt>(in, lr_curr, b, t, h, w, x_tiles, color);
    else
      decode_yuv420<kFmt>(in, lr_curr, b, t, h, w, x_tiles, color);
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
                    float* hr_prev, int n, int c, int h, int w, int s, int bgr, int color, cudaStream_t stream) {
  TG_REQUIRE(in || reset, TG_E_INVALID, "%s: in_u8 and reset are both NULL", name);
  TG_REQUIRE(lr_curr && lr_prev && hr_prev, TG_E_INVALID, "%s: null pointer (lr_curr / lr_prev / hr_prev)", name);
  TG_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0, TG_E_INVALID, "%s: bad size n=%d c=%d h=%d w=%d", name, n, c, h, w);
  TG_REQUIRE(c <= kMaxC, TG_E_UNSUPPORTED, "%s: %d channels (at most %d)", name, c, kMaxC);
  constexpr bool k420 = fmt_420(kFmt);
  TG_REQUIRE(!k420 || (h % 2 == 0 && w % 2 == 0), TG_E_UNSUPPORTED,
             "%s: YUV 4:2:0 needs an even height and width, got %dx%d", name, h, w);
  TG_REQUIRE(!fmt_packed(kFmt) || w % 2 == 0, TG_E_UNSUPPORTED, "%s: YUV 4:2:2 needs an even width, got %d", name,
             w);
  TG_REQUIRE(s == 2 || s == 4, TG_E_UNSUPPORTED, "%s: scale %d (2 or 4)", name, s);
  TG_REQUIRE((((uintptr_t)lr_curr | (uintptr_t)lr_prev | (uintptr_t)hr_prev) & 3u) == 0, TG_E_INVALID,
             "%s: fp32 buffers must be 4-byte aligned", name);
  TG_REQUIRE(!fmt_10(kFmt) || ((uintptr_t)in & 1u) == 0, TG_E_INVALID,
             "%s: 10-bit frames must be 2-byte aligned", name);
  TG_REQUIRE(!fmt_packed(kFmt) || ((uintptr_t)in & 3u) == 0, TG_E_INVALID,
             "%s: packed 4:2:2 frames must be 4-byte aligned", name);
  const int x_tiles = tg_ceil_div(fmt_packed(kFmt) ? w / 2 : w, kTilePx);
  const size_t decode = in ? (size_t)x_tiles * (k420 ? h / 2 : h) * n : 0;
  const size_t hr4 = (size_t)c * s * h * s * w / 4;
  const int zpc = reset ? (int)(hr4 / (kThreads * 8) + 1 < 64 ? hr4 / (kThreads * 8) + 1 : 64) : 0;
  const size_t ctas = decode + (size_t)zpc * n;
  TG_REQUIRE(ctas <= 0x7fffffff, TG_E_UNSUPPORTED, "%s: grid too large", name);
  tg_launch(stream_frame_in_kernel<kFmt>, dim3((unsigned)ctas), dim3(kThreads), 0, stream,
            static_cast<const uint8_t*>(in), reset, lr_curr, lr_prev, hr_prev, c, h, w, s, bgr, x_tiles, (int)decode,
            zpc, color);
  TG_CUDA_LAUNCH_CHECK(name);
  return TG_OK;
}

// one CTA: kTilePx pixels of the RGB rows 2*yp and 2*yp + 1 -> their Y words and the chroma words of the pair
// (U and V of a 2x2 block from its top-left pixel, as cv2 COLOR_RGB2YUV_I420).  The source is the step's uint8
// NHWC RGB (8-bit output; staged with 16-byte loads) or its fp32 NCHW HR frame (kF32, 10-bit output: coalesced
// row reads of the three planes, q = clip(rint(x * 1023), 0, 1023)).  Colour row `color` of the table.
template <int kFmt, bool kF32>
__global__ void __launch_bounds__(kThreads)
rgb_to_yuv420_kernel(const void* __restrict__ rgb, uint8_t* __restrict__ out, int H, int W, int x_tiles,
                     int color) {
  using F = Yuv<kFmt>;
  using Wd = typename F::Word;
  static_assert(kF32 == F::k10, "8-bit output reads uint8 RGB, 10-bit output the fp32 frame");
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
  int li0 = 0, li1 = 0;
  if constexpr (!kF32) {
    const uint8_t* src = static_cast<const uint8_t*>(rgb) + (((size_t)img * H + 2 * yp) * W + x0) * 3;
    li0 = stage_bytes(sin[0], src, npx * 3, t);
    li1 = stage_bytes(sin[1], src + (size_t)W * 3, npx * 3, t);
  }
  Wd* frame = reinterpret_cast<Wd*>(out) + (size_t)img * (3 * hp) * W;
  Wd* yrow = frame + (size_t)(2 * yp) * W + x0;
  Wd* crow = frame + (size_t)H * W;
  Wd *c0, *c1 = nullptr;
  if (F::kInterleaved) {
    c0 = crow + (size_t)yp * W + x0;
  } else {
    c0 = crow + (size_t)yp * (W >> 1) + (x0 >> 1);
    c1 = c0 + (size_t)hp * (W >> 1);
  }
  const int ly0 = lead_of(yrow), ly1 = lead_of(yrow + W), lc0 = lead_of(c0), lc1 = F::kInterleaved ? 0 : lead_of(c1);
  auto put = [](uint8_t* sb, int lead, int j, int v) { reinterpret_cast<Wd*>(sb + lead)[j] = F::word(v); };
  const int* k = c_yuv.v[F::k10][color];
  constexpr int kHalf = 1 << (F::kShift - 1);
  const int yoff = k[15] << F::kShift;
  constexpr int coff = F::kCoff << F::kShift;
  auto q = [](int a) { return min(max(a >> F::kShift, 0), F::kTop); };
  if constexpr (!kF32) __syncthreads();
  if (t < npx) {
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
      int R, G, B;
      if constexpr (kF32) {
        const size_t plane = (size_t)H * W;
        const float* p = static_cast<const float*>(rgb) + (size_t)img * 3 * plane + (size_t)(2 * yp + dy) * W + x0 + t;
        auto q10 = [](float x) { return (int)fminf(fmaxf(rintf(x * 1023.f), 0.f), 1023.f); };
        R = q10(__ldg(p));
        G = q10(__ldg(p + plane));
        B = q10(__ldg(p + 2 * plane));
      } else {
        const uint8_t* p = sin[dy] + (dy ? li1 : li0) + 3 * t;
        R = p[0], G = p[1], B = p[2];
      }
      put(sy[dy], dy ? ly1 : ly0, t, q(k[0] * R + k[1] * G + k[2] * B + kHalf + yoff));
      if (dy == 0 && (t & 1) == 0) {
        const int u = q(k[3] * R + k[4] * G + k[5] * B + kHalf + coff);
        const int v = q(k[6] * R + k[7] * G + k[8] * B + kHalf + coff);
        if (F::kInterleaved) {
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
  flush(yrow + W, sy[1], npx);
  if (F::kInterleaved) {
    flush(c0, sc[0], npx);
  } else {
    flush(c0, sc[0], npx >> 1);
    flush(c1, sc[1], npx >> 1);
  }
}

// one CTA: kTilePx pixel pairs of one uint8 NHWC RGB row (6 bytes a pair, staged with 16-byte loads) -> one
// 4-byte YUY2 / UYVY group per pair: Y of each pixel, U and V of the pair's sum (c_yuv422 row `color`)
template <int kFmt>
__global__ void __launch_bounds__(kThreads)
rgb_to_yuv422_kernel(const uint8_t* __restrict__ rgb, uint8_t* __restrict__ out, int H, int W, int x_tiles,
                     int color) {
  using F = Yuv<kFmt>;
  static_assert(fmt_packed(kFmt) && !F::k10, "packed 4:2:2 is 8 bit");
  __shared__ __align__(16) uint8_t sin[kTilePx * 6 + 16];
  // rgb is the previous kernel's output; out may still be read by the copy of an earlier step
  tg_pdl_wait();
  tg_pdl_trigger();
  const int t = threadIdx.x;
  const int xt = blockIdx.x % x_tiles, r = blockIdx.x / x_tiles;
  const int y = r % H, img = r / H;
  const int p0 = xt * kTilePx;
  const int npair = min(kTilePx, (W >> 1) - p0);
  const size_t row = (size_t)img * H + y;
  const int li = stage_bytes(sin, rgb + (row * W + 2 * p0) * 3, npair * 6, t);
  __syncthreads();
  if (t >= npair) return;
  const uint8_t* p = sin + li + 6 * t;
  const int R0 = p[0], G0 = p[1], B0 = p[2], R1 = p[3], G1 = p[4], B1 = p[5];
  const int* k = c_yuv422.v[color];
  const int sy = k[9], sc = k[10];
  const int yo = (c_yuv.v[0][color][15] << sy) + (1 << (sy - 1));
  const int co = (F::kCoff << sc) + (1 << (sc - 1));
  auto q = [](int a, int s) { return (uint32_t)min(max(a >> s, 0), 255); };
  const uint32_t y0 = q(k[0] * R0 + k[1] * G0 + k[2] * B0 + yo, sy);
  const uint32_t y1 = q(k[0] * R1 + k[1] * G1 + k[2] * B1 + yo, sy);
  const int sr = R0 + R1, sg = G0 + G1, sb = B0 + B1;
  const uint32_t u = q(k[3] * sr + k[4] * sg + k[5] * sb + co, sc);
  const uint32_t v = q(k[6] * sr + k[7] * sg + k[8] * sb + co, sc);
  reinterpret_cast<uint32_t*>(out)[row * (W >> 1) + p0 + t] =
      y0 << (8 * packed_y0(kFmt)) | y1 << (8 * (packed_y0(kFmt) + 2)) | u << (8 * packed_u(kFmt)) |
      v << (8 * (packed_u(kFmt) + 2));
}

// one CTA: kTilePx pixels of one row -> their Y, U and V words in the three planes of a 4:4:4 frame.  The source is
// the uint8 NHWC RGB (8 bit, staged with 16-byte loads) or the fp32 NCHW HR frame (kF32, 10 bit, quantised as in
// rgb_to_yuv420_kernel).  Colour row `color` of the table, per pixel.
template <int kFmt, bool kF32>
__global__ void __launch_bounds__(kThreads)
rgb_to_yuv444_kernel(const void* __restrict__ rgb, uint8_t* __restrict__ out, int H, int W, int x_tiles,
                     int color) {
  using F = Yuv<kFmt>;
  using Wd = typename F::Word;
  static_assert(fmt_444(kFmt) && kF32 == F::k10, "8-bit output reads uint8 RGB, 10-bit output the fp32 frame");
  __shared__ __align__(16) uint8_t sin[kF32 ? 16 : kTilePx * 3 + 16];
  tg_pdl_wait();
  tg_pdl_trigger();
  const int t = threadIdx.x;
  const int xt = blockIdx.x % x_tiles, r = blockIdx.x / x_tiles;
  const int y = r % H, img = r / H;
  const int x0 = xt * kTilePx;
  const int npx = min(kTilePx, W - x0);
  const size_t plane = (size_t)H * W;
  int li = 0;
  if constexpr (!kF32) {
    li = stage_bytes(sin, static_cast<const uint8_t*>(rgb) + (((size_t)img * H + y) * W + x0) * 3, npx * 3, t);
    __syncthreads();
  }
  if (t >= npx) return;
  int R, G, B;
  if constexpr (kF32) {
    const float* p = static_cast<const float*>(rgb) + (size_t)img * 3 * plane + (size_t)y * W + x0 + t;
    auto q10 = [](float x) { return (int)fminf(fmaxf(rintf(x * 1023.f), 0.f), 1023.f); };
    R = q10(__ldg(p));
    G = q10(__ldg(p + plane));
    B = q10(__ldg(p + 2 * plane));
  } else {
    const uint8_t* p = sin + li + 3 * t;
    R = p[0], G = p[1], B = p[2];
  }
  const int* k = c_yuv.v[F::k10][color];
  constexpr int kHalf = 1 << (F::kShift - 1);
  constexpr int coff = F::kCoff << F::kShift;
  auto q = [](int a) { return F::word(min(max(a >> F::kShift, 0), F::kTop)); };
  Wd* dst = reinterpret_cast<Wd*>(out) + (size_t)img * 3 * plane + (size_t)y * W + x0 + t;
  dst[0] = q(k[0] * R + k[1] * G + k[2] * B + kHalf + (k[15] << F::kShift));
  dst[plane] = q(k[3] * R + k[4] * G + k[5] * B + kHalf + coff);
  dst[2 * plane] = q(k[6] * R + k[7] * G + k[8] * B + kHalf + coff);
}

template <int kFmt>
int launch_to_yuv(const char* name, const void* rgb, void* out, int n, int H, int W, int color,
                  cudaStream_t stream) {
  using F = Yuv<kFmt>;
  TG_REQUIRE(n > 0 && H > 0 && W > 0, TG_E_INVALID, "%s: bad size n=%d H=%d W=%d", name, n, H, W);
  TG_REQUIRE(fmt_packed(kFmt) || fmt_444(kFmt) || (H % 2 == 0 && W % 2 == 0), TG_E_UNSUPPORTED,
             "%s: YUV 4:2:0 needs an even height and width, got %dx%d", name, H, W);
  TG_REQUIRE(!fmt_packed(kFmt) || W % 2 == 0, TG_E_UNSUPPORTED, "%s: YUV 4:2:2 needs an even width, got %d", name, W);
  TG_REQUIRE(!fmt_packed(kFmt) || ((uintptr_t)out & 3u) == 0, TG_E_INVALID,
             "%s: packed 4:2:2 output must be 4-byte aligned", name);
  const int x_tiles = tg_ceil_div(fmt_packed(kFmt) ? W / 2 : W, kTilePx);
  const size_t ctas = (size_t)x_tiles * (fmt_packed(kFmt) || fmt_444(kFmt) ? H : H / 2) * n;
  TG_REQUIRE(ctas <= 0x7fffffff, TG_E_UNSUPPORTED, "%s: grid too large", name);
  uint8_t* o = static_cast<uint8_t*>(out);
  if constexpr (fmt_packed(kFmt))
    tg_launch(rgb_to_yuv422_kernel<kFmt>, dim3((unsigned)ctas), dim3(kThreads), 0, stream,
              static_cast<const uint8_t*>(rgb), o, H, W, x_tiles, color);
  else if constexpr (fmt_444(kFmt))
    tg_launch(rgb_to_yuv444_kernel<kFmt, F::k10>, dim3((unsigned)ctas), dim3(kThreads), 0, stream, rgb, o, H, W,
              x_tiles, color);
  else
    tg_launch(rgb_to_yuv420_kernel<kFmt, F::k10>, dim3((unsigned)ctas), dim3(kThreads), 0, stream, rgb, o, H, W,
              x_tiles, color);
  TG_CUDA_LAUNCH_CHECK(name);
  return TG_OK;
}

// tg_yuv_format -> (frame format, colour row)
int parse_yuv_format(const char* name, const tg_yuv_format* f, int* fmt, int* color) {
  TG_REQUIRE(f, TG_E_INVALID, "%s: null format", name);
  TG_REQUIRE(f->reserved == 0, TG_E_INVALID, "%s: format.reserved must be 0, got %d", name, f->reserved);
  TG_REQUIRE(f->full_range == 0 || f->full_range == 1, TG_E_INVALID, "%s: format.full_range must be 0 or 1, got %d",
             name, f->full_range);
  TG_REQUIRE(f->matrix == 601 || f->matrix == 709, TG_E_UNSUPPORTED, "%s: matrix %d (601 or 709)", name, f->matrix);
  switch (f->layout) {
    case TG_YUV_NV12: *fmt = kNV12; break;
    case TG_YUV_I420: *fmt = kI420; break;
    case TG_YUV_P010: *fmt = kP010; break;
    case TG_YUV_I420_10: *fmt = kI420_10; break;
    case TG_YUV_YUY2: *fmt = kYUY2; break;
    case TG_YUV_UYVY: *fmt = kUYVY; break;
    case TG_YUV_I444: *fmt = kI444; break;
    case TG_YUV_I444_10: *fmt = kI444_10; break;
    default: TG_REQUIRE(false, TG_E_UNSUPPORTED, "%s: unknown layout %d", name, f->layout);
  }
  *color = (f->matrix == 709 ? 1 : 0) + 2 * f->full_range;
  return TG_OK;
}

}  // namespace

extern "C" int tg_stream_frame_in(const uint8_t* in_u8, const int32_t* reset, float* lr_curr, float* lr_prev,
                                  float* hr_prev, int n, int c, int h, int w, int s, int bgr, void* stream) {
  return launch_frame_in<kHWC>("stream_frame_in", in_u8, reset, lr_curr, lr_prev, hr_prev, n, c, h, w, s, bgr, 0,
                               (cudaStream_t)stream);
}

extern "C" int tg_stream_frame_in_yuv420(const uint8_t* in, int nv12, const int32_t* reset, float* lr_curr,
                                         float* lr_prev, float* hr_prev, int n, int h, int w, int s, void* stream) {
  return nv12 ? launch_frame_in<kNV12>("stream_frame_in_yuv420", in, reset, lr_curr, lr_prev, hr_prev, n, 3, h, w,
                                       s, 0, 0, (cudaStream_t)stream)
              : launch_frame_in<kI420>("stream_frame_in_yuv420", in, reset, lr_curr, lr_prev, hr_prev, n, 3, h, w,
                                       s, 0, 0, (cudaStream_t)stream);
}

extern "C" int tg_rgb_u8_to_yuv420(const uint8_t* rgb, uint8_t* out, int nv12, int n, int H, int W, void* stream) {
  TG_REQUIRE(rgb && out, TG_E_INVALID, "rgb_u8_to_yuv420: null pointer (rgb / out)");
  return nv12 ? launch_to_yuv<kNV12>("rgb_u8_to_yuv420", rgb, out, n, H, W, 0, (cudaStream_t)stream)
              : launch_to_yuv<kI420>("rgb_u8_to_yuv420", rgb, out, n, H, W, 0, (cudaStream_t)stream);
}

extern "C" int tg_stream_frame_in_yuv(const void* in, const tg_yuv_format* fmt, const int32_t* reset, float* lr_curr,
                                      float* lr_prev, float* hr_prev, int n, int h, int w, int s, void* stream) {
  const char* name = "stream_frame_in_yuv";
  int f = 0, color = 0;
  const int rc = parse_yuv_format(name, fmt, &f, &color);
  if (rc != TG_OK) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  switch (f) {
    case kNV12: return launch_frame_in<kNV12>(name, in, reset, lr_curr, lr_prev, hr_prev, n, 3, h, w, s, 0, color, st);
    case kI420: return launch_frame_in<kI420>(name, in, reset, lr_curr, lr_prev, hr_prev, n, 3, h, w, s, 0, color, st);
    case kP010: return launch_frame_in<kP010>(name, in, reset, lr_curr, lr_prev, hr_prev, n, 3, h, w, s, 0, color, st);
    case kYUY2: return launch_frame_in<kYUY2>(name, in, reset, lr_curr, lr_prev, hr_prev, n, 3, h, w, s, 0, color, st);
    case kUYVY: return launch_frame_in<kUYVY>(name, in, reset, lr_curr, lr_prev, hr_prev, n, 3, h, w, s, 0, color, st);
    case kI444: return launch_frame_in<kI444>(name, in, reset, lr_curr, lr_prev, hr_prev, n, 3, h, w, s, 0, color, st);
    case kI444_10:
      return launch_frame_in<kI444_10>(name, in, reset, lr_curr, lr_prev, hr_prev, n, 3, h, w, s, 0, color, st);
    default:
      return launch_frame_in<kI420_10>(name, in, reset, lr_curr, lr_prev, hr_prev, n, 3, h, w, s, 0, color, st);
  }
}

extern "C" int tg_rgb_to_yuv(const uint8_t* rgb_u8, const float* rgb_f32, void* out, const tg_yuv_format* fmt, int n,
                             int H, int W, void* stream) {
  const char* name = "rgb_to_yuv";
  int f = 0, color = 0;
  const int rc = parse_yuv_format(name, fmt, &f, &color);
  if (rc != TG_OK) return rc;
  const bool ten = f == kP010 || f == kI420_10 || f == kI444_10;
  TG_REQUIRE(out, TG_E_INVALID, "%s: null pointer (out)", name);
  TG_REQUIRE(ten ? (rgb_f32 && !rgb_u8) : (rgb_u8 && !rgb_f32), TG_E_INVALID,
             "%s: %s output is encoded from %s (and only that source)", name, ten ? "10-bit" : "8-bit",
             ten ? "rgb_f32" : "rgb_u8");
  TG_REQUIRE(!ten || ((((uintptr_t)rgb_f32) & 3u) == 0 && (((uintptr_t)out) & 1u) == 0), TG_E_INVALID,
             "%s: rgb_f32 must be 4-byte and 10-bit output 2-byte aligned", name);
  const cudaStream_t st = (cudaStream_t)stream;
  switch (f) {
    case kNV12: return launch_to_yuv<kNV12>(name, rgb_u8, out, n, H, W, color, st);
    case kI420: return launch_to_yuv<kI420>(name, rgb_u8, out, n, H, W, color, st);
    case kP010: return launch_to_yuv<kP010>(name, rgb_f32, out, n, H, W, color, st);
    case kYUY2: return launch_to_yuv<kYUY2>(name, rgb_u8, out, n, H, W, color, st);
    case kUYVY: return launch_to_yuv<kUYVY>(name, rgb_u8, out, n, H, W, color, st);
    case kI444: return launch_to_yuv<kI444>(name, rgb_u8, out, n, H, W, color, st);
    case kI444_10: return launch_to_yuv<kI444_10>(name, rgb_f32, out, n, H, W, color, st);
    default: return launch_to_yuv<kI420_10>(name, rgb_f32, out, n, H, W, color, st);
  }
}

extern "C" int tg_yuv_coefficients(const tg_yuv_format* fmt, int32_t* out16) {
  int f = 0, color = 0;
  const int rc = parse_yuv_format("yuv_coefficients", fmt, &f, &color);
  if (rc != TG_OK) return rc;
  TG_REQUIRE(out16, TG_E_INVALID, "yuv_coefficients: null pointer (out16)");
  const int* r = kYuvTable.v[(f == kP010 || f == kI420_10 || f == kI444_10) ? 1 : 0][color];
  for (int k = 0; k < 16; ++k) out16[k] = r[k];
  return TG_OK;
}
