// The per-pixel decode of streamed frames, shared by the frame-input launches of tg_stream.cu and the resizing frame
// input of tg_resample.cu: the frame layouts (uint8 HWC; YUV 4:2:0 NV12 / I420 / P010 / I420_10, packed 4:2:2 YUY2 /
// UYVY, planar 4:4:4 I444 / I444_10, 10-bit 4:2:2 P210 / I422_10 / v210), the fixed-point colour table, the row decoders of the frame-input CTAs and the
// per-pixel sample fetch of any layout, the picture-window check and the format dispatch.  Every decoder computes the
// same fp32 value of a pixel: float(code) / 255 (8 bit) or / 1023 (10 bit) by IEEE division.
// Contract: include/tecogan_b200.h (tg_yuv_format, tg_frame_window, tg_stream_frame_in*).
#pragma once
#include <type_traits>

#include "tg_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kTilePx = 256;            // decode / encode CTA: kTilePx pixels of a row, one per thread
constexpr int kMaxC = 4;

enum FrameFormat { kHWC = 0, kNV12 = 1, kI420 = 2, kP010 = 3, kI420_10 = 4, kYUY2 = 5, kUYVY = 6, kI444 = 7,
                   kI444_10 = 8, kP210 = 9, kI422_10 = 10, kV210 = 11 };

constexpr bool fmt_10(int f) {
  return f == kP010 || f == kI420_10 || f == kI444_10 || f == kP210 || f == kI422_10 || f == kV210;
}
constexpr bool fmt_packed(int f) { return f == kYUY2 || f == kUYVY; }     // 4:2:2, one 4-byte group per pair
constexpr bool fmt_444(int f) { return f == kI444 || f == kI444_10; }     // three full-size planes
constexpr bool fmt_p422(int f) { return f == kP210 || f == kI422_10; }    // 10-bit 4:2:2, [2h, w] uint16 words
constexpr bool fmt_422(int f) { return fmt_packed(f) || fmt_p422(f) || f == kV210; }   // needs an even width
constexpr bool fmt_420(int f) { return f != kHWC && !fmt_422(f) && !fmt_444(f); }
// byte of Y0 (Y1 two bytes later) and of U (V two bytes later) in a packed group: YUY2 is Y0 U Y1 V, UYVY U Y0 V Y1
constexpr int packed_y0(int f) { return f == kUYVY ? 1 : 0; }
constexpr int packed_u(int f) { return f == kUYVY ? 0 : 1; }

template <int kFmt>
struct Yuv {
  static constexpr bool kInterleaved = kFmt == kNV12 || kFmt == kP010;     // NV12 plane layout
  static constexpr bool k10 = fmt_10(kFmt);
  // v210 packs its 10-bit samples into the 32-bit words of 16-byte groups: its frames are addressed in bytes
  using Word = typename std::conditional<k10 && kFmt != kV210, uint16_t, uint8_t>::type;
  static constexpr int kShift = k10 ? 18 : 20;                              // fraction bits of the table row
  static constexpr int kTop = k10 ? 1023 : 255;
  static constexpr int kCoff = k10 ? 512 : 128;
  static constexpr bool kHigh = kFmt == kP010 || kFmt == kP210;           // sample in the high 10 bits
  // the sample of a stored word: P010 / P210 keep it in the high 10 bits, I420_10 / I444_10 / I422_10 in the low 10
  // (larger words clamp)
  static __device__ __forceinline__ int sample(Word v) {
    return kHigh ? (int)(v >> 6) : (kFmt == kI420_10 || kFmt == kI444_10 || kFmt == kI422_10) ? min((int)v, 1023)
                                                                                             : (int)v;
  }
  static __device__ __forceinline__ Word word(int v) { return (Word)(kHigh ? v << 6 : v); }
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
static_assert(Yuv<kP210>::kShift == 18 && Yuv<kI422_10>::kTop == 1023 && Yuv<kV210>::kCoff == 512 &&
                  sizeof(Yuv<kP210>::Word) == 2 && sizeof(Yuv<kV210>::Word) == 1 && !Yuv<kP210>::kInterleaved,
              "10-bit 4:2:2 is the 10-bit table row; v210 frames are bytes");

// v210: a row of a frame_w-pixel frame is 128 * ceil(frame_w / 48) bytes, ceil(frame_w / 6) 16-byte groups of 6
// pixels used.  The 12 fields of a group, f = 3 * word + k at bits 10k of word f / 3, are
//   Cb0 Y0 Cr0 Y1 Cb2 Y2 Cr2 Y3 Cb4 Y4 Cr4 Y5:
// Y of pixel j at field 2j + 1, Cb / Cr of pair p (pixels 2p, 2p + 1) at fields 4p / 4p + 2.
__host__ __device__ constexpr size_t v210_stride(int fw) { return (size_t)128 * ((fw + 47) / 48); }
__device__ __forceinline__ int v210_field(const uint32_t* g, int f) { return (int)((g[f / 3] >> (10 * (f % 3))) & 1023u); }

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

__device__ __forceinline__ int lead_of(const void* p) { return (int)((uintptr_t)p & 15u); }

// Every decode reads the h x w picture at (win.top, win.left) of frames of win.frame_h x win.frame_w pixels and
// writes the h x w lr_curr; the encodes write their H x W picture there.  {h, w, 0, 0} is the whole frame.

// the fp32 value of an 8-bit HWC code: IEEE division, == numpy float32(v) / 255.0 (paired_folder_dataset.py:49);
// v * (1/255) differs
__device__ __forceinline__ float hwc_value(int v) { return __fdiv_rn((float)v, 255.f); }

// decode CTA of HWC frames: kTilePx pixels of one image row
__device__ __forceinline__ void decode_hwc(const uint8_t* __restrict__ in, float* __restrict__ lr_curr, int b, int t,
                                           int c, int h, int w, tg_frame_window win, int bgr, int x_tiles) {
  __shared__ __align__(16) uint8_t sb[kTilePx * kMaxC + 32];
  const int xt = b % x_tiles, r = b / x_tiles;
  const int y = r % h, img = r / h;
  const int x0 = xt * kTilePx;
  const int npx = min(kTilePx, w - x0);
  const size_t src = ((size_t)img * win.frame_h + win.top + y) * win.frame_w + win.left + x0;
  const int lead = stage_bytes(sb, in + src * c, npx * c, t);
  __syncthreads();
  if (t < npx) {
    float* dst = lr_curr + ((size_t)img * c * h + y) * w + x0 + t;
    const size_t plane = (size_t)h * w;
    for (int k = 0; k < c; ++k) {
      const int ks = bgr ? c - 1 - k : k;
      dst[k * plane] = hwc_value(sb[lead + t * c + ks]);
    }
  }
}

// decode CTA of YUV 4:2:0 frames ([3h/2, w] words each): kTilePx pixels of the luma rows 2*yp and 2*yp + 1 and
// the chroma samples they share (nearest chroma), written as RGB / 255 (8 bit) or RGB / 1023 (10 bit).  Colour
// row `color` of the table; with the 8-bit bt601 row this is cv2 COLOR_YUV2RGB_NV12 / _I420 bit for bit.
template <int kFmt>
__device__ __forceinline__ void decode_yuv420(const uint8_t* __restrict__ in, float* __restrict__ lr_curr, int b,
                                              int t, int h, int w, tg_frame_window win, int x_tiles, int color) {
  using F = Yuv<kFmt>;
  using W = typename F::Word;
  constexpr int kB = (int)sizeof(W);
  __shared__ __align__(16) uint8_t sy[2][kTilePx * kB + 16];
  __shared__ __align__(16) uint8_t sc[2][kTilePx * kB + 16];   // NV12 layout: sc[0] = U V U V ...; I420: U, V
  const int xt = b % x_tiles, r = b / x_tiles;
  const int hp = h >> 1, yp = r % hp, img = r / hp;
  const int x0 = xt * kTilePx;
  const int npx = min(kTilePx, w - x0);                      // even: w and x0 are
  const int fh = win.frame_h, fw = win.frame_w;              // even, as are top and left
  const int fx = win.left + x0, fyp = (win.top >> 1) + yp;   // the tile's column and row pair in the frame
  const W* frame = reinterpret_cast<const W*>(in) + (size_t)img * (3 * (fh >> 1)) * fw;
  const W* yrow = frame + (size_t)(2 * fyp) * fw + fx;
  const W* crow = frame + (size_t)fh * fw;                   // chroma of the frame
  const uint8_t* ysrc = reinterpret_cast<const uint8_t*>(yrow);
  const uint8_t* csrc = reinterpret_cast<const uint8_t*>(crow);
  const uint8_t* c0 = csrc + (F::kInterleaved ? (size_t)fyp * fw + fx : (size_t)fyp * (fw >> 1) + (fx >> 1)) * kB;
  const uint8_t* c1 = c0 + (size_t)(fh >> 1) * (fw >> 1) * kB;   // I420 layout: the V sample of the same block
  stage_bytes(sy[0], ysrc, npx * kB, t);
  stage_bytes(sy[1], ysrc + (size_t)fw * kB, npx * kB, t);
  if (F::kInterleaved) {
    stage_bytes(sc[0], c0, npx * kB, t);
  } else {
    stage_bytes(sc[0], c0, (npx >> 1) * kB, t);
    stage_bytes(sc[1], c1, (npx >> 1) * kB, t);
  }
  __syncthreads();
  if (t >= npx) return;
  // the staged words start at the sources' offsets within 16 bytes (cheaper to recompute than to keep live)
  const int ly0 = lead_of(ysrc), ly1 = lead_of(ysrc + (size_t)fw * kB), lc0 = lead_of(c0);
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
  // out(k, value) for k = 0, 1, 2: R, G, B / 255 (8 bit) or / 1023 (10 bit)
  template <class Out>
  __device__ __forceinline__ void emit(int y, Out out) const {
    constexpr float kScale = F::k10 ? 1023.f : 255.f;
    auto rgb = [](int a) { return __fdiv_rn((float)min(max(a >> F::kShift, 0), F::kTop), kScale); };
    int yv = y - yoff;
    if (cv2_clamp) yv = max(yv, 0);
    const int yy = yv * cy;
    out(0, rgb(yy + ruv));
    out(1, rgb(yy + guv));
    out(2, rgb(yy + buv));
  }
  // dst[0], dst[plane], dst[2 * plane] = R, G, B
  __device__ __forceinline__ void put(float* dst, size_t plane, int y) const {
    emit(y, [&](int k, float v) { dst[k * plane] = v; });
  }
  // v[0], v[1], v[2] = R, G, B
  __device__ __forceinline__ void rgb(int y, float* v) const {
    emit(y, [&](int k, float x) { v[k] = x; });
  }
};

// The samples (Y, U, V) of pixel (y, x) of frame `img` of n stored frames of layout kFmt (YUV), win.frame_h x
// win.frame_w pixels each; y and x count in the frame (the picture's offset added).  Nearest chroma: the sample of
// the 2x2 block (4:2:0) or of the pixel pair (4:2:2) the pixel lies in, as the row decoders above take it.
template <int kFmt>
__device__ __forceinline__ void yuv_samples(const uint8_t* __restrict__ in, tg_frame_window win, int img, int y, int x,
                                            int& Y, int& U, int& V) {
  using F = Yuv<kFmt>;
  using W = typename F::Word;
  const int fh = win.frame_h, fw = win.frame_w;
  if constexpr (fmt_packed(kFmt)) {
    const uint32_t g = __ldg(reinterpret_cast<const uint32_t*>(in) + ((size_t)img * fh + y) * (fw >> 1) + (x >> 1));
    const auto byte = [g](int k) { return (int)((g >> (8 * k)) & 255u); };
    Y = byte(packed_y0(kFmt) + 2 * (x & 1));
    U = byte(packed_u(kFmt));
    V = byte(packed_u(kFmt) + 2);
  } else if constexpr (kFmt == kV210) {
    const uint32_t* g = reinterpret_cast<const uint32_t*>(in + ((size_t)img * fh + y) * v210_stride(fw)) + 4 * (x / 6);
    const int j = x % 6, p = j >> 1;
    const auto field = [g](int f) { return (int)((__ldg(g + f / 3) >> (10 * (f % 3))) & 1023u); };
    Y = field(2 * j + 1);
    U = field(4 * p);
    V = field(4 * p + 2);
  } else if constexpr (fmt_p422(kFmt)) {
    const size_t fplane = (size_t)fh * fw;
    const W* frame = reinterpret_cast<const W*>(in) + (size_t)img * 2 * fplane;
    Y = F::sample(__ldg(frame + (size_t)y * fw + x));
    if (kFmt == kP210) {
      const W* c = frame + fplane + (size_t)y * fw + (x & ~1);
      U = F::sample(__ldg(c));
      V = F::sample(__ldg(c + 1));
    } else {
      const W* c = frame + fplane + (size_t)y * (fw >> 1) + (x >> 1);
      U = F::sample(__ldg(c));
      V = F::sample(__ldg(c + fplane / 2));
    }
  } else if constexpr (fmt_444(kFmt)) {
    const size_t fplane = (size_t)fh * fw;
    const W* src = reinterpret_cast<const W*>(in) + (size_t)img * 3 * fplane + (size_t)y * fw + x;
    Y = F::sample(__ldg(src));
    U = F::sample(__ldg(src + fplane));
    V = F::sample(__ldg(src + 2 * fplane));
  } else {
    const W* frame = reinterpret_cast<const W*>(in) + (size_t)img * (3 * (fh >> 1)) * fw;
    const W* chroma = frame + (size_t)fh * fw;
    Y = F::sample(__ldg(frame + (size_t)y * fw + x));
    if (F::kInterleaved) {
      const W* c = chroma + (size_t)(y >> 1) * fw + (x & ~1);
      U = F::sample(__ldg(c));
      V = F::sample(__ldg(c + 1));
    } else {
      const W* c = chroma + (size_t)(y >> 1) * (fw >> 1) + (x >> 1);
      U = F::sample(__ldg(c));
      V = F::sample(__ldg(c + (size_t)(fh >> 1) * (fw >> 1)));
    }
  }
}

// The fp32 value of pixel (y, x) of the picture at `win` of frame `img`, v[k] for channel k < c (HWC: c channels,
// reversed by bgr; YUV: the 3 RGB channels, colour row `color`): the value every frame-input decode writes there.
template <int kFmt>
__device__ __forceinline__ void decode_pixel(const uint8_t* __restrict__ in, tg_frame_window win, int c, int bgr,
                                             int color, int img, int y, int x, float* v) {
  y += win.top;
  x += win.left;
  if constexpr (kFmt == kHWC) {
    const uint8_t* p = in + (((size_t)img * win.frame_h + y) * win.frame_w + x) * c;
#pragma unroll
    for (int k = 0; k < kMaxC; ++k)
      if (k < c) v[k] = hwc_value(__ldg(p + (bgr ? c - 1 - k : k)));
  } else {
    int Y, U, V;
    yuv_samples<kFmt>(in, win, img, y, x, Y, U, V);
    YuvDecode<kFmt>(U, V, color).rgb(Y, v);
  }
}

// decode CTA of packed 4:2:2 frames ([h, 2w] bytes each): kTilePx pixel pairs of one row, one 4-byte group per
// thread; both pixels of a pair take its U and V (nearest chroma).  With the 8-bit bt601 row this is cv2
// COLOR_YUV2RGB_YUY2 / _UYVY bit for bit.  The frames are 4-byte aligned (the launch checks).
template <int kFmt>
__device__ __forceinline__ void decode_yuv422(const uint8_t* __restrict__ in, float* __restrict__ lr_curr, int b,
                                              int t, int h, int w, tg_frame_window win, int x_tiles, int color) {
  using F = Yuv<kFmt>;
  const int xt = b % x_tiles, r = b / x_tiles;
  const int y = r % h, img = r / h;
  const int pair = xt * kTilePx + t;
  if (pair >= (w >> 1)) return;
  const size_t frow = (size_t)img * win.frame_h + win.top + y;   // frame_w and left are even
  const uint32_t g =
      __ldg(reinterpret_cast<const uint32_t*>(in) + frow * (win.frame_w >> 1) + (win.left >> 1) + pair);
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
                                              int t, int h, int w, tg_frame_window win, int x_tiles, int color) {
  using F = Yuv<kFmt>;
  using W = typename F::Word;
  const int xt = b % x_tiles, r = b / x_tiles;
  const int y = r % h, img = r / h;
  const int x = xt * kTilePx + t;
  if (x >= w) return;
  const size_t plane = (size_t)h * w, fplane = (size_t)win.frame_h * win.frame_w;
  const W* src = reinterpret_cast<const W*>(in) + (size_t)img * 3 * fplane + (size_t)(win.top + y) * win.frame_w +
                 win.left + x;
  const YuvDecode<kFmt> d(F::sample(__ldg(src + fplane)), F::sample(__ldg(src + 2 * fplane)), color);
  d.put(lr_curr + (size_t)img * 3 * plane + (size_t)y * w + x, plane, F::sample(__ldg(src)));
}

// decode CTA of planar 10-bit 4:2:2 frames ([2h, w] uint16 words each: the Y plane, then P210's interleaved UV plane
// of h x w or I422_10's U and V planes of h x w/2): kTilePx pixel pairs of one row, one pair per thread; both
// pixels take the pair's U and V (nearest chroma)
template <int kFmt>
__device__ __forceinline__ void decode_yuv422_10(const uint8_t* __restrict__ in, float* __restrict__ lr_curr, int b,
                                                 int t, int h, int w, tg_frame_window win, int x_tiles, int color) {
  using F = Yuv<kFmt>;
  using W = typename F::Word;
  const int xt = b % x_tiles, r = b / x_tiles;
  const int y = r % h, img = r / h;
  const int pair = xt * kTilePx + t;
  if (pair >= (w >> 1)) return;
  const int fw = win.frame_w, fy = win.top + y, fx = win.left + 2 * pair;   // frame_w and left are even
  const size_t fplane = (size_t)win.frame_h * fw;
  const W* frame = reinterpret_cast<const W*>(in) + (size_t)img * 2 * fplane;
  const W* ys = frame + (size_t)fy * fw + fx;
  int u, v;
  if (kFmt == kP210) {
    const W* c = frame + fplane + (size_t)fy * fw + fx;
    u = F::sample(__ldg(c));
    v = F::sample(__ldg(c + 1));
  } else {
    const W* c = frame + fplane + (size_t)fy * (fw >> 1) + (fx >> 1);
    u = F::sample(__ldg(c));
    v = F::sample(__ldg(c + fplane / 2));
  }
  const YuvDecode<kFmt> d(u, v, color);
  const size_t plane = (size_t)h * w;
  float* dst = lr_curr + (size_t)img * 3 * plane + (size_t)y * w + 2 * pair;
  d.put(dst, plane, F::sample(__ldg(ys)));
  d.put(dst + 1, plane, F::sample(__ldg(ys + 1)));
}

// decode CTA of v210 frames ([h, v210_stride(frame_w)] bytes each): kTilePx 16-byte groups of one row, one group
// (6 pixels, 3 pairs) per thread with one 16-byte load; the pixels past w of a partial last group are not written.
// The frames are 16-byte aligned and the picture starts on a group (the launch checks).
__device__ __forceinline__ void decode_v210(const uint8_t* __restrict__ in, float* __restrict__ lr_curr, int b, int t,
                                            int h, int w, tg_frame_window win, int x_tiles, int color) {
  const int xt = b % x_tiles, r = b / x_tiles;
  const int y = r % h, img = r / h;
  const int grp = xt * kTilePx + t;
  const int x0 = 6 * grp;
  if (x0 >= w) return;
  const size_t frow = (size_t)img * win.frame_h + win.top + y;
  const uint4 q = __ldg(reinterpret_cast<const uint4*>(in + frow * v210_stride(win.frame_w)) + win.left / 6 + grp);
  const uint32_t g[4] = {q.x, q.y, q.z, q.w};
  const size_t plane = (size_t)h * w;
  float* dst = lr_curr + (size_t)img * 3 * plane + (size_t)y * w + x0;
#pragma unroll
  for (int p = 0; p < 3; ++p) {
    if (x0 + 2 * p >= w) break;                      // w is even: a pair is whole or absent
    const YuvDecode<kV210> d(v210_field(g, 4 * p), v210_field(g, 4 * p + 2), color);
    d.put(dst + 2 * p, plane, v210_field(g, 4 * p + 1));
    d.put(dst + 2 * p + 1, plane, v210_field(g, 4 * p + 3));
  }
}

// A window of an h x w picture in frames of layout kFmt: TG_E_INVALID outside the frame, TG_E_UNSUPPORTED off the
// chroma grid (4:2:0: even frame size, top and left; 4:2:2: even frame width and left; v210: the picture starts on
// a 6-pixel group and ends on one or at the frame's right edge)
template <int kFmt>
int check_window(const char* name, const tg_frame_window* win, int h, int w) {
  TG_REQUIRE(win, TG_E_INVALID, "%s: null window", name);
  const long long fh = win->frame_h, fw = win->frame_w, top = win->top, left = win->left;
  TG_REQUIRE(fh > 0 && fw > 0 && top >= 0 && left >= 0 && top + h <= fh && left + w <= fw, TG_E_INVALID,
             "%s: a %dx%d picture at (%lld, %lld) does not fit a %lldx%lld frame", name, h, w, top, left, fh, fw);
  TG_REQUIRE(!fmt_420(kFmt) || ((fh | fw | top | left) & 1) == 0, TG_E_UNSUPPORTED,
             "%s: YUV 4:2:0 needs an even frame size, top and left, got %lldx%lld at (%lld, %lld)", name, fh, fw, top,
             left);
  TG_REQUIRE(!fmt_422(kFmt) || ((fw | left) & 1) == 0, TG_E_UNSUPPORTED,
             "%s: YUV 4:2:2 needs an even frame width and left, got width %lld at column %lld", name, fw, left);
  TG_REQUIRE(kFmt != kV210 || (left % 6 == 0 && ((left + w) % 6 == 0 || left + w == fw)), TG_E_UNSUPPORTED,
             "%s: a v210 picture of width %d at column %lld of a %lld-wide frame must start on a 6-pixel group and "
             "end on one or at the frame's right edge", name, w, left, fw);
  return TG_OK;
}

// frame format kFmt -> fn(std::integral_constant<int, kFmt>)
template <class Fn>
int dispatch_format(int f, Fn&& fn) {
  switch (f) {
    case kHWC: return fn(std::integral_constant<int, kHWC>());
    case kNV12: return fn(std::integral_constant<int, kNV12>());
    case kI420: return fn(std::integral_constant<int, kI420>());
    case kP010: return fn(std::integral_constant<int, kP010>());
    case kI420_10: return fn(std::integral_constant<int, kI420_10>());
    case kYUY2: return fn(std::integral_constant<int, kYUY2>());
    case kUYVY: return fn(std::integral_constant<int, kUYVY>());
    case kI444: return fn(std::integral_constant<int, kI444>());
    case kP210: return fn(std::integral_constant<int, kP210>());
    case kI422_10: return fn(std::integral_constant<int, kI422_10>());
    case kV210: return fn(std::integral_constant<int, kV210>());
    default: return fn(std::integral_constant<int, kI444_10>());
  }
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
    case TG_YUV_P210: *fmt = kP210; break;
    case TG_YUV_I422_10: *fmt = kI422_10; break;
    case TG_YUV_V210: *fmt = kV210; break;
    default: TG_REQUIRE(false, TG_E_UNSUPPORTED, "%s: unknown layout %d", name, f->layout);
  }
  *color = (f->matrix == 709 ? 1 : 0) + 2 * f->full_range;
  return TG_OK;
}

}  // namespace
