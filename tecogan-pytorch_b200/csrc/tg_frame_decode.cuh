// The per-pixel decode of streamed frames, shared by the frame-input launches of tg_stream.cu and the resizing frame
// input of tg_resample.cu: the frame layouts (uint8 HWC; YUV 4:2:0 NV12 / I420 / P010 / I420_10, packed 4:2:2 YUY2 /
// UYVY, planar 4:4:4 I444 / I444_10, 10-bit 4:2:2 P210 / I422_10 / v210) and what each of them is (Yuv), the
// fixed-point colour table, the row decoders of the frame-input CTAs and the per-pixel sample fetch of any layout,
// the frame and picture-window check and the format dispatch.  Every decoder computes the
// same fp32 value of a pixel: float(code) / 255 (8 bit) or / 1023 (10 bit) by IEEE division.
// Contract: include/tecogan_b200.h (tg_yuv_format, tg_frame_window, tg_stream_frame_in*).
#pragma once
#include <type_traits>

#include "tg_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kTilePx = 256;            // decode / encode CTA: kTilePx pixels (or units) of a row, one per thread
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

// v210: a row of a frame_w-pixel frame is 128 * ceil(frame_w / 48) bytes, ceil(frame_w / 6) 16-byte groups of 6
// pixels used.  The 12 fields of a group, f = 3 * word + k at bits 10k of word f / 3, are
//   Cb0 Y0 Cr0 Y1 Cb2 Y2 Cr2 Y3 Cb4 Y4 Cr4 Y5:
// Y of pixel j at field 2j + 1, Cb / Cr of pair p (pixels 2p, 2p + 1) at fields 4p / 4p + 2.
__host__ __device__ constexpr size_t v210_stride(int fw) { return (size_t)128 * ((fw + 47) / 48); }

// What a frame layout is: its words, chroma grid, alignment and where the Y, U and V samples of a pixel live.  The
// layout predicates above are read here only.
template <int kFmt>
struct Yuv {
  static constexpr bool k420 = fmt_420(kFmt), k422 = fmt_422(kFmt), k10 = fmt_10(kFmt);
  // packed 4:2:2 and v210 store a row as aligned groups of 32-bit words (a pair in 4 bytes, 6 pixels in 16); the
  // planar layouts store a Y plane and the chroma of the grid, U and V interleaved (kSemi) or in two planes
  static constexpr bool kGrouped = fmt_packed(kFmt) || kFmt == kV210;
  static constexpr bool kSemi = kFmt == kNV12 || kFmt == kP010 || kFmt == kP210;
  // the chroma grid: pixels that share one U, V sample (v210: the 6 pixels of a group, 3 pairs), and the pixels of
  // a row one thread of the row kernels owns (4:2:0: one pixel of each of two rows; else a pixel, a pair or a group)
  static constexpr int kGy = k420 ? 2 : 1;
  static constexpr int kGx = kFmt == kV210 ? 6 : k420 || k422 ? 2 : 1;
  static constexpr int kUnitPx = k420 || kFmt == kHWC ? 1 : kGx;
  // v210 packs its 10-bit samples into the 32-bit words of 16-byte groups: its frames are addressed in bytes
  using Word = typename std::conditional<k10 && kFmt != kV210, uint16_t, uint8_t>::type;
  // the widest access of a frame's unit: the group (packed 4:2:2, v210) or a word
  static constexpr int kAlign = kFmt == kV210 ? 16 : fmt_packed(kFmt) ? 4 : (int)sizeof(Word);
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

  // words of one fh x fw frame (kHWC: c bytes a pixel)
  static __host__ __device__ size_t frame_words(int c, int fh, int fw) {
    if (kFmt == kHWC) return (size_t)fh * fw * c;
    if (kGrouped) return (size_t)fh * row_bytes(fw);
    return (size_t)fh * fw + 2 * (size_t)(fh / kGy) * (fw / kGx);
  }
  // planar: word offsets in its frame of pixel (y, x)'s Y, and of the U and V it takes (nearest chroma): the offset
  // of its chroma sample in a chroma plane (chroma_at) plus that of the U or V plane (u_plane / v_plane, the same
  // for every pixel of a frame)
  static __device__ __forceinline__ size_t y_at(int fw, int y, int x) { return (size_t)y * fw + x; }
  static __device__ __forceinline__ size_t chroma_at(int fw, int y, int x) {
    const unsigned cy = (unsigned)y / kGy, cx = (unsigned)x / kGx;   // coordinates are non-negative
    return kSemi ? (size_t)cy * fw + 2 * cx : (size_t)cy * ((unsigned)fw / kGx) + cx;
  }
  static __host__ __device__ size_t u_plane(int fh, int fw) { return (size_t)fh * fw; }
  static __host__ __device__ size_t v_plane(int fh, int fw) {
    return u_plane(fh, fw) + (kSemi ? 1 : (size_t)((unsigned)fh / kGy) * ((unsigned)fw / kGx));
  }
  // grouped: bytes of a row, the byte offset of the group holding pixel (y, x) of frame img, and the fields of a
  // group: Y of its pixel j, U and V of its pair p.  A field is byte f of the group (packed: YUY2 is Y0 U Y1 V, UYVY
  // U Y0 V Y1) or the 10-bit field f (v210)
  static __host__ __device__ size_t row_bytes(int fw) { return kFmt == kV210 ? v210_stride(fw) : (size_t)2 * fw; }
  static __device__ __forceinline__ size_t group_at(int fh, int fw, int img, int y, int x) {
    return ((size_t)img * fh + y) * row_bytes(fw) + (size_t)(x / kGx) * kAlign;
  }
  static constexpr int kFieldBits = kFmt == kV210 ? 10 : 8, kFieldsPerWord = kFmt == kV210 ? 3 : 4;
  static constexpr int y_field(int j) { return kFmt == kV210 ? 2 * j + 1 : (kFmt == kUYVY ? 1 : 0) + 2 * j; }
  static constexpr int u_field(int p) { return kFmt == kV210 ? 4 * p : kFmt == kUYVY ? 0 : 1; }
  static constexpr int v_field(int p) { return u_field(p) + 2; }
  // field f of a group whose word f / kFieldsPerWord is w, and the bits of value v at field f
  static __device__ __forceinline__ int field(uint32_t w, int f) {
    return (int)((w >> (kFieldBits * (f % kFieldsPerWord))) & ((1u << kFieldBits) - 1));
  }
  static __device__ __forceinline__ uint32_t field_bits(int f, int v) {
    return (uint32_t)v << (kFieldBits * (f % kFieldsPerWord));
  }
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
static_assert(Yuv<kP210>::kShift == 18 && Yuv<kI422_10>::kTop == 1023 && Yuv<kV210>::kCoff == 512 &&
                  sizeof(Yuv<kP210>::Word) == 2 && sizeof(Yuv<kV210>::Word) == 1,
              "10-bit 4:2:2 is the 10-bit table row; v210 frames are bytes");

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

// one pixel's RGB from its Y and the (U, V) it takes, colour row `color` of the table.  With the 8-bit bt601 row
// this is cv2's COLOR_YUV2RGB_* bit for bit.
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
  const int fx = win.left + x0, fy = win.top + 2 * yp;       // the tile's column and first row in the frame
  const W* frame = reinterpret_cast<const W*>(in) + (size_t)img * F::frame_words(3, fh, fw);
  const uint8_t* ysrc = reinterpret_cast<const uint8_t*>(frame + F::y_at(fw, fy, fx));
  const W* chroma = frame + F::chroma_at(fw, fy, fx);
  const uint8_t* c0 = reinterpret_cast<const uint8_t*>(chroma + F::u_plane(fh, fw));
  const uint8_t* c1 = reinterpret_cast<const uint8_t*>(chroma + F::v_plane(fh, fw));   // I420 layout
  stage_bytes(sy[0], ysrc, npx * kB, t);
  stage_bytes(sy[1], ysrc + (size_t)fw * kB, npx * kB, t);
  if (F::kSemi) {
    stage_bytes(sc[0], c0, npx * kB, t);
  } else {
    stage_bytes(sc[0], c0, (npx >> 1) * kB, t);
    stage_bytes(sc[1], c1, (npx >> 1) * kB, t);
  }
  __syncthreads();
  if (t >= npx) return;
  // the staged words start at the sources' offsets within 16 bytes (cheaper to recompute than to keep live)
  const int ly0 = lead_of(ysrc), ly1 = lead_of(ysrc + (size_t)fw * kB), lc0 = lead_of(c0);
  const int lc1 = F::kSemi ? 0 : lead_of(c1);
  // the leads are multiples of the word size: sources are word aligned
  const auto at = [](const uint8_t* sb, int lead, int j) { return F::sample(reinterpret_cast<const W*>(sb + lead)[j]); };
  const int j = t >> 1;
  const int u = F::kSemi ? at(sc[0], lc0, 2 * j) : at(sc[0], lc0, j);
  const int v = F::kSemi ? at(sc[0], lc0, 2 * j + 1) : at(sc[1], lc1, j);
  const YuvDecode<kFmt> d(u, v, color);
  const size_t plane = (size_t)h * w;
  float* dst = lr_curr + (size_t)img * 3 * plane + (size_t)(2 * yp) * w + x0 + t;
#pragma unroll
  for (int dy = 0; dy < 2; ++dy) d.put(dst + dy * w, plane, at(sy[dy], dy ? ly1 : ly0, t));
}

// The samples of the kUnitPx pixels of a row one thread of the per-unit row kernels owns (packed 4:2:2 and
// P210 / I422_10: a pair; 4:4:4: a pixel; v210: a 6-pixel group): Y of each pixel, U and V of each pair (4:4:4: of
// the pixel).  Grouped layouts keep the group's 32-bit words (fields never set are 0), planar ones the samples.
template <int kFmt>
struct Unit {
  using F = Yuv<kFmt>;
  static constexpr int kPx = F::kUnitPx, kC = kPx > 1 ? kPx / 2 : 1;
  uint32_t w[F::kGrouped ? F::kAlign / 4 : kPx + 2] = {};
  __device__ __forceinline__ int get(int f, int i) const {
    return F::kGrouped ? F::field(w[f / F::kFieldsPerWord], f) : (int)w[i];
  }
  __device__ __forceinline__ void set(int f, int i, int v) {
    if (F::kGrouped) w[f / F::kFieldsPerWord] |= F::field_bits(f, v);
    else w[i] = (uint32_t)v;
  }
  __device__ __forceinline__ int y(int j) const { return get(F::y_field(j), j); }
  __device__ __forceinline__ int u(int p) const { return get(F::u_field(p), kPx); }
  __device__ __forceinline__ int v(int p) const { return get(F::v_field(p), kPx + 1); }
  __device__ __forceinline__ void set_y(int j, int v) { set(F::y_field(j), j, v); }
  __device__ __forceinline__ void set_uv(int p, int u, int v) {
    set(F::u_field(p), kPx, u);
    set(F::v_field(p), kPx + 1, v);
  }
};

// the unit whose first pixel is (y, x) of frame img (fh x fw pixels): one 4-byte (packed 4:2:2) or 16-byte (v210)
// load of its group, or one word of each plane per sample
template <int kFmt>
__device__ __forceinline__ Unit<kFmt> load_unit(const uint8_t* __restrict__ in, int fh, int fw, int img, int y, int x) {
  using F = Yuv<kFmt>;
  Unit<kFmt> q;
  if constexpr (kFmt == kV210) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(in + F::group_at(fh, fw, img, y, x)));
    q.w[0] = a.x, q.w[1] = a.y, q.w[2] = a.z, q.w[3] = a.w;
  } else if constexpr (F::kGrouped) {
    q.w[0] = __ldg(reinterpret_cast<const uint32_t*>(in + F::group_at(fh, fw, img, y, x)));
  } else {
    const typename F::Word* f = reinterpret_cast<const typename F::Word*>(in) + (size_t)img * F::frame_words(3, fh, fw);
#pragma unroll
    for (int j = 0; j < q.kPx; ++j) q.set_y(j, F::sample(__ldg(f + F::y_at(fw, y, x + j))));
    const typename F::Word* c = f + F::chroma_at(fw, y, x);
    q.set_uv(0, F::sample(__ldg(c + F::u_plane(fh, fw))), F::sample(__ldg(c + F::v_plane(fh, fw))));
  }
  return q;
}

// decode CTA of the per-unit layouts (packed 4:2:2, 4:4:4, 10-bit 4:2:2): kTilePx units of one row, one per thread;
// every pixel takes its pair's U and V (nearest chroma).  The pixels past w of a partial last v210 group are not
// written.  The frames are aligned to their group and the picture starts on one (the launch checks).
template <int kFmt>
__device__ __forceinline__ void decode_units(const uint8_t* __restrict__ in, float* __restrict__ lr_curr, int b, int t,
                                             int h, int w, tg_frame_window win, int x_tiles, int color) {
  using U = Unit<kFmt>;
  const int xt = b % x_tiles, r = b / x_tiles;
  const int y = r % h, img = r / h;
  const int x0 = (xt * kTilePx + t) * U::kPx;
  if (x0 >= w) return;
  const U q = load_unit<kFmt>(in, win.frame_h, win.frame_w, img, win.top + y, win.left + x0);
  const size_t plane = (size_t)h * w;
  float* dst = lr_curr + (size_t)img * 3 * plane + (size_t)y * w + x0;
#pragma unroll
  for (int p = 0; p < U::kC; ++p) {
    if (x0 + 2 * p >= w) break;                      // w is even: a pair is whole or absent
    const YuvDecode<kFmt> d(q.u(p), q.v(p), color);
#pragma unroll
    for (int j = 0; j < U::kPx / U::kC; ++j) d.put(dst + 2 * p + j, plane, q.y(2 * p + j));
  }
}

// The samples (Y, U, V) of pixel (y, x) of frame `img` of n stored frames of layout kFmt (YUV), win.frame_h x
// win.frame_w pixels each; y and x count in the frame (the picture's offset added).  Nearest chroma, as the row
// decoders above take it.
template <int kFmt>
__device__ __forceinline__ void yuv_samples(const uint8_t* __restrict__ in, tg_frame_window win, int img, int y, int x,
                                            int& Y, int& U, int& V) {
  using F = Yuv<kFmt>;
  const int fh = win.frame_h, fw = win.frame_w;
  if constexpr (F::kGrouped) {
    // one load of a packed group; the words of a v210 group that hold the three fields
    const uint32_t* g = reinterpret_cast<const uint32_t*>(in + F::group_at(fh, fw, img, y, x));
    const int j = x % F::kGx;
    const auto get = [g](int f) { return F::field(__ldg(g + f / F::kFieldsPerWord), f); };
    Y = get(F::y_field(j));
    U = get(F::u_field(j >> 1));
    V = get(F::v_field(j >> 1));
  } else {
    const typename F::Word* f = reinterpret_cast<const typename F::Word*>(in) + (size_t)img * F::frame_words(3, fh, fw);
    Y = F::sample(__ldg(f + F::y_at(fw, y, x)));
    const typename F::Word* c = f + F::chroma_at(fw, y, x);
    U = F::sample(__ldg(c + F::u_plane(fh, fw)));
    V = F::sample(__ldg(c + F::v_plane(fh, fw)));
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

// The frames an h x w picture of layout kFmt is read from or written to, at `win` (nullptr: the whole frame), by a
// kernel whose widest access of the frames at p is `align` bytes: TG_E_UNSUPPORTED for a picture off the chroma
// grid (4:2:0: even height and width; 4:2:2: even width), TG_E_INVALID for misaligned frames, and for a window
// (checked when p is given) TG_E_INVALID outside the frame, TG_E_UNSUPPORTED off the chroma grid (4:2:0: even frame
// size, top and left; 4:2:2: even frame width and left; v210: the picture starts on a 6-pixel group and ends on
// one or at the frame's right edge).  `what` names the frames in the messages.
template <int kFmt>
int check_frames(const char* name, const void* p, int h, int w, const tg_frame_window* win, int align,
                 const char* what = "frames") {
  using F = Yuv<kFmt>;
  TG_REQUIRE(!F::k420 || (h % 2 == 0 && w % 2 == 0), TG_E_UNSUPPORTED,
             "%s: YUV 4:2:0 needs an even height and width, got %dx%d", name, h, w);
  TG_REQUIRE(!F::k422 || w % 2 == 0, TG_E_UNSUPPORTED, "%s: YUV 4:2:2 needs an even width, got %d", name, w);
  const uintptr_t a = (uintptr_t)p;
  TG_REQUIRE(!F::k10 || (a & 1u) == 0, TG_E_INVALID, "%s: 10-bit %s must be 2-byte aligned", name, what);
  TG_REQUIRE(!F::kGrouped || (a & (uintptr_t)(align - 1)) == 0, TG_E_INVALID, "%s: %s %s must be %d-byte aligned",
             name, kFmt == kV210 ? "v210" : "packed 4:2:2", what, align);
  if (!p || !win) return TG_OK;
  const long long fh = win->frame_h, fw = win->frame_w, top = win->top, left = win->left;
  TG_REQUIRE(fh > 0 && fw > 0 && top >= 0 && left >= 0 && top + h <= fh && left + w <= fw, TG_E_INVALID,
             "%s: a %dx%d picture at (%lld, %lld) does not fit a %lldx%lld frame", name, h, w, top, left, fh, fw);
  TG_REQUIRE(!F::k420 || ((fh | fw | top | left) & 1) == 0, TG_E_UNSUPPORTED,
             "%s: YUV 4:2:0 needs an even frame size, top and left, got %lldx%lld at (%lld, %lld)", name, fh, fw, top,
             left);
  TG_REQUIRE(!F::k422 || ((fw | left) & 1) == 0, TG_E_UNSUPPORTED,
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
