// Frame I/O of one streamed inference step: uint8 HWC or YUV 4:2:0 (NV12 / I420) frames decoded on the device
// into the step's fp32 NCHW lr_curr, the per-slot reset of the recurrent state, and the encode of the step's
// uint8 RGB output into NV12 / I420.  Contract: include/tecogan_b200.h (tg_stream_frame_in,
// tg_stream_frame_in_yuv420, tg_rgb_u8_to_yuv420).
#include "tg_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kTilePx = 256;            // decode / encode CTA: kTilePx pixels of a row, one per thread
constexpr int kMaxC = 4;

enum FrameFormat { kHWC = 0, kNV12 = 1, kI420 = 2 };

// cv2's BT.601 limited-range YUV 4:2:0 conversions (color_yuv: 20-bit fixed point); oracle/yuv_oracle.py restates
// them in numpy.  Every intermediate fits in int32: |sum| < 2^30.
constexpr int kShift = 20, kHalf = 1 << (kShift - 1);
constexpr int kCRY = 269484, kCGY = 528482, kCBY = 102760;
constexpr int kCRU = -155188, kCGU = -305135, kCBU = 460324;
constexpr int kCRV = 460324, kCGV = -385875, kCBV = -74448;
constexpr int kCY = 1220542, kCUB = 2116026, kCUG = -409993, kCVG = -852492, kCVR = 1673527;

__device__ __forceinline__ int clamp_u8(int v) { return min(max(v, 0), 255); }

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

// decode CTA of YUV 4:2:0 frames ([3h/2, w] bytes each): kTilePx pixels of the luma rows 2*yp and 2*yp + 1 and
// the chroma samples they share (cv2 COLOR_YUV2RGB_NV12 / _I420: nearest chroma), written as RGB / 255
template <int kFmt>
__device__ __forceinline__ void decode_yuv420(const uint8_t* __restrict__ in, float* __restrict__ lr_curr, int b,
                                              int t, int h, int w, int x_tiles) {
  __shared__ __align__(16) uint8_t sy[2][kTilePx + 16];
  __shared__ __align__(16) uint8_t sc[2][kTilePx + 16];     // NV12: sc[0] = U V U V ...; I420: sc[0] = U, sc[1] = V
  const int xt = b % x_tiles, r = b / x_tiles;
  const int hp = h >> 1, yp = r % hp, img = r / hp;
  const int x0 = xt * kTilePx;
  const int npx = min(kTilePx, w - x0);                      // even: w and x0 are
  const uint8_t* frame = in + (size_t)img * (3 * hp) * w;
  const uint8_t* yrow = frame + (size_t)(2 * yp) * w + x0;
  const uint8_t* crow = frame + (size_t)h * w;               // chroma of the frame
  int lc0, lc1 = 0;
  const int ly0 = stage_bytes(sy[0], yrow, npx, t);
  const int ly1 = stage_bytes(sy[1], yrow + w, npx, t);
  if (kFmt == kNV12) {
    lc0 = stage_bytes(sc[0], crow + (size_t)yp * w + x0, npx, t);
  } else {
    const size_t cu = (size_t)yp * (w >> 1) + (x0 >> 1);
    lc0 = stage_bytes(sc[0], crow + cu, npx >> 1, t);
    lc1 = stage_bytes(sc[1], crow + (size_t)hp * (w >> 1) + cu, npx >> 1, t);
  }
  __syncthreads();
  if (t >= npx) return;
  const int j = t >> 1;
  const int u = kFmt == kNV12 ? sc[0][lc0 + 2 * j] : sc[0][lc0 + j];
  const int v = kFmt == kNV12 ? sc[0][lc0 + 2 * j + 1] : sc[1][lc1 + j];
  const int ruv = kHalf + kCVR * (v - 128);
  const int guv = kHalf + kCVG * (v - 128) + kCUG * (u - 128);
  const int buv = kHalf + kCUB * (u - 128);
  const size_t plane = (size_t)h * w;
  float* dst = lr_curr + (size_t)img * 3 * plane + (size_t)(2 * yp) * w + x0 + t;
#pragma unroll
  for (int dy = 0; dy < 2; ++dy) {
    const int yy = max((int)sy[dy][(dy ? ly1 : ly0) + t] - 16, 0) * kCY;
    dst[dy * w] = __fdiv_rn((float)clamp_u8((yy + ruv) >> kShift), 255.f);
    dst[dy * w + plane] = __fdiv_rn((float)clamp_u8((yy + guv) >> kShift), 255.f);
    dst[dy * w + 2 * plane] = __fdiv_rn((float)clamp_u8((yy + buv) >> kShift), 255.f);
  }
}

// blockIdx.x < decode_ctas: decode CTA, row-major over x tiles (kHWC: one image row; YUV: a pair of rows);
// the rest: zpc CTAs per slot, each zeroing a strided share of that slot's lr_prev and hr_prev when flagged.
template <int kFmt>
__global__ void __launch_bounds__(kThreads)
stream_frame_in_kernel(const uint8_t* __restrict__ in, const int32_t* __restrict__ reset,
                       float* __restrict__ lr_curr, float* __restrict__ lr_prev, float* __restrict__ hr_prev,
                       int c, int h, int w, int s, int bgr, int x_tiles, int decode_ctas, int zpc) {
  // lr_curr, lr_prev and hr_prev belong to the previous step until it has finished
  tg_pdl_wait();
  tg_pdl_trigger();
  const int t = threadIdx.x;
  const int b = blockIdx.x;
  if (b < decode_ctas) {
    if constexpr (kFmt == kHWC)
      decode_hwc(in, lr_curr, b, t, c, h, w, bgr, x_tiles);
    else
      decode_yuv420<kFmt>(in, lr_curr, b, t, h, w, x_tiles);
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
int launch_frame_in(const char* name, const uint8_t* in, const int32_t* reset, float* lr_curr, float* lr_prev,
                    float* hr_prev, int n, int c, int h, int w, int s, int bgr, cudaStream_t stream) {
  TG_REQUIRE(in || reset, TG_E_INVALID, "%s: in_u8 and reset are both NULL", name);
  TG_REQUIRE(lr_curr && lr_prev && hr_prev, TG_E_INVALID, "%s: null pointer (lr_curr / lr_prev / hr_prev)", name);
  TG_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0, TG_E_INVALID, "%s: bad size n=%d c=%d h=%d w=%d", name, n, c, h, w);
  TG_REQUIRE(c <= kMaxC, TG_E_UNSUPPORTED, "%s: %d channels (at most %d)", name, c, kMaxC);
  TG_REQUIRE(kFmt == kHWC || (h % 2 == 0 && w % 2 == 0), TG_E_UNSUPPORTED,
             "%s: YUV 4:2:0 needs an even height and width, got %dx%d", name, h, w);
  TG_REQUIRE(s == 2 || s == 4, TG_E_UNSUPPORTED, "%s: scale %d (2 or 4)", name, s);
  TG_REQUIRE((((uintptr_t)lr_curr | (uintptr_t)lr_prev | (uintptr_t)hr_prev) & 3u) == 0, TG_E_INVALID,
             "%s: fp32 buffers must be 4-byte aligned", name);
  const int x_tiles = tg_ceil_div(w, kTilePx);
  const size_t decode = in ? (size_t)x_tiles * (kFmt == kHWC ? h : h / 2) * n : 0;
  const size_t hr4 = (size_t)c * s * h * s * w / 4;
  const int zpc = reset ? (int)(hr4 / (kThreads * 8) + 1 < 64 ? hr4 / (kThreads * 8) + 1 : 64) : 0;
  const size_t ctas = decode + (size_t)zpc * n;
  TG_REQUIRE(ctas <= 0x7fffffff, TG_E_UNSUPPORTED, "%s: grid too large", name);
  tg_launch(stream_frame_in_kernel<kFmt>, dim3((unsigned)ctas), dim3(kThreads), 0, stream, in, reset, lr_curr,
            lr_prev, hr_prev, c, h, w, s, bgr, x_tiles, (int)decode, zpc);
  TG_CUDA_LAUNCH_CHECK(name);
  return TG_OK;
}

// one CTA: kTilePx pixels of the RGB rows 2*yp and 2*yp + 1 -> their Y bytes and the chroma bytes of the pair
// (cv2 COLOR_RGB2YUV_I420: U and V of a 2x2 block from its top-left pixel)
template <int kFmt>
__global__ void __launch_bounds__(kThreads)
rgb_u8_to_yuv420_kernel(const uint8_t* __restrict__ rgb, uint8_t* __restrict__ out, int H, int W, int x_tiles) {
  __shared__ __align__(16) uint8_t sin[2][kTilePx * 3 + 16];
  __shared__ __align__(16) uint8_t sy[2][kTilePx + 16];
  __shared__ __align__(16) uint8_t sc[2][kTilePx + 16];     // NV12: sc[0] = U V U V ...; I420: sc[0] = U, sc[1] = V
  // rgb is the previous kernel's output; out may still be read by the copy of an earlier step
  tg_pdl_wait();
  tg_pdl_trigger();
  const int t = threadIdx.x;
  const int xt = blockIdx.x % x_tiles, r = blockIdx.x / x_tiles;
  const int hp = H >> 1, yp = r % hp, img = r / hp;
  const int x0 = xt * kTilePx;
  const int npx = min(kTilePx, W - x0);                      // even
  const uint8_t* src = rgb + (((size_t)img * H + 2 * yp) * W + x0) * 3;
  const int li0 = stage_bytes(sin[0], src, npx * 3, t);
  const int li1 = stage_bytes(sin[1], src + (size_t)W * 3, npx * 3, t);
  uint8_t* frame = out + (size_t)img * (3 * hp) * W;
  uint8_t* yrow = frame + (size_t)(2 * yp) * W + x0;
  uint8_t* crow = frame + (size_t)H * W;
  uint8_t *c0, *c1 = nullptr;
  if (kFmt == kNV12) {
    c0 = crow + (size_t)yp * W + x0;
  } else {
    c0 = crow + (size_t)yp * (W >> 1) + (x0 >> 1);
    c1 = c0 + (size_t)hp * (W >> 1);
  }
  const int ly0 = lead_of(yrow), ly1 = lead_of(yrow + W), lc0 = lead_of(c0), lc1 = kFmt == kNV12 ? 0 : lead_of(c1);
  __syncthreads();
  if (t < npx) {
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
      const uint8_t* p = sin[dy] + (dy ? li1 : li0) + 3 * t;
      const int R = p[0], G = p[1], B = p[2];
      sy[dy][(dy ? ly1 : ly0) + t] =
          (uint8_t)clamp_u8((kCRY * R + kCGY * G + kCBY * B + kHalf + (16 << kShift)) >> kShift);
      if (dy == 0 && (t & 1) == 0) {
        const uint8_t u = (uint8_t)clamp_u8((kCRU * R + kCGU * G + kCBU * B + kHalf + (128 << kShift)) >> kShift);
        const uint8_t v = (uint8_t)clamp_u8((kCRV * R + kCGV * G + kCBV * B + kHalf + (128 << kShift)) >> kShift);
        if (kFmt == kNV12) {
          sc[0][lc0 + t] = u;
          sc[0][lc0 + t + 1] = v;
        } else {
          sc[0][lc0 + (t >> 1)] = u;
          sc[1][lc1 + (t >> 1)] = v;
        }
      }
    }
  }
  __syncthreads();
  flush_bytes(yrow, sy[0], npx, t);
  flush_bytes(yrow + W, sy[1], npx, t);
  if (kFmt == kNV12) {
    flush_bytes(c0, sc[0], npx, t);
  } else {
    flush_bytes(c0, sc[0], npx >> 1, t);
    flush_bytes(c1, sc[1], npx >> 1, t);
  }
}

}  // namespace

extern "C" int tg_stream_frame_in(const uint8_t* in_u8, const int32_t* reset, float* lr_curr, float* lr_prev,
                                  float* hr_prev, int n, int c, int h, int w, int s, int bgr, void* stream) {
  return launch_frame_in<kHWC>("stream_frame_in", in_u8, reset, lr_curr, lr_prev, hr_prev, n, c, h, w, s, bgr,
                               (cudaStream_t)stream);
}

extern "C" int tg_stream_frame_in_yuv420(const uint8_t* in, int nv12, const int32_t* reset, float* lr_curr,
                                         float* lr_prev, float* hr_prev, int n, int h, int w, int s, void* stream) {
  return nv12 ? launch_frame_in<kNV12>("stream_frame_in_yuv420", in, reset, lr_curr, lr_prev, hr_prev, n, 3, h, w,
                                       s, 0, (cudaStream_t)stream)
              : launch_frame_in<kI420>("stream_frame_in_yuv420", in, reset, lr_curr, lr_prev, hr_prev, n, 3, h, w,
                                       s, 0, (cudaStream_t)stream);
}

extern "C" int tg_rgb_u8_to_yuv420(const uint8_t* rgb, uint8_t* out, int nv12, int n, int H, int W, void* stream) {
  TG_REQUIRE(rgb && out, TG_E_INVALID, "rgb_u8_to_yuv420: null pointer (rgb / out)");
  TG_REQUIRE(n > 0 && H > 0 && W > 0, TG_E_INVALID, "rgb_u8_to_yuv420: bad size n=%d H=%d W=%d", n, H, W);
  TG_REQUIRE(H % 2 == 0 && W % 2 == 0, TG_E_UNSUPPORTED,
             "rgb_u8_to_yuv420: YUV 4:2:0 needs an even height and width, got %dx%d", H, W);
  const int x_tiles = tg_ceil_div(W, kTilePx);
  const size_t ctas = (size_t)x_tiles * (H / 2) * n;
  TG_REQUIRE(ctas <= 0x7fffffff, TG_E_UNSUPPORTED, "rgb_u8_to_yuv420: grid too large");
  if (nv12)
    tg_launch(rgb_u8_to_yuv420_kernel<kNV12>, dim3((unsigned)ctas), dim3(kThreads), 0, (cudaStream_t)stream, rgb,
              out, H, W, x_tiles);
  else
    tg_launch(rgb_u8_to_yuv420_kernel<kI420>, dim3((unsigned)ctas), dim3(kThreads), 0, (cudaStream_t)stream, rgb,
              out, H, W, x_tiles);
  TG_CUDA_LAUNCH_CHECK("rgb_u8_to_yuv420");
  return TG_OK;
}
