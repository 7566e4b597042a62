// Frame input of one streamed inference step: uint8 HWC frames decoded on the device into the step's fp32
// NCHW lr_curr, and the per-slot reset of the recurrent state.  Contract: include/tecogan_b200.h
// (tg_stream_frame_in).
#include "tg_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kTilePx = 256;            // decode CTA: kTilePx pixels of one image row, one per thread
constexpr int kMaxC = 4;

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

// blockIdx.x < decode_ctas: decode CTA (x tile, row, image), row-major over x tiles;
// the rest: zpc CTAs per slot, each zeroing a strided share of that slot's lr_prev and hr_prev when flagged.
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
    // HWC bytes of up to kTilePx pixels, placed so that sb[lead + j] = src[j] with lead = src % 16: the
    // 16-byte-aligned interior of the source lands on 16-byte-aligned shared memory
    __shared__ __align__(16) uint8_t sb[kTilePx * kMaxC + 32];
    const int xt = b % x_tiles, r = b / x_tiles;
    const int y = r % h, img = r / h;
    const int x0 = xt * kTilePx;
    const int npx = min(kTilePx, w - x0);
    const int bytes = npx * c;
    const uint8_t* src = in + (((size_t)img * h + y) * w + x0) * c;
    const int lead = (int)((uintptr_t)src & 15u);
    const int a0 = min(lead ? 16 - lead : 0, bytes);   // bytes before the first aligned 16-byte vector
    const int nv = (bytes - a0) / 16;
    const int tail0 = a0 + 16 * nv;
    for (int i = t; i < nv; i += kThreads)
      *reinterpret_cast<uint4*>(sb + lead + a0 + 16 * i) = __ldg(reinterpret_cast<const uint4*>(src + a0) + i);
    if (t < a0) sb[lead + t] = __ldg(src + t);
    if (tail0 + t < bytes) sb[lead + tail0 + t] = __ldg(src + tail0 + t);
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

}  // namespace

extern "C" int tg_stream_frame_in(const uint8_t* in_u8, const int32_t* reset, float* lr_curr, float* lr_prev,
                                  float* hr_prev, int n, int c, int h, int w, int s, int bgr, void* stream) {
  TG_REQUIRE(in_u8 || reset, TG_E_INVALID, "stream_frame_in: in_u8 and reset are both NULL");
  TG_REQUIRE(lr_curr && lr_prev && hr_prev, TG_E_INVALID, "stream_frame_in: null pointer (lr_curr / lr_prev / hr_prev)");
  TG_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0, TG_E_INVALID, "stream_frame_in: bad size n=%d c=%d h=%d w=%d", n, c,
             h, w);
  TG_REQUIRE(c <= kMaxC, TG_E_UNSUPPORTED, "stream_frame_in: %d channels (at most %d)", c, kMaxC);
  TG_REQUIRE(s == 2 || s == 4, TG_E_UNSUPPORTED, "stream_frame_in: scale %d (2 or 4)", s);
  TG_REQUIRE((((uintptr_t)lr_curr | (uintptr_t)lr_prev | (uintptr_t)hr_prev) & 3u) == 0, TG_E_INVALID,
             "stream_frame_in: fp32 buffers must be 4-byte aligned");
  const int x_tiles = tg_ceil_div(w, kTilePx);
  const size_t decode = in_u8 ? (size_t)x_tiles * h * n : 0;
  const size_t hr4 = (size_t)c * s * h * s * w / 4;
  const int zpc = reset ? (int)(hr4 / (kThreads * 8) + 1 < 64 ? hr4 / (kThreads * 8) + 1 : 64) : 0;
  const size_t ctas = decode + (size_t)zpc * n;
  TG_REQUIRE(ctas <= 0x7fffffff, TG_E_UNSUPPORTED, "stream_frame_in: grid too large");
  tg_launch(stream_frame_in_kernel, dim3((unsigned)ctas), dim3(kThreads), 0, (cudaStream_t)stream, in_u8, reset,
            lr_curr, lr_prev, hr_prev, c, h, w, s, bgr, x_tiles, (int)decode, zpc);
  TG_CUDA_LAUNCH_CHECK("stream_frame_in");
  return TG_OK;
}
