// Shared host/device helpers for libtecogan_b200 (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#include "../../include/tecogan_b200.h"

// ---------------------------------------------------------------- error plumbing
void tg_set_error(const char* fmt, ...);

#define TG_REQUIRE(cond, code, ...)            \
  do {                                         \
    if (!(cond)) {                             \
      tg_set_error(__VA_ARGS__);               \
      return (code);                           \
    }                                          \
  } while (0)

#define TG_CUDA_LAUNCH_CHECK(name)                                         \
  do {                                                                     \
    cudaError_t e__ = cudaGetLastError();                                  \
    if (e__ != cudaSuccess) {                                              \
      tg_set_error("%s: launch failed: %s", name, cudaGetErrorString(e__)); \
      return (int)e__;                                                     \
    }                                                                      \
  } while (0)

static inline int tg_ceil_div(int a, int b) { return (a + b - 1) / b; }
// SMs of the current device, for grid caps (1 if the query fails: a small grid is still correct)
static inline int tg_sms() {
  int s = 0;
  return tg_device_sm_count(&s) == TG_OK && s > 0 ? s : 1;
}

// ---------------------------------------------------------------- programmatic dependent launch
// Every kernel of the library is launched with cudaLaunchAttributeProgrammaticStreamSerialization
// and begins with tg_pdl_wait(): the next kernel of the stream (or captured graph) is scheduled onto
// SMs as the previous one drains and runs its prologue (barrier init, TMEM allocation, weight
// loads) before blocking on the predecessor's completion -- launch latency and tail imbalance of
// the ~48 dependent launches of a step overlap instead of adding up.  TECOGAN_B200_PDL=0 disables.
bool tg_pdl_enabled();
#ifdef __CUDACC__
__device__ __forceinline__ void tg_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void tg_pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename... KArgs, typename... Args>
static inline cudaError_t tg_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                    cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = tg_pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// tg_launch with a 1-D thread-block cluster of `cluster_x` CTAs (gridDim.x must be a multiple of it)
template <typename... KArgs, typename... Args>
static inline cudaError_t tg_launch_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                            cudaStream_t stream, int cluster_x, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)cluster_x;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = tg_pdl_enabled() ? 2 : 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// Cooperative launch: the driver schedules the grid only when EVERY CTA can be resident at once
// (or fails the launch) -- required by kernels whose CTAs wait on each other (conv_chain_kernel).
// Not combined with programmatic dependent launch: such a kernel starts after its predecessor.
template <typename... KArgs, typename... Args>
static inline cudaError_t tg_launch_cooperative(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                                cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#endif

// cudaFuncSetAttribute is per DEVICE: run `fn` once for every device this process launches on.
struct TgPerDeviceOnce {
  int done[64] = {};
  cudaError_t err[64] = {};
  template <typename F>
  cudaError_t run(F fn) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return fn();
    if (!done[dev]) { err[dev] = fn(); done[dev] = 1; }
    return err[dev];
  }
};

// ---------------------------------------------------------------- packed-weight geometry
// One weight tile = [cout_pad rows][64 k] fp16, 128-byte rows, 128B swizzle:
// byte offset of (row n, k) = n*128 + (((k>>3) ^ (n&7))<<4) + (k&7)*2.
__host__ __device__ static inline uint32_t tg_wtile_off(uint32_t n, uint32_t k) {
  return n * 128u + ((((k >> 3) ^ (n & 7u)) << 4) | ((k & 7u) << 1));
}

// conv3x3: group g = ky*3+kx reads input pixel (y+ky-1, x+kx-1).
// convT 3x3 s2 p1 op1 (SURVEY.md 8-a7): 9 groups ordered by output parity acc = py*2+px:
//   acc0: in[y,x]*Wt[1,1]
//   acc1: in[y,x]*Wt[1,2] + in[y,x+1]*Wt[1,0]
//   acc2: in[y,x]*Wt[2,1] + in[y+1,x]*Wt[0,1]
//   acc3: in[y,x]*Wt[2,2] + in[y,x+1]*Wt[2,0] + in[y+1,x]*Wt[0,2] + in[y+1,x+1]*Wt[0,0]
// conv 3x3 s2 p1 (TG_CONV_3X3_S2, the convT's data gradient): group g = ky*3+kx reads input pixel
//   (2y+ky-1, 2x+kx-1) = pixel (y+dy, x+dx) of the input's PARITY PLANE (py,px) [plane (py,px) holds the
//   pixels (2i+py, 2j+px)]:  k=0 -> parity 1, offset -1;  k=1 -> parity 0, offset 0;  k=2 -> parity 1, offset 0.
struct TgGroup { int acc, dy, dx, ky, kx; };
__host__ __device__ constexpr int tg_s2_par(int k) { return k == 1 ? 0 : 1; }
__host__ __device__ constexpr int tg_s2_off(int k) { return k == 0 ? -1 : 0; }
// parity plane (py*2+px) that group g of a TG_CONV_3X3_S2 layer reads
__host__ __device__ constexpr int tg_s2_plane(int g) { return tg_s2_par(g / 3) * 2 + tg_s2_par(g % 3); }
__host__ __device__ constexpr TgGroup tg_group(int kind, int g) {
  if (kind == TG_CONV_3X3) return TgGroup{0, g / 3 - 1, g % 3 - 1, g / 3, g % 3};
  if (kind == TG_CONV_3X3_S2) return TgGroup{0, tg_s2_off(g / 3), tg_s2_off(g % 3), g / 3, g % 3};
  switch (g) {
    case 0: return TgGroup{0, 0, 0, 1, 1};
    case 1: return TgGroup{1, 0, 0, 1, 2};
    case 2: return TgGroup{1, 0, 1, 1, 0};
    case 3: return TgGroup{2, 0, 0, 2, 1};
    case 4: return TgGroup{2, 1, 0, 0, 1};
    case 5: return TgGroup{3, 0, 0, 2, 2};
    case 6: return TgGroup{3, 0, 1, 2, 0};
    case 7: return TgGroup{3, 1, 0, 0, 2};
    default: return TgGroup{3, 1, 1, 0, 0};
  }
}

// ---------------------------------------------------------------- sampling helpers (device)
#ifdef __CUDACC__
// BicubicUpsampler taps (net_utils.py:116-131), a=-0.75, t = d/scale. Exact in fp32.
__device__ __forceinline__ void tg_cubic_taps(int d, int s, float k[4]) {
  const float a = -0.75f;
  const float t = (float)d / (float)s, t2 = t * t, t3 = t2 * t;
  k[0] = a * t - 2.f * a * t2 + a * t3;
  k[1] = 1.f - (a + 3.f) * t2 + (a + 2.f) * t3;
  k[2] = -a * t + (2.f * a + 3.f) * t2 - (a + 2.f) * t3;
  k[3] = a * t2 - a * t3;
}

// upsample_func as a separable 4-tap filter over source indices clamp(i-1 .. i+2) (replicate):
//   bicubic : BicubicUpsampler kernels[d]                           (net_utils.py:116-131)
//   bilinear: F.interpolate(align_corners=False): src = max((s*i+d+0.5)/s-0.5, 0) falls between
//             i-1,i (d < s/2) or i,i+1 (d >= s/2) with fraction f; clamping the INDEX is
//             equivalent to clamping src at 0 / L-1 (both taps hit the same border sample).
__device__ __forceinline__ void tg_up_taps(int up_mode, int d, int s, float k[4]) {
  if (up_mode == TG_UP_BICUBIC) { tg_cubic_taps(d, s, k); return; }
  const float src = ((float)d + 0.5f) / (float)s - 0.5f;      // in (-0.5, 0.5)
  k[0] = k[1] = k[2] = k[3] = 0.f;
  if (src < 0.f) { const float f = src + 1.f; k[0] = 1.f - f; k[1] = f; }
  else           { k[1] = 1.f - src; k[2] = src; }
}

// reflect index of F.pad(...,'reflect') on the bottom/right only: i in [0, L) over a source of
// length Ls <= L: i >= Ls -> 2*Ls-2-i   (tecogan_nets.py:239-241)
__device__ __forceinline__ int tg_reflect_hi(int i, int Ls) { return i < Ls ? i : 2 * Ls - 2 - i; }

__device__ __forceinline__ int tg_clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// upsample_func evaluated at HR position (Y,X) of one plane of a (reflect-padded) LR image.
// src: plane [hs][ws]; logical padded size (h,w); bicubic = BicubicUpsampler (no half-pixel
// shift, replicate pad (1,2)); bilinear = F.interpolate(align_corners=False).
__device__ __forceinline__ float tg_upsample_at(const float* __restrict__ src, int hs, int ws,
                                                int h, int w, int s, int up_mode, int Y, int X) {
  if (up_mode == TG_UP_BICUBIC) {
    const int y = Y / s, dy = Y - y * s, x = X / s, dx = X - x * s;
    float ky[4], kx[4];
    tg_cubic_taps(dy, s, ky);
    tg_cubic_taps(dx, s, kx);
    float acc = 0.f;
    // vertical pass first then horizontal (net_utils.py:144-151); separable so order only
    // affects fp32 rounding.
    float col[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int xx = tg_reflect_hi(tg_clampi(x - 1 + j, 0, w - 1), ws);
      float v = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int yy = tg_reflect_hi(tg_clampi(y - 1 + i, 0, h - 1), hs);
        v += ky[i] * __ldg(src + (size_t)yy * ws + xx);
      }
      col[j] = v;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) acc += kx[j] * col[j];
    return acc;
  } else {
    const float fs = (float)s;
    float sy = fmaxf(((float)Y + 0.5f) / fs - 0.5f, 0.f);
    float sx = fmaxf(((float)X + 0.5f) / fs - 0.5f, 0.f);
    int y0 = min((int)floorf(sy), h - 1), x0 = min((int)floorf(sx), w - 1);
    int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
    const float fy = sy - (float)y0, fx = sx - (float)x0;
    y0 = tg_reflect_hi(y0, hs); y1 = tg_reflect_hi(y1, hs);
    x0 = tg_reflect_hi(x0, ws); x1 = tg_reflect_hi(x1, ws);
    const float v00 = __ldg(src + (size_t)y0 * ws + x0), v01 = __ldg(src + (size_t)y0 * ws + x1);
    const float v10 = __ldg(src + (size_t)y1 * ws + x0), v11 = __ldg(src + (size_t)y1 * ws + x1);
    const float top = v00 * (1.f - fx) + v01 * fx;
    const float bot = v10 * (1.f - fx) + v11 * fx;
    return top * (1.f - fy) + bot * fy;
  }
}

// branch-free: act(v) = max(v, slope*v) with slope 1 (none) / 0 (ReLU) / 0.2 (LeakyReLU); `act` is
// warp-uniform, so the slope selection hoists out of the per-element epilogue loops
__device__ __forceinline__ float tg_act_slope(int act) {
  return act == TG_ACT_NONE ? 1.f : (act == TG_ACT_RELU ? 0.f : 0.2f);
}
__device__ __forceinline__ float tg_act(float v, int act) { return fmaxf(v, v * tg_act_slope(act)); }
// data-gradient epilogues: derivative of ReLU / LeakyReLU(0.2) taken from the stored forward OUTPUT m
__device__ __forceinline__ float tg_dact(float m, int act) {
  return m > 0.f ? 1.f : (act == TG_ACT_DRELU ? 0.f : 0.2f);
}
#endif  // __CUDACC__
