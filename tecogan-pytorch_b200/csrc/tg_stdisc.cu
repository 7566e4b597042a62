// Input builder of the spatio-temporal discriminator (SURVEY.md 8-f3): replaces the tensor plumbing of
// SpatioTemporalDiscriminator.forward_sequence, codes/models/networks/tecogan_nets.py:438-463 --
// three backward_warps per 3-frame clip, the centre crop + zero pad of the warped frames, the
// "rrrgggbbb" permutes and the 27-channel concat -- by ONE bandwidth-bound kernel (and one for its
// gradient w.r.t. the frames; the flows are detached by the reference at :431, bi_data carries no grad).
//
//   out[clip, 0 + c*3 + f]  = data[n, 3k+f, c]                      (original frames)
//   out[clip, 9 + c*3 + f]  = crop_pad(backward_warp(data[n, 3k+f], flow[clip*3 + f]))[c]
//   out[clip, 18 + c*3 + f] = bi[n, 3k+f, c]                        (bicubic-upsampled LR, the condition)
// with clip = n*(t/3) + k, f = 0..2, c = 0..C-1 (C*3 channels per part; C = 3 -> 27).
#include "tg_common.cuh"

namespace {

inline int sgrid(size_t total, int block) {
  size_t g = (total + block - 1) / block;
  const size_t cap = (size_t)tg_sms() * 32;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

struct StCorners { int xa, ya; float ax, ay; };
__device__ __forceinline__ StCorners st_corners(float fx, float fy, int H, int W) {
  StCorners c;
  fx = fminf(fmaxf(fx, 0.f), (float)(W - 1));
  fy = fminf(fmaxf(fy, 0.f), (float)(H - 1));
  c.xa = min((int)floorf(fx), W - 2);
  c.ya = min((int)floorf(fy), H - 2);
  c.ax = fx - (float)c.xa;
  c.ay = fy - (float)c.ya;
  return c;
}

// one thread = one pixel of one frame of one clip
__global__ void st_input_kernel(const float* __restrict__ data, const float* __restrict__ bi,
                                const float* __restrict__ flow, float* __restrict__ out, int n, int t_full, int t,
                                int C, int H, int W, int pad, int csize) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const size_t HW = (size_t)H * W;
  const int clips_per_n = t / 3;
  const size_t total = (size_t)n * clips_per_n * 3 * HW;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t sp = i % HW;
    size_t r = i / HW;
    const int f = (int)(r % 3); r /= 3;
    const int k = (int)(r % clips_per_n);
    const int nn = (int)(r / clips_per_n);
    const int y = (int)(sp / W), x = (int)(sp % W);
    const size_t clip = (size_t)nn * clips_per_n + k;
    const size_t frame = (size_t)nn * t_full + 3 * k + f;          // index into [n, t_full]
    const float* dfr = data + frame * C * HW;
    const float* bfr = bi + frame * C * HW;
    float* o = out + clip * (size_t)(9 * C) * HW + sp;
    const bool inside = y >= pad && y < pad + csize && x >= pad && x < pad + csize;
    StCorners cc = {0, 0, 0.f, 0.f};
    if (inside) {
      const float* fl = flow + (clip * 3 + f) * 2 * HW;
      cc = st_corners((float)x + __ldg(fl + sp), (float)y + __ldg(fl + HW + sp), H, W);
    }
    for (int c = 0; c < C; ++c) {
      const float* pl = dfr + (size_t)c * HW;
      o[(size_t)(c * 3 + f) * HW] = __ldg(pl + sp);
      float wv = 0.f;
      if (inside) {
        const float* q = pl + (size_t)cc.ya * W + cc.xa;
        const float v00 = __ldg(q), v01 = __ldg(q + 1), v10 = __ldg(q + W), v11 = __ldg(q + W + 1);
        wv = v00 * (1.f - cc.ax) * (1.f - cc.ay) + v01 * cc.ax * (1.f - cc.ay) + v10 * (1.f - cc.ax) * cc.ay +
             v11 * cc.ax * cc.ay;
      }
      o[(size_t)(3 * C + c * 3 + f) * HW] = wv;
      o[(size_t)(6 * C + c * 3 + f) * HW] = __ldg(bfr + (size_t)c * HW + sp);
    }
  }
}

// gradient w.r.t. data (fp32 atomics into a zeroed [n,t_full,C,H,W] buffer)
__global__ void st_input_bwd_kernel(const float* __restrict__ gout, const float* __restrict__ flow,
                                    float* __restrict__ gdata, int n, int t_full, int t, int C, int H, int W, int pad,
                                    int csize) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const size_t HW = (size_t)H * W;
  const int clips_per_n = t / 3;
  const size_t total = (size_t)n * clips_per_n * 3 * HW;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t sp = i % HW;
    size_t r = i / HW;
    const int f = (int)(r % 3); r /= 3;
    const int k = (int)(r % clips_per_n);
    const int nn = (int)(r / clips_per_n);
    const int y = (int)(sp / W), x = (int)(sp % W);
    const size_t clip = (size_t)nn * clips_per_n + k;
    const size_t frame = (size_t)nn * t_full + 3 * k + f;
    float* gfr = gdata + frame * C * HW;
    const float* g = gout + clip * (size_t)(9 * C) * HW + sp;
    const bool inside = y >= pad && y < pad + csize && x >= pad && x < pad + csize;
    StCorners cc = {0, 0, 0.f, 0.f};
    if (inside) {
      const float* fl = flow + (clip * 3 + f) * 2 * HW;
      cc = st_corners((float)x + __ldg(fl + sp), (float)y + __ldg(fl + HW + sp), H, W);
    }
    for (int c = 0; c < C; ++c) {
      float* pl = gfr + (size_t)c * HW;
      atomicAdd(pl + sp, __ldg(g + (size_t)(c * 3 + f) * HW));
      if (inside) {
        const float gw = __ldg(g + (size_t)(3 * C + c * 3 + f) * HW);
        float* q = pl + (size_t)cc.ya * W + cc.xa;
        const float w00 = (1.f - cc.ax) * (1.f - cc.ay), w01 = cc.ax * (1.f - cc.ay);
        const float w10 = (1.f - cc.ax) * cc.ay, w11 = cc.ax * cc.ay;
        if (gw != 0.f) {
          if (w00 != 0.f) atomicAdd(q, gw * w00);
          if (w01 != 0.f) atomicAdd(q + 1, gw * w01);
          if (w10 != 0.f) atomicAdd(q + W, gw * w10);
          if (w11 != 0.f) atomicAdd(q + W + 1, gw * w11);
        }
      }
    }
  }
}

}  // namespace

extern "C" {

static int st_check(const char* who, const void* a, const void* b, const void* c, int n, int t_full, int t, int ch, int h,
                    int w, int pad, int csize) {
  TG_REQUIRE(a && b && c, TG_E_INVALID, "%s: null pointer", who);
  TG_REQUIRE(n > 0 && ch > 0 && h >= 2 && w >= 2 && t >= 3 && t % 3 == 0 && t <= t_full, TG_E_INVALID,
             "%s: bad shape n=%d t=%d/%d c=%d h=%d w=%d", who, n, t, t_full, ch, h, w);
  TG_REQUIRE(pad >= 0 && csize >= 0 && pad + csize <= h && pad + csize <= w, TG_E_INVALID, "%s: bad crop %d+%d", who,
             pad, csize);
  return TG_OK;
}

int tg_st_disc_input_nchw_f32(const float* data, const float* bi, const float* flow, float* out, int n, int t_full,
                              int t, int c, int h, int w, int pad, int csize, void* stream) {
  int rc = st_check("st_disc_input", data, bi, flow, n, t_full, t, c, h, w, pad, csize);
  if (rc != TG_OK) return rc;
  TG_REQUIRE(out != nullptr, TG_E_INVALID, "st_disc_input: null output");
  const size_t total = (size_t)n * t * h * w;
  tg_launch(st_input_kernel, dim3(sgrid(total, 256)), dim3(256), 0, (cudaStream_t)stream, data, bi, flow, out, n, t_full,
            t, c, h, w, pad, csize);
  TG_CUDA_LAUNCH_CHECK("st_disc_input");
  return TG_OK;
}

int tg_st_disc_input_bwd_nchw_f32(const float* gout, const float* flow, float* gdata, int n, int t_full, int t, int c,
                                  int h, int w, int pad, int csize, void* stream) {
  int rc = st_check("st_disc_input_bwd", gout, flow, gdata, n, t_full, t, c, h, w, pad, csize);
  if (rc != TG_OK) return rc;
  const size_t total = (size_t)n * t * h * w;
  tg_launch(st_input_bwd_kernel, dim3(sgrid(total, 256)), dim3(256), 0, (cudaStream_t)stream, gout, flow, gdata, n,
            t_full, t, c, h, w, pad, csize);
  TG_CUDA_LAUNCH_CHECK("st_disc_input_bwd");
  return TG_OK;
}

}  // extern "C"
