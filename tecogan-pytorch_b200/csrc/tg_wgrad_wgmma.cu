// Weight gradient of a 3x3 convolution / stride-2 transposed convolution as a persistent wgmma
// GEMM whose K dimension is the PIXELS (sm_90a).
//
//   dW[tap][ci][co] = sum over pixels p of  x[p + shift(tap)][ci] * dz[p][co]
//
//   A (M) : activations x, NHWC fp16 -- channels contiguous, i.e. "MN-major" for this GEMM.  One
//           18x10 (conv) / 17x9 (convT) halo box per 16x8 pixel tile by TMA (128B swizzle, zero fill
//           outside the image = the conv's zero padding); the nine taps are nine shifted views of it,
//           addressed through the wgmma descriptor exactly like the forward's HALO mode.  M = 64
//           input channels.
//   B (N) : output gradient dz, NHWC fp16, one 16x8 box per tile (convT: one per output parity,
//           through strided tensor maps), N = 64 output channels, also MN-major.
//   K     : wgmma K = 16 pixels = two 8-pixel tile rows; the 8 pixels of a row are consecutive
//           128-byte smem rows (the swizzle atom), the second row sits one box row further
//           (stride byte offset = box_w * 128).
//   D     : fp32 in registers: three consumer warpgroups own three taps each (3 x 64x64
//           accumulators) for the WHOLE kernel: a CTA walks its share of the pixel tiles and only
//           ever accumulates; there is one epilogue per CTA (fp32 atomics into the gradient in the
//           parameter's own layout, times 1/loss-scale).  Channel counts above 64 are covered by
//           giving every CTA one (ci chunk, co chunk) pair.  The fused bias gradient is a separate
//           reduction over dz (tg_bias_grad_nhwc_f16).
//
// Replaces the weight-gradient half of autograd through nn.Conv2d / nn.ConvTranspose2d
// (tecogan_nets.py:24-65,93-95,112,120-131 under loss.backward(), vsr_model.py:92).
#include <cuda.h>

#include <cstdlib>

#include "tg_common.cuh"
#include "tg_wgmma.cuh"

namespace {

constexpr int kThreads = 512;            // warpgroup 0: TMA producer; warpgroups 1-3: taps 0-2, 3-5, 6-8
constexpr uint32_t kDzTileBytes = TH * TW * 128;   // 16 KB
constexpr int kMaxStages = 6;

struct WParams {
  CUtensorMap map_x;
  CUtensorMap map_dz[4];
  int kind, n, h, w;
  int cin, cout, cin_real, cout_real;
  int tiles_x, tiles_y, num_tiles;
  int ci_chunks, co_chunks, ctas_per_pair;
  int n_stages, n_planes, box_w, box_h;
  uint32_t stage_bytes, x_bytes;
  float* dw;
  const float* scale;        // device [scale, 1/scale] or null
};

// MN-major wgmma shared-memory descriptor, 128B swizzle (cute::GMMA canonical layout
// ((8,m),(8,k)) : ((1,LBO),(8,SBO)) in 16-byte units): 64 contiguous elements along M/N, further
// 64-element chunks LBO bytes apart (unused: M = N = 64); 8 K rows = 8 consecutive 128-byte rows,
// 8-row K groups SBO apart.
__device__ __forceinline__ uint64_t make_sdesc_mn(uint32_t saddr, uint32_t sbo_bytes) {
  return static_cast<uint64_t>(gmma_addr16(saddr)) | (static_cast<uint64_t>(1024u >> 4) << 16) |
         (static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32) | (static_cast<uint64_t>(1) << 62);
}

// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T with both operands MN-major
__device__ __forceinline__ void wgmma_n64_mn(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}

// view offset (in pixels of the halo box) of tap group g
template <int KIND>
__host__ __device__ constexpr int tap_off(int g, int box_w) {
  const TgGroup gr = tg_group(KIND, g);
  return KIND == TG_CONV_3X3 ? (gr.dy + 1) * box_w + (gr.dx + 1) : gr.dy * box_w + gr.dx;
}

template <int KIND>
__global__ void __launch_bounds__(kThreads, 1)
wgrad_wgmma_kernel(const __grid_constant__ WParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const int warp = __shfl_sync(0xFFFFFFFFu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;

  const uint32_t bar_full = base;                       // [kMaxStages]
  const uint32_t bar_empty = base + 8 * kMaxStages;     // [kMaxStages]
  const uint32_t smem_stage0 = base + 1024;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.map_x);
    for (int i = 0; i < p.n_planes; ++i) tma_prefetch_desc(&p.map_dz[i]);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < p.n_stages; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, 12);   // every warp of the three consumer warpgroups
    }
    fence_barrier_init();
  }
  __syncthreads();
  tg_pdl_wait();
  tg_pdl_trigger();

  // this CTA's (ci chunk, co chunk) pair and its share of the pixel tiles
  const int pair = blockIdx.x / p.ctas_per_pair, sub = blockIdx.x - pair * p.ctas_per_pair;
  const int cic = pair / p.co_chunks, coc = pair - cic * p.co_chunks;
  const int per_img = p.tiles_x * p.tiles_y;
  const uint32_t dz_off = (p.x_bytes + 1023u) & ~1023u;

  if (warp == 0) {
    // ============================================================ TMA producer
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = sub; tile < p.num_tiles; tile += p.ctas_per_pair) {
        const int img = tile / per_img, r = tile - img * per_img;
        const int y0 = (r / p.tiles_x) * TH, x0 = (r % p.tiles_x) * TW;
        mbar_wait_mma(bar_empty + 8 * stage, phase ^ 1);
        const uint32_t sa = smem_stage0 + stage * p.stage_bytes;
        mbar_expect_tx(bar_full + 8 * stage, p.x_bytes + (uint32_t)p.n_planes * kDzTileBytes);
        const int org = KIND == TG_CONV_3X3 ? -1 : 0;
        tma_load_4d(sa, &p.map_x, bar_full + 8 * stage, cic * 64, x0 + org, y0 + org, img);
        for (int pl = 0; pl < p.n_planes; ++pl)
          tma_load_4d(sa + dz_off + pl * kDzTileBytes, &p.map_dz[pl], bar_full + 8 * stage, coc * 64, x0, y0, img);
        if (++stage == p.n_stages) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    // ============================================================ consumers: taps 3*cw .. 3*cw+2
    const int cw = (warp - 4) >> 2;
    const int t = threadIdx.x - 128 * (1 + cw);
    const uint32_t box_row = (uint32_t)p.box_w * 128u;
    float acc[3][32];
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[j][i] = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    bool first = true;
    int pend = -1;
    for (int tile = sub; tile < p.num_tiles; tile += p.ctas_per_pair) {
      mbar_wait_mma(bar_full + 8 * stage, phase);
      const uint32_t sa = smem_stage0 + stage * p.stage_bytes;
      const uint32_t sdz = sa + dz_off;
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        const uint32_t xrow = sa + (uint32_t)(2 * ks) * box_row;
        const uint32_t sc = (first && ks == 0) ? 0u : 1u;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          const int g = 3 * cw + j;
          const int o0 = tap_off<KIND>(g, 0), o0w = tap_off<KIND>(g, 1) - o0;   // off = o0 + o0w*box_w
          const uint32_t off0 = (uint32_t)(o0 + o0w * p.box_w) * 128u;
          const int plane = KIND == TG_CONV_3X3 ? 0 : tg_group(KIND, g).acc;
          wgmma_n64_mn(acc[j], make_sdesc_mn(xrow + off0, box_row),
                       make_sdesc_mn(sdz + plane * kDzTileBytes + ks * 2048u, 1024u), sc);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (pend >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * pend);
      }
      pend = stage;
      first = false;
      if (++stage == p.n_stages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (!first) {
      // epilogue: fragment register i of thread t holds (ci row, co column) of the 64x64 accumulator
      const float inv = p.scale ? __ldg(p.scale + 1) : 1.f;
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const TgGroup gr = tg_group(KIND, 3 * cw + j);
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int ci = cic * 64 + 16 * (t >> 5) + ((t & 31) >> 2) + 8 * ((i >> 1) & 1);
          const int co = coc * 64 + 8 * (i >> 2) + 2 * (t & 3) + (i & 1);
          if (ci < p.cin_real && co < p.cout_real) {
            // nn.Conv2d weight [cout,cin,3,3]; nn.ConvTranspose2d weight [cin,cout,3,3]
            const size_t idx = KIND == TG_CONV_3X3 ? (((size_t)co * p.cin_real + ci) * 3 + gr.ky) * 3 + gr.kx
                                                   : (((size_t)ci * p.cout_real + co) * 3 + gr.ky) * 3 + gr.kx;
            atomicAdd(p.dw + idx, acc[j][i] * inv);
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------ CUDA-core cross-check
// One block per (tap, co, 32 ci); threads reduce over pixels.  Bring-up / test kernel only.
template <int KIND>
__global__ void __launch_bounds__(256)
wgrad_simt_kernel(const __half* __restrict__ x, const __half* __restrict__ dz, float* __restrict__ dw,
                  const float* __restrict__ scale, int n, int h, int w, int cin, int cout, int cin_real, int cout_real) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int g = blockIdx.x, co = blockIdx.y, ci = blockIdx.z * 32 + (threadIdx.x & 31);
  const int slice = threadIdx.x >> 5;                      // 8 pixel slices
  const TgGroup gr = tg_group(KIND, g);
  const int OH = KIND == TG_CONV_3X3 ? h : 2 * h, OW = KIND == TG_CONV_3X3 ? w : 2 * w;
  float acc = 0.f;
  const size_t npx = (size_t)n * h * w;
  for (size_t pidx = slice; pidx < npx; pidx += 8) {
    const int xx = (int)(pidx % w), yy = (int)((pidx / w) % h), nn = (int)(pidx / ((size_t)w * h));
    const int iy = yy + gr.dy, ix = xx + gr.dx;
    if (iy < 0 || iy >= h || ix < 0 || ix >= w) continue;
    int oy = yy, ox = xx;
    if (KIND != TG_CONV_3X3) { oy = 2 * yy + (gr.acc >> 1); ox = 2 * xx + (gr.acc & 1); }
    const float xv = ci < cin ? __half2float(x[(((size_t)nn * h + iy) * w + ix) * cin + ci]) : 0.f;
    acc += xv * __half2float(dz[(((size_t)nn * OH + oy) * OW + ox) * cout + co]);
  }
  __shared__ float red[8][33];
  red[slice][threadIdx.x & 31] = acc;
  __syncthreads();
  if (slice == 0 && ci < cin_real && co < cout_real) {
    float s = 0.f;
    for (int k = 0; k < 8; ++k) s += red[k][threadIdx.x & 31];
    const float inv = scale ? __ldg(scale + 1) : 1.f;
    const size_t idx = KIND == TG_CONV_3X3 ? (((size_t)co * cin_real + ci) * 3 + gr.ky) * 3 + gr.kx
                                           : (((size_t)ci * cout_real + co) * 3 + gr.ky) * 3 + gr.kx;
    atomicAdd(dw + idx, s * inv);
  }
}

int wgrad_validate(const tg_wgrad_desc* d, const char* who) {
  TG_REQUIRE(d != nullptr, TG_E_INVALID, "%s: null descriptor", who);
  TG_REQUIRE(d->x && d->dz && d->dw, TG_E_INVALID, "%s: null pointer", who);
  TG_REQUIRE(d->n > 0 && d->h > 0 && d->w > 0, TG_E_INVALID, "%s: bad size", who);
  TG_REQUIRE(d->kind == TG_CONV_3X3 || d->kind == TG_CONVT_3X3_S2, TG_E_INVALID, "%s: kind", who);
  TG_REQUIRE(d->cin == 64 || d->cin == 128 || d->cin == 256, TG_E_UNSUPPORTED, "%s: cin=%d", who, d->cin);
  TG_REQUIRE(d->cout == 64 || d->cout == 128 || d->cout == 256, TG_E_UNSUPPORTED, "%s: cout=%d", who, d->cout);
  TG_REQUIRE(d->cin_real >= 1 && d->cin_real <= d->cin && d->cout_real >= 1 && d->cout_real <= d->cout, TG_E_INVALID,
             "%s: real channel counts", who);
  TG_REQUIRE(d->reserved == 0, TG_E_INVALID, "%s: reserved must be 0", who);
  return TG_OK;
}

}  // namespace

extern "C" {

int tg_wgrad_tcgen05(const tg_wgrad_desc* d, void* stream) {
  int rc = wgrad_validate(d, "wgrad");
  if (rc != TG_OK) return rc;
  TG_REQUIRE(((uintptr_t)d->x & 15) == 0 && ((uintptr_t)d->dz & 15) == 0, TG_E_INVALID,
             "wgrad: pointers must be 16-byte aligned");
  WParams p;
  p.kind = d->kind; p.n = d->n; p.h = d->h; p.w = d->w;
  p.cin = d->cin; p.cout = d->cout; p.cin_real = d->cin_real; p.cout_real = d->cout_real;
  p.tiles_x = tg_ceil_div(d->w, TW);
  p.tiles_y = tg_ceil_div(d->h, TH);
  p.num_tiles = p.tiles_x * p.tiles_y * d->n;
  p.ci_chunks = d->cin / 64;
  p.co_chunks = d->cout / 64;
  p.dw = d->dw;
  p.scale = d->scale;
  const bool conv = d->kind == TG_CONV_3X3;
  TG_REQUIRE(!(d->db && !conv), TG_E_UNSUPPORTED, "wgrad: fused bias gradient is for conv3x3 layers");
  p.box_w = conv ? TW + 2 : TW + 1;
  p.box_h = conv ? TH + 2 : TH + 1;
  p.n_planes = conv ? 1 : 4;
  p.x_bytes = (uint32_t)p.box_w * p.box_h * 128u;
  p.stage_bytes = ((p.x_bytes + 1023u) & ~1023u) + (uint32_t)p.n_planes * kDzTileBytes;
  int stages = (int)((kSmemLimit - 2048u) / p.stage_bytes);
  if (stages > kMaxStages) stages = kMaxStages;
  TG_REQUIRE(stages >= 2, TG_E_UNSUPPORTED, "wgrad: shared memory budget");
  p.n_stages = stages;

  rc = encode_nhwc(&p.map_x, d->x, d->cin, d->w, d->h, d->n, (size_t)d->cin, (size_t)d->w * d->cin,
                   (size_t)d->h * d->w * d->cin, 64, p.box_w, p.box_h);
  if (rc != TG_OK) return rc;
  if (conv) {
    rc = encode_nhwc(&p.map_dz[0], d->dz, d->cout, d->w, d->h, d->n, (size_t)d->cout, (size_t)d->w * d->cout,
                     (size_t)d->h * d->w * d->cout, 64, TW, TH);
    if (rc != TG_OK) return rc;
    for (int i = 1; i < 4; ++i) p.map_dz[i] = p.map_dz[0];
  } else {
    // dz [n,2h,2w,cout]: parity plane (py,px) = pixels (2y+py, 2x+px)
    const size_t W2 = (size_t)2 * d->w, C = (size_t)d->cout;
    for (int pl = 0; pl < 4; ++pl) {
      const __half* base = reinterpret_cast<const __half*>(d->dz) + ((size_t)(pl >> 1) * W2 + (pl & 1)) * C;
      rc = encode_nhwc(&p.map_dz[pl], base, d->cout, d->w, d->h, d->n, 2 * C, 2 * W2 * C,
                       (size_t)4 * d->h * d->w * C, 64, TW, TH);
      if (rc != TG_OK) return rc;
    }
  }

  static TgPerDeviceOnce attr_once;
  const cudaError_t attr_err = attr_once.run([] {
    cudaError_t e = cudaFuncSetAttribute(wgrad_wgmma_kernel<TG_CONV_3X3>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)kSmemLimit);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(wgrad_wgmma_kernel<TG_CONVT_3X3_S2>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)kSmemLimit);
  });
  TG_REQUIRE(attr_err == cudaSuccess, (int)attr_err, "wgrad: cudaFuncSetAttribute: %s",
             cudaGetErrorString(attr_err));
  int sms = 0;
  rc = tg_device_sm_count(&sms);
  if (rc != TG_OK) return rc;
  const int pairs = p.ci_chunks * p.co_chunks;
  int budget = d->max_ctas > 0 && d->max_ctas < sms ? d->max_ctas : sms;
  if (budget < pairs) budget = pairs;
  p.ctas_per_pair = budget / pairs;
  if (p.ctas_per_pair > p.num_tiles) p.ctas_per_pair = p.num_tiles;
  const int grid = p.ctas_per_pair * pairs;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t lerr = conv ? tg_launch(wgrad_wgmma_kernel<TG_CONV_3X3>, dim3(grid), dim3(kThreads), kSmemLimit, st, p)
                          : tg_launch(wgrad_wgmma_kernel<TG_CONVT_3X3_S2>, dim3(grid), dim3(kThreads), kSmemLimit, st, p);
  TG_REQUIRE(lerr == cudaSuccess, (int)lerr, "wgrad: launch failed: %s", cudaGetErrorString(lerr));
  TG_CUDA_LAUNCH_CHECK("wgrad");
  if (d->db != nullptr)
    return tg_bias_grad_nhwc_f16(d->dz, (size_t)d->n * d->h * d->w, d->cout, d->cout_real, d->scale, d->db, stream);
  return TG_OK;
}

int tg_wgrad_simt(const tg_wgrad_desc* d, void* stream) {
  int rc = wgrad_validate(d, "wgrad_simt");
  if (rc != TG_OK) return rc;
  dim3 grid(9, d->cout, d->cin / 32);
  cudaStream_t st = (cudaStream_t)stream;
  const __half* x = reinterpret_cast<const __half*>(d->x);
  const __half* dz = reinterpret_cast<const __half*>(d->dz);
  if (d->kind == TG_CONV_3X3)
    tg_launch(wgrad_simt_kernel<TG_CONV_3X3>, grid, dim3(256), 0, st, x, dz, d->dw, d->scale, d->n, d->h, d->w, d->cin,
              d->cout, d->cin_real, d->cout_real);
  else
    tg_launch(wgrad_simt_kernel<TG_CONVT_3X3_S2>, grid, dim3(256), 0, st, x, dz, d->dw, d->scale, d->n, d->h, d->w,
              d->cin, d->cout, d->cin_real, d->cout_real);
  TG_CUDA_LAUNCH_CHECK("wgrad_simt");
  return TG_OK;
}

}  // extern "C"
