// Two fused parts of SRNet on sm_90a (H100), built from the same TMA / mbarrier / wgmma pieces as
// tg_conv_wgmma.cu:
//
// conv_chain_kernel -- SRNet conv_in + the residual blocks (64->64 3x3 convs) as ONE persistent
//   cooperative launch.  Every CTA walks all layers over its fixed set of 16x8 tiles (halo mode: one
//   18x10 TMA box per tile, the nine taps are shifted wgmma descriptor views of it).  A tile of layer l
//   is loaded as soon as the (up to 9) tiles of layer l-1 under its halo have been published: per-tile
//   progress flags in the caller's workspace, stamped with a launch epoch so the workspace is zeroed only
//   once.  There is no launch, pipeline fill / drain or grid-wide barrier between layers; a layer's
//   weights are reloaded into shared memory as soon as both consumers are done with the previous ones.
//
// convT_convout_kernel -- SRNet tail: last ConvTranspose2d(64,64,3,2,1,op=1) + ReLU -> conv_out 3x3
//   (64 -> out_nc <= 3) -> + upsample_func(lr_curr) or + the pre-written frame -> fp32 NCHW (+ uint8 NHWC).
//   Per 16x8 tile of the transposed conv's input (17x9 halo box), parity by parity: the transposed conv
//   runs pixels-on-N (M = 64 couts, N = the 128 input pixels, one m64n128k16 per (tap group, k-step));
//   its accumulators are written, +bias, ReLU, fp16, by stmatrix into one 128-pixel K-major 128B-swizzled
//   operand block (pixels outside the image are zero = conv_out's zero padding); conv_out runs as
//   "tap-major N" wgmmas (N = 48 = 9 taps x 4 couts) on that block; each thread adds the fp32 tap
//   products that land on its 4 output pixels into registers.  The tile's 30x14 interior HR pixels are
//   outputs (tiles advance by 15x7 input pixels, the transposed conv is recomputed on a one-pixel ring).
//   Warpgroup 0 runs the transposed conv with two accumulator sets, so parity a + 1's MMAs are in flight
//   under parity a's epilogue; warpgroups 1 and 2 run conv_out, the summation and the global I/O of
//   alternate tiles, each fed through its own two operand blocks.  The 64-channel HR map never reaches HBM.
#include <cuda.h>

#include <mutex>

#include "tg_common.cuh"
#include "tg_wgmma.cuh"

namespace {

constexpr int TH = 16, TW = 8;
constexpr uint32_t kSmemLimit = 232448;
constexpr uint32_t kWtBytes = 9 * 64 * 128;          // nine [64 cout][64 cin] fp16 weight tiles
constexpr uint32_t kFlagBase = 32;                   // workspace words: [0] epoch, [1] done count, [32..] tile flags
constexpr uint32_t kEpochStride = 32;                // flag value = epoch * 32 + layer + 1 (<= 24 layers)

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}
// NHWC fp16 [n][h][w][64] with a (box_w x box_h) pixel box of all 64 channels, 128B swizzle
int encode_c64(CUtensorMap* m, const void* ptr, int n, int h, int w, int box_w, int box_h) {
  EncodeTiledFn fn = encode_fn();
  TG_REQUIRE(fn != nullptr, TG_E_DRIVER, "cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t dims[4] = {64, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
  cuuint64_t strides[3] = {128, (cuuint64_t)w * 128, (cuuint64_t)h * w * 128};
  cuuint32_t box[4] = {64, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  TG_REQUIRE(r == CUDA_SUCCESS, TG_E_DRIVER, "cuTensorMapEncodeTiled failed (%d) n=%d h=%d w=%d", (int)r, n, h, w);
  return TG_OK;
}

__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
// plain (L1-coherent within the SM) 16-byte load: chain residuals were written earlier in the same launch
__device__ __forceinline__ uint4 ld_global_u4(const void* p) {
  uint4 v;
  asm volatile("ld.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}

// halo-mode conv taps of one 16x8 tile (18x10 box, origin -1): acc[h] (+)= A view(tap) x W[tap], tile rows 8h..8h+7
__device__ __forceinline__ void halo_mmas(float (&acc)[2][32], uint32_t sa16, uint32_t w16) {
  constexpr int kBoxW = TW + 2;
  const uint64_t a_hi = gmma_desc_hi((uint32_t)kBoxW * 128u), b_hi = gmma_desc_hi(1024u);
  constexpr uint32_t half16 = (8u * kBoxW * 128u) >> 4;
#pragma unroll
  for (int g = 0; g < 9; ++g) {
    const TgGroup gr = tg_group(TG_CONV_3X3, g);
    const uint32_t a16 = sa16 + (uint32_t)((gr.dy + 1) * kBoxW + (gr.dx + 1)) * 8u;
    const uint32_t b16 = w16 + (uint32_t)g * (kWtBytes / 9 / 16);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t sc = (g == 0 && k == 0) ? 0u : 1u;
      wgmma_n64(acc[0], a_hi | (uint64_t)(a16 + 2u * k), b_hi | (uint64_t)(b16 + 2u * k), sc);
      wgmma_n64(acc[1], a_hi | (uint64_t)(a16 + half16 + 2u * k), b_hi | (uint64_t)(b16 + 2u * k), sc);
    }
  }
}

// ================================================================== conv chain
constexpr int kChainThreads = 384;                   // producer warpgroup + 2 consumer warpgroups
constexpr uint32_t kChainHalo = (TW + 2) * (TH + 2) * 128;           // 23040
constexpr uint32_t kChainStage = (kChainHalo + 1023u) & ~1023u;      // 23552
constexpr uint32_t kChainStride = 68;                                // fp32 staging row pitch (floats)
constexpr uint32_t kChainScratch = 128 * kChainStride * 4;           // 34816 per consumer
constexpr uint32_t kChainOffW = 2048;
constexpr uint32_t kChainOffStage = kChainOffW + kWtBytes;           // 75776
constexpr uint32_t kChainOffScratch = kChainOffStage + 2 * kChainStage;
constexpr uint32_t kChainSmem = 1024 + kChainOffScratch + 2 * kChainScratch;
static_assert(kChainSmem <= kSmemLimit, "chain smem");
constexpr int kMaxMaps = 4;

struct ChainLayerP {
  const unsigned char* w;
  const float* bias;
  const __half* res;
  __half* y;
  int map, act;
};
struct ChainParams {
  CUtensorMap maps[kMaxMaps];
  ChainLayerP layers[TG_CHAIN_MAX_LAYERS];
  int n_layers, n, h, w, tiles_x, tiles_y, num_tiles;
  uint32_t* sync;
};

__global__ void __launch_bounds__(kChainThreads, 1) conv_chain_kernel(const __grid_constant__ ChainParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (base - raw);
  const int warp = __shfl_sync(0xFFFFFFFFu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const uint32_t bar_full = base, bar_empty = base + 16, bar_w = base + 32, bar_wfree = base + 40;

  if (warp == 1 && lane == 0) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, 4);
    }
    mbar_init(bar_w, 1);
    mbar_init(bar_wfree, 8);               // every warp of both consumers, once per layer
    fence_barrier_init();
  }
  __syncthreads();
  const uint32_t epoch = *reinterpret_cast<volatile const uint32_t*>(p.sync);
  uint32_t* flags = p.sync + kFlagBase;
  const int grid = (int)gridDim.x;
  const int cnt = (p.num_tiles - (int)blockIdx.x + grid - 1) / grid;   // tiles of this CTA per layer
  const int per_img = p.tiles_x * p.tiles_y;

  if (warp == 0) {
    // ============================================================ producer: weights per layer + halo boxes
    if (lane == 0) {
      uint32_t phase[2] = {0, 0};
      for (int l = 0; l < p.n_layers; ++l) {
        const ChainLayerP& L = p.layers[l];
        if (l > 0) mbar_wait_mma(bar_wfree, (uint32_t)(l - 1) & 1u);
        mbar_expect_tx(bar_w, kWtBytes);
        for (int t = 0; t < 9; ++t) bulk_load(base + kChainOffW + t * 8192u, L.w + (size_t)t * 8192u, 8192u, bar_w);
        for (int k = 0; k < cnt; ++k) {
          const int tile = (int)blockIdx.x + k * grid, cw = (l * cnt + k) & 1;
          const int img = tile / per_img, rr = tile - img * per_img, ty = rr / p.tiles_x, tx = rr - ty * p.tiles_x;
          if (l > 0) {
            // the tiles of layer l-1 under this tile's halo must have been published
            const uint32_t want = epoch * kEpochStride + (uint32_t)l;
            for (int dy = -1; dy <= 1; ++dy)
              for (int dx = -1; dx <= 1; ++dx) {
                const int y2 = ty + dy, x2 = tx + dx;
                if (y2 < 0 || y2 >= p.tiles_y || x2 < 0 || x2 >= p.tiles_x) continue;
                const uint32_t* f = flags + img * per_img + y2 * p.tiles_x + x2;
                if ((int)(ld_acquire_u32(f) - want) >= 0) continue;
                const long long t0 = clock64();
                while ((int)(ld_acquire_u32(f) - want) < 0) {
                  if (clock64() - t0 > 3000000000LL) __trap();   // bounded: a missing CTA must not hang the GPU
                }
              }
            fence_proxy_async_global();   // the halo is read by TMA (async proxy) after generic-proxy stores
          }
          const int s = cw;                 // one stage per consumer
          mbar_wait_mma(bar_empty + 8 * s, phase[cw] ^ 1);
          mbar_expect_tx(bar_full + 8 * s, kChainHalo);
          tma_load_4d(base + kChainOffStage + (uint32_t)s * kChainStage, &p.maps[L.map], bar_full + 8 * s, 0,
                      tx * TW - 1, ty * TH - 1, img);
          phase[cw] ^= 1u;
        }
      }
    }
  } else if (warp >= 4) {
    // ============================================================ consumers
    const int cw = (warp - 4) >> 2;
    const int r = threadIdx.x - 128 * (1 + cw), q = r >> 5;
    float* S = reinterpret_cast<float*>(sm + kChainOffScratch + (uint32_t)cw * kChainScratch);
    float* bias_s = reinterpret_cast<float*>(sm + 1024 + cw * 256);
    const uint32_t sa16 = gmma_addr16(base + kChainOffStage + (uint32_t)cw * kChainStage);
    const uint32_t w16 = gmma_addr16(base + kChainOffW);
    const int bar_id = 1 + cw;
    uint32_t phase = 0;
    float acc[2][32];
    for (int l = 0; l < p.n_layers; ++l) {
      const ChainLayerP& L = p.layers[l];
      if (r < 64) bias_s[r] = __ldg(L.bias + r);
      named_bar_sync(bar_id, 128);
      mbar_wait_mma(bar_w, (uint32_t)l & 1u);
      for (int k = 0; k < cnt; ++k) {
        if (((l * cnt + k) & 1) != cw) continue;
        const int tile = (int)blockIdx.x + k * grid;
        const int img = tile / per_img, rr = tile - img * per_img, ty = rr / p.tiles_x, tx = rr - ty * p.tiles_x;
        mbar_wait_mma(bar_full + 8 * cw, phase);
        phase ^= 1u;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int i = 0; i < 32; ++i) acc[h][i] = 0.f;
        wgmma_fence();
        halo_mmas(acc, sa16, w16);
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * cw);
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int i = 0; i < 32; i += 2) {
            const int row = h * 64 + q * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
            const int col = 8 * (i >> 2) + 2 * (lane & 3);
            *reinterpret_cast<float2*>(S + row * kChainStride + col) = make_float2(acc[h][i], acc[h][i + 1]);
          }
        named_bar_sync(bar_id, 128);
        // epilogue: thread = pixel, act(acc + bias) [+ residual] -> fp16 -> the pixel's 128-byte NHWC row
        const int py = ty * TH + (r >> 3), px = tx * TW + (r & 7);
        if (py < p.h && px < p.w) {
          const size_t off = (((size_t)img * p.h + py) * p.w + px) * 64;
          const float* srow = S + r * kChainStride;
#pragma unroll
          for (int c8 = 0; c8 < 8; ++c8) {
            uint4 rv = make_uint4(0u, 0u, 0u, 0u);
            if (L.res) rv = ld_global_u4(L.res + off + c8 * 8);
            const __half2* rh = reinterpret_cast<const __half2*>(&rv);
            const float4 a0 = reinterpret_cast<const float4*>(srow + c8 * 8)[0];
            const float4 a1 = reinterpret_cast<const float4*>(srow + c8 * 8)[1];
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            uint4 ov;
            __half2* o = reinterpret_cast<__half2*>(&ov);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              float v0 = tg_act(av[2 * j] + bias_s[c8 * 8 + 2 * j], L.act);
              float v1 = tg_act(av[2 * j + 1] + bias_s[c8 * 8 + 2 * j + 1], L.act);
              if (L.res) {
                const float2 rf = __half22float2(rh[j]);
                v0 += rf.x; v1 += rf.y;
              }
              o[j] = __floats2half2_rn(v0, v1);
            }
            *reinterpret_cast<uint4*>(L.y + off + c8 * 8) = ov;
          }
        }
        named_bar_sync(bar_id, 128);
        if (r == 0) {
          __threadfence();
          st_release_u32(flags + tile, epoch * kEpochStride + (uint32_t)l + 1u);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_wfree);   // this consumer no longer reads layer l's weights
    }
  }
  // the last CTA to finish advances the epoch for the next launch on this workspace
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const uint32_t done = atomicAdd(p.sync + 1, 1u);
    if (done == gridDim.x - 1) {
      p.sync[1] = 0;
      __threadfence();
      atomicAdd(p.sync, 1u);
    }
  }
}

// ================================================================== SRNet tail
// warpgroup 0 (WG-T) runs the transposed conv and its epilogue; warpgroups 1 and 2 (WG-O 0 / 1) run conv_out and
// the output of alternate tiles.  No producer warp: WG-T's thread 0 issues the halo TMAs.  WG-T holds two
// 64-register accumulator sets, each WG-O the conv_out products and the 12 output sums.
constexpr int kTailThreads = 384;
constexpr int kStepY = 15, kStepX = 7;               // input pixels a tile advances by
constexpr uint32_t kTailHalo = (TW + 1) * (TH + 1) * 128;            // 19584
constexpr uint32_t kTailStage = (kTailHalo + 1023u) & ~1023u;        // 20480
constexpr int kTailStages = 2;                       // halo ring: the tile in use + the next one loading
constexpr uint32_t kWoBytes = TG_TAPN_ROWS * 128;                    // [48 rows = tap*4+co][64]
constexpr uint32_t kHrBlock = 128 * 128;                             // one parity block: 128 px x 128 B
constexpr int kD2Pitch = 27;                         // tap products kept per HR pixel: 9 taps x 3 couts (fp32)
// the tap products of one parity block [128 px][27] fp32, + room for the shift-add's reads one block row and one
// tap row past the end; its reads up to one block row before the start land in the weights placed before it
constexpr uint32_t kD2Bytes = (((128 + 9) * kD2Pitch + 12) * 4 + 1023u) & ~1023u;   // 15360
// layout: header | w_up | D2 of WG-O 0 | w_out | D2 of WG-O 1 | 2 halo stages | 2 operand blocks per WG-O (each D2
// follows static weights, so the reads before its start never race with a write)
constexpr uint32_t kTailOffWt = 2048;
constexpr uint32_t kTailOffD2a = kTailOffWt + kWtBytes;              // 75776
constexpr uint32_t kTailOffWo = kTailOffD2a + kD2Bytes;              // 91136
constexpr uint32_t kTailOffD2b = kTailOffWo + kWoBytes;              // 97280
constexpr uint32_t kTailOffHalo = kTailOffD2b + kD2Bytes;            // 112640
constexpr uint32_t kTailOffBlk = kTailOffHalo + kTailStages * kTailStage;   // 153600
constexpr uint32_t kTailSmem = 1024 + kTailOffBlk + 4 * kHrBlock;    // 220160
static_assert(kTailSmem <= kSmemLimit, "tail smem");
static_assert(kWoBytes >= 9 * kD2Pitch * 4, "w_out must cover the reads before D2[1] (one block row + 1 pixel)");
static_assert(kTailOffWo % 1024 == 0 && kTailOffHalo % 1024 == 0 && kTailOffBlk % 1024 == 0, "swizzle atoms");

struct TailParams {
  CUtensorMap map_x;
  const unsigned char* w_up;
  const unsigned char* w_out;
  const float* b_up;
  const float* b_out;
  const float* lr;
  float* y;
  uint8_t* y_u8;
  int n, h, w, cout_real, lr_scale, up_mode, accumulate;
  int tiles_x, tiles_y, num_tiles;
};

// WG-T's epilogue of one parity: +bias, ReLU, zero for input pixels outside the image (conv_out's zero padding),
// fp16 -> stmatrix.trans into an operand block.  lane l of warp q addresses pixel row l%8 of 8x8 matrix m = l/8 =
// (tile row 2*jp + m/2, 8-channel chunk 2*q + m%2) through mat_off.
__device__ __forceinline__ void tail_convT_epilogue(const float (&acc)[64], uint32_t blk, uint32_t mat_off, float b0,
                                                    float b1, int y0, int x0, int lane, int h, int w) {
#pragma unroll
  for (int jp = 0; jp < 8; ++jp) {
    uint32_t ov[4];
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int i = 4 * (2 * jp + (m >> 1)) + 2 * (m & 1);
      const int iy = y0 + 2 * jp + (m >> 1), ix = x0 + 2 * (lane & 3);
      const bool rin = iy >= 0 && iy < h;
      const float bb = (m & 1) ? b1 : b0;
      const float v0 = rin && ix >= 0 && ix < w ? tg_act(acc[i] + bb, TG_ACT_RELU) : 0.f;
      const float v1 = rin && ix + 1 >= 0 && ix + 1 < w ? tg_act(acc[i + 1] + bb, TG_ACT_RELU) : 0.f;
      const __half2 hv = __floats2half2_rn(v0, v1);
      ov[m] = *reinterpret_cast<const uint32_t*>(&hv);
    }
    stmatrix_x4_trans(blk + (uint32_t)jp * 2048u + mat_off, ov);
  }
}

__global__ void __launch_bounds__(kTailThreads, 1) convT_convout_kernel(const __grid_constant__ TailParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_raw + (base - raw);
  const int warp = __shfl_sync(0xFFFFFFFFu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  // bar_halo[s]: halo stage s has landed (TMA bytes).  bar_full[2c + b] / bar_empty[2c + b]: WG-O c's operand
  // block b has been written by WG-T (one arrival per WG-T warp) / read by WG-O c's conv_out MMAs (one arrival per
  // WG-O warp).
  const uint32_t bar_halo = base, bar_w = base + 32, bar_full = base + 40, bar_empty = base + 72;
  float* bup_s = reinterpret_cast<float*>(sm + 1024);
  float* bout_s = reinterpret_cast<float*>(sm + 1024 + 256);

  if (threadIdx.x == 0) {
    for (int s = 0; s < kTailStages; ++s) mbar_init(bar_halo + 8 * s, 1);
    mbar_init(bar_w, 1);
    for (int b = 0; b < 4; ++b) {
      mbar_init(bar_full + 8 * b, 4);
      mbar_init(bar_empty + 8 * b, 4);
    }
    fence_barrier_init();
  }
  __syncthreads();
  // weights are static: load them before the programmatic-dependent-launch wait
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.map_x);
    mbar_expect_tx(bar_w, kWtBytes + kWoBytes);
    for (int t = 0; t < 9; ++t) bulk_load(base + kTailOffWt + t * 8192u, p.w_up + (size_t)t * 8192u, 8192u, bar_w);
    bulk_load(base + kTailOffWo, p.w_out, kWoBytes, bar_w);
  }
  tg_pdl_wait();
  tg_pdl_trigger();
  if (threadIdx.x < 64) bup_s[threadIdx.x] = __ldg(p.b_up + threadIdx.x);
  if (threadIdx.x < 4) bout_s[threadIdx.x] = threadIdx.x < p.cout_real ? __ldg(p.b_out + threadIdx.x) : 0.f;
  __syncthreads();
  const int per_img = p.tiles_x * p.tiles_y;
  const int grid = (int)gridDim.x;
  const int r = threadIdx.x & 127, q = r >> 5;
  const uint32_t blk0 = base + kTailOffBlk;

  // WG-T walks the CTA's tiles blockIdx.x + i * gridDim.x, parity a = 0..3 of each; WG-O c takes the tiles with
  // i % 2 == c.  Parity a of a tile goes through its WG-O's operand block a & 1, so each block is used twice per
  // tile of that WG-O and its k-th use has mbarrier phase k & 1 = a >> 1.  Deadlock-free: WG-T waits only on halo
  // stages (its own TMAs) and on bar_empty of a block whose previous use it has already published; WG-O waits only
  // on bar_full, which WG-T arrives on without waiting for anything later than that block's previous release.
  // Waits and arrivals on each block barrier alternate, so a parity wait is never more than one phase behind.
  if (warp < 4) {
    // ============================================================ WG-T: halo TMAs, transposed conv, epilogue
    const uint32_t wt16 = gmma_addr16(base + kTailOffWt);
    const uint32_t mat_off = (uint32_t)(8 * ((lane >> 3) >> 1) + (lane & 7)) * 128u +
                             ((uint32_t)((2 * q + ((lane >> 3) & 1)) ^ (lane & 7)) << 4);
    const float b0 = bup_s[16 * q + (lane >> 2)], b1 = bup_s[16 * q + (lane >> 2) + 8];
    // the CTA's i-th tile goes to halo stage i % 2
    auto load_halo = [&](int tile, int st) {
      const int img = tile / per_img, rr = tile - img * per_img;
      mbar_expect_tx(bar_halo + 8 * st, kTailHalo);
      tma_load_4d(base + kTailOffHalo + (uint32_t)st * kTailStage, &p.map_x, bar_halo + 8 * st, 0,
                  (rr % p.tiles_x) * kStepX - 1, (rr / p.tiles_x) * kStepY - 1, img);
    };
    if (r == 0)
      for (int k = 0; k < 2; ++k)
        if ((int)blockIdx.x + k * grid < p.num_tiles) load_halo((int)blockIdx.x + k * grid, k);
    int stage = 0;
    uint32_t phase = 0;
    int py0 = 0, px0 = 0;     // origin of the previous tile: its parity 3 is written under this tile's parity 0
    uint32_t cur = 0;         // 2 * (WG-O of the current tile): index of its first operand block
    float acc[2][64];         // parity a accumulates into acc[a & 1]
    mbar_wait_mma(bar_w, 0);
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += grid, cur ^= 2u) {
      const int img = tile / per_img, rr = tile - img * per_img;
      const int y0 = (rr / p.tiles_x) * kStepY - 1, x0 = (rr % p.tiles_x) * kStepX - 1;
      const int s = stage;
      mbar_wait_mma(bar_halo + 8 * s, phase);
      if (++stage == kTailStages) { stage = 0; phase ^= 1u; }
      const uint32_t x16 = gmma_addr16(base + kTailOffHalo + (uint32_t)s * kTailStage);
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        wgmma_fence();
        convT_pxn_mmas(acc[a & 1], x16, wt16, a);
        wgmma_commit();
        // parity a - 1 (for a = 0: the previous tile's parity 3) has landed; parity a stays in flight under its
        // epilogue
        wgmma_wait<1>();
        if (a == 0) {
          // every warp is past the previous tile's last MMAs: its halo stage takes the next tile
          named_bar_sync(1, 128);
          if (r == 0 && tile != (int)blockIdx.x && tile + grid < p.num_tiles) load_halo(tile + grid, s ^ 1);
        }
        if (a > 0 || tile != (int)blockIdx.x) {
          const int e = (a + 3) & 3;       // the parity written now
          const uint32_t b = (a > 0 ? cur : cur ^ 2u) + ((uint32_t)e & 1u);
          // the WG-O's MMAs have read this block's previous use (parity e - 2 of its tile, or of its previous tile)
          mbar_wait_mma(bar_empty + 8 * b, (uint32_t)((e >> 1) & 1) ^ 1u);
          tail_convT_epilogue(acc[e & 1], blk0 + b * kHrBlock, mat_off, b0, b1, a > 0 ? y0 : py0, a > 0 ? x0 : px0,
                              lane, p.h, p.w);
          fence_proxy_async_smem();        // generic-proxy writes -> read by wgmma (async proxy)
          __syncwarp();
          if (lane == 0) mbar_arrive(bar_full + 8 * b);
        }
      }
      py0 = y0;
      px0 = x0;
    }
    // the last tile's parity 3
    wgmma_wait<0>();
    if ((int)blockIdx.x < p.num_tiles) {
      const uint32_t b = (cur ^ 2u) + 1u;
      mbar_wait_mma(bar_empty + 8 * b, 0u);
      tail_convT_epilogue(acc[1], blk0 + b * kHrBlock, mat_off, b0, b1, py0, px0, lane, p.h, p.w);
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_full + 8 * b);
    }
  } else {
    // ============================================================ WG-O c: conv_out, shift-add, output
    const int c = (warp >> 2) - 1;
    const uint32_t wo16 = gmma_addr16(base + kTailOffWo);
    const uint64_t k_hi = gmma_desc_hi(1024u);
    float* D2 = reinterpret_cast<float*>(sm + (c ? kTailOffD2b : kTailOffD2a));
    // this thread's HR pixels of the tile's 32x16: (Y0 + 8j, X), j = 0..3; the interior 30x14 are outputs
    const int Y0 = r >> 4, X = r & 15;
    const int H = 2 * p.h, W = 2 * p.w;
    const int lh = H / p.lr_scale, lw = W / p.lr_scale;
    mbar_wait_mma(bar_w, 0);
    for (int tile = blockIdx.x + c * grid; tile < p.num_tiles; tile += 2 * grid) {
      const int img = tile / per_img, rr = tile - img * per_img;
      const int y0 = (rr / p.tiles_x) * kStepY - 1, x0 = (rr % p.tiles_x) * kStepX - 1;
      // the frame this tile adds onto is loaded into the output registers now; the loads complete under the MMAs
      float o[4][3];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int Y = Y0 + 8 * j, gy = 2 * y0 + Y, gx = 2 * x0 + X;
        const bool ok = Y >= 1 && Y <= 30 && X >= 1 && X <= 14 && gy >= 0 && gy < H && gx >= 0 && gx < W;
#pragma unroll
        for (int co = 0; co < 3; ++co) {
          o[j][co] = 0.f;
          if (p.accumulate && ok && co < p.cout_real)
            o[j][co] = p.y[(((size_t)img * p.cout_real + co) * H + gy) * W + gx];
        }
      }
      // parity a = (py, px) of the HR pixels: operand block -> conv_out tap products -> summed into the output
      // pixels they land on
#pragma unroll 1
      for (int a = 0; a < 4; ++a) {
        const uint32_t b = 2u * (uint32_t)c + ((uint32_t)a & 1u);
        const uint32_t blk16 = gmma_addr16(blk0 + b * kHrBlock);
        mbar_wait_mma(bar_full + 8 * b, (uint32_t)(a >> 1) & 1u);
        // conv_out as tap-major N (N = 48 = 9 taps x 4 couts) on the block
        float d2[2][24];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_n48(d2[0], k_hi | (uint64_t)(blk16 + 2u * k), k_hi | (uint64_t)(wo16 + 2u * k), k > 0 ? 1u : 0u);
          wgmma_n48(d2[1], k_hi | (uint64_t)(blk16 + 512u + 2u * k), k_hi | (uint64_t)(wo16 + 2u * k), k > 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * b);   // WG-T may write the block's next use
        named_bar_sync(2 + c, 128);                      // every thread has read the previous parity's D2
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int i = 0; i < 24; ++i) {
            const int row = h * 64 + q * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
            const int col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);   // = tap * 4 + co
            if (col < 36 && (col & 3) < 3) D2[row * kD2Pitch + (col >> 2) * 3 + (col & 3)] = d2[h][i];
          }
        named_bar_sync(2 + c, 128);
        // HR pixel (Y, X) takes tap (ty, tx) from HR pixel (Y + ty - 1, X + tx - 1); that pixel has parity a for
        // ty = ty0, ty0 + 2 (< 3) and tx = tx0, tx0 + 2 (< 3).  Only those slots are loaded (predicated, in slot
        // order); the padding around D2 keeps the reads for the ring pixels inside shared memory.
        const int ty0 = 1 - ((a >> 1) ^ (Y0 & 1)), tx0 = 1 - ((a & 1) ^ (X & 1));
#pragma unroll
        for (int sl = 0; sl < 4; ++sl) {
          const int ty = ty0 + 2 * (sl >> 1), tx = tx0 + 2 * (sl & 1);
          if (ty > 2 || tx > 2) continue;
          const float* d = D2 + (((Y0 + ty - 1) >> 1) * 8 + ((X + tx - 1) >> 1)) * kD2Pitch + (ty * 3 + tx) * 3;
#pragma unroll
          for (int j = 0; j < 4; ++j)        // HR row Y0 + 8j = block row ((Y0 + ty - 1) >> 1) + 4j
#pragma unroll
            for (int co = 0; co < 3; ++co) o[j][co] += d[j * 32 * kD2Pitch + co];
        }
      }
      // + bias (+ upsample_func(lr)) -> fp32 NCHW (+ uint8 NHWC).  One pixel per iteration (the selects keep o in
      // registers): the in-kernel upsample is inlined three times rather than twelve.
#pragma unroll 1
      for (int j = 0; j < 4; ++j) {
        float oj[3];
#pragma unroll
        for (int co = 0; co < 3; ++co) oj[co] = j == 0 ? o[0][co] : j == 1 ? o[1][co] : j == 2 ? o[2][co] : o[3][co];
        const int Y = Y0 + 8 * j, gy = 2 * y0 + Y, gx = 2 * x0 + X;
        if (Y < 1 || Y > 30 || X < 1 || X > 14 || gy < 0 || gy >= H || gx < 0 || gx >= W) continue;
        uint32_t q8[3] = {0u, 0u, 0u};
#pragma unroll
        for (int co = 0; co < 3; ++co) {
          if (co >= p.cout_real) continue;
          float v = oj[co] + bout_s[co];
          if (p.lr) v = v + tg_upsample_at(p.lr + ((size_t)img * p.cout_real + co) * lh * lw, lh, lw, lh, lw,
                                           p.lr_scale, p.up_mode, gy, gx);
          p.y[(((size_t)img * p.cout_real + co) * H + gy) * W + gx] = v;
          q8[co] = (uint32_t)fminf(fmaxf(rintf(v * 255.f), 0.f), 255.f);
        }
        if (p.y_u8) {
          uint8_t* up = p.y_u8 + (((size_t)img * H + gy) * W + gx) * p.cout_real;
#pragma unroll
          for (int co = 0; co < 3; ++co)
            if (co < p.cout_real) up[co] = (uint8_t)q8[co];
        }
      }
    }
  }
}

}  // namespace

extern "C" {

size_t tg_conv_chain_workspace_bytes(int n, int h, int w) {
  if (n <= 0 || h <= 0 || w <= 0) return 0;
  const size_t tiles = (size_t)tg_ceil_div(w, TW) * tg_ceil_div(h, TH) * n;
  return (kFlagBase + tiles) * sizeof(uint32_t);
}

int tg_conv_chain_tcgen05(const tg_chain_layer* layers, int n_layers, int n, int h, int w, void* sync_ws,
                          int max_ctas, void* stream) {
  TG_REQUIRE(layers != nullptr && sync_ws != nullptr, TG_E_INVALID, "conv_chain: null pointer");
  TG_REQUIRE(n_layers >= 1 && n_layers <= TG_CHAIN_MAX_LAYERS, TG_E_UNSUPPORTED,
             "conv_chain: n_layers=%d (1..%d)", n_layers, TG_CHAIN_MAX_LAYERS);
  TG_REQUIRE(n > 0 && h > 0 && w > 0, TG_E_INVALID, "conv_chain: bad size n=%d h=%d w=%d", n, h, w);
  TG_REQUIRE(((uintptr_t)sync_ws & 15) == 0, TG_E_INVALID, "conv_chain: sync_ws must be 16-byte aligned");
  ChainParams p;
  p.n_layers = n_layers; p.n = n; p.h = h; p.w = w;
  p.tiles_x = tg_ceil_div(w, TW);
  p.tiles_y = tg_ceil_div(h, TH);
  p.num_tiles = p.tiles_x * p.tiles_y * n;
  p.sync = reinterpret_cast<uint32_t*>(sync_ws);
  const void* bufs[kMaxMaps];
  int n_maps = 0;
  for (int l = 0; l < n_layers; ++l) {
    const tg_chain_layer& s = layers[l];
    TG_REQUIRE(s.x && s.weights && s.bias && s.y, TG_E_INVALID, "conv_chain: layer %d: null pointer", l);
    TG_REQUIRE(s.act >= TG_ACT_NONE && s.act <= TG_ACT_LRELU02, TG_E_INVALID, "conv_chain: layer %d: act", l);
    TG_REQUIRE(s.reserved == 0, TG_E_INVALID, "conv_chain: layer %d: reserved must be 0", l);
    TG_REQUIRE(s.y != s.x, TG_E_INVALID, "conv_chain: layer %d: y aliases x (halo reads of other tiles)", l);
    TG_REQUIRE(((uintptr_t)s.x & 15) == 0 && ((uintptr_t)s.y & 31) == 0 && ((uintptr_t)s.weights & 15) == 0 &&
                   ((uintptr_t)s.residual & 31) == 0 && ((uintptr_t)s.bias & 3) == 0,
               TG_E_INVALID, "conv_chain: layer %d: pointer alignment", l);
    int m = -1;
    for (int i = 0; i < n_maps; ++i)
      if (bufs[i] == s.x) m = i;
    if (m < 0) {
      TG_REQUIRE(n_maps < kMaxMaps, TG_E_UNSUPPORTED, "conv_chain: more than %d distinct input buffers", kMaxMaps);
      const int rc = encode_c64(&p.maps[n_maps], s.x, n, h, w, TW + 2, TH + 2);
      if (rc != TG_OK) return rc;
      bufs[n_maps] = s.x;
      m = n_maps++;
    }
    p.layers[l] = ChainLayerP{reinterpret_cast<const unsigned char*>(s.weights), s.bias,
                              reinterpret_cast<const __half*>(s.residual), reinterpret_cast<__half*>(s.y), m, s.act};
  }
  for (int i = n_maps; i < kMaxMaps; ++i) p.maps[i] = p.maps[0];
  for (int l = n_layers; l < TG_CHAIN_MAX_LAYERS; ++l) p.layers[l] = p.layers[0];

  static TgPerDeviceOnce attr_once;
  const cudaError_t attr_err = attr_once.run([] {
    return cudaFuncSetAttribute(conv_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kChainSmem);
  });
  TG_REQUIRE(attr_err == cudaSuccess, (int)attr_err, "conv_chain: cudaFuncSetAttribute: %s", cudaGetErrorString(attr_err));
  int sms = 0;
  int rc = tg_device_sm_count(&sms);
  if (rc != TG_OK) return rc;
  // Every CTA must be resident at once (tiles wait on tiles of other CTAs): one CTA per SM, and a
  // COOPERATIVE launch, so the driver starts the grid only when all of its CTAs can be co-scheduled.
  int per_sm = 0;
  const cudaError_t oerr =
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, conv_chain_kernel, kChainThreads, kChainSmem);
  TG_REQUIRE(oerr == cudaSuccess, (int)oerr, "conv_chain: occupancy query: %s", cudaGetErrorString(oerr));
  TG_REQUIRE(per_sm >= 1, TG_E_UNSUPPORTED, "conv_chain: kernel does not fit on an SM of this device");
  int grid = (max_ctas > 0 && max_ctas < sms) ? max_ctas : sms;
  if (grid > p.num_tiles) grid = p.num_tiles;
  const cudaError_t lerr =
      tg_launch_cooperative(conv_chain_kernel, dim3(grid), dim3(kChainThreads), kChainSmem, (cudaStream_t)stream, p);
  TG_REQUIRE(lerr == cudaSuccess, (int)lerr, "conv_chain: launch failed: %s", cudaGetErrorString(lerr));
  TG_CUDA_LAUNCH_CHECK("conv_chain");
  return TG_OK;
}

int tg_convT_convout_tcgen05(const tg_tail_desc* d, void* stream) {
  TG_REQUIRE(d != nullptr, TG_E_INVALID, "convT_convout: null descriptor");
  TG_REQUIRE(d->x && d->w_up && d->b_up && d->w_out && d->b_out && d->y, TG_E_INVALID, "convT_convout: null pointer");
  TG_REQUIRE(d->n > 0 && d->h > 0 && d->w > 0, TG_E_INVALID, "convT_convout: bad size");
  TG_REQUIRE(d->cout_real >= 1 && d->cout_real <= 3, TG_E_UNSUPPORTED, "convT_convout: out_nc=%d (1..3)", d->cout_real);
  TG_REQUIRE(d->reserved == 0, TG_E_INVALID, "convT_convout: reserved must be 0");
  TG_REQUIRE(!(d->accumulate && d->lr), TG_E_INVALID, "convT_convout: accumulate and lr are exclusive");
  TG_REQUIRE(((uintptr_t)d->x & 15) == 0 && ((uintptr_t)d->w_up & 15) == 0 && ((uintptr_t)d->w_out & 15) == 0 &&
                 ((uintptr_t)d->y & 7) == 0, TG_E_INVALID, "convT_convout: pointer alignment");
  if (d->lr != nullptr) {
    TG_REQUIRE(d->lr_scale == 2 || d->lr_scale == 4, TG_E_UNSUPPORTED, "convT_convout: lr_scale %d (2 or 4)", d->lr_scale);
    TG_REQUIRE((2 * d->h) % d->lr_scale == 0 && (2 * d->w) % d->lr_scale == 0, TG_E_INVALID,
               "convT_convout: output size is not lr_scale x the LR size");
    TG_REQUIRE(d->up_mode == TG_UP_BICUBIC || d->up_mode == TG_UP_BILINEAR, TG_E_INVALID, "convT_convout: up_mode");
  }
  TailParams p;
  int rc = encode_c64(&p.map_x, d->x, d->n, d->h, d->w, TW + 1, TH + 1);
  if (rc != TG_OK) return rc;
  p.w_up = reinterpret_cast<const unsigned char*>(d->w_up);
  p.w_out = reinterpret_cast<const unsigned char*>(d->w_out);
  p.b_up = d->b_up; p.b_out = d->b_out; p.lr = d->lr; p.y = d->y; p.y_u8 = d->y_u8;
  p.n = d->n; p.h = d->h; p.w = d->w; p.cout_real = d->cout_real;
  p.lr_scale = d->lr ? d->lr_scale : 2; p.up_mode = d->up_mode; p.accumulate = d->accumulate;
  // HR rows -1 .. 2h-1 are covered in strips of 30 (the first strip starts at the even row -2)
  p.tiles_y = tg_ceil_div(2 * d->h + 1, 2 * kStepY);
  p.tiles_x = tg_ceil_div(2 * d->w + 1, 2 * kStepX);
  p.num_tiles = p.tiles_x * p.tiles_y * d->n;
  static TgPerDeviceOnce attr_once;
  const cudaError_t attr_err = attr_once.run([] {
    return cudaFuncSetAttribute(convT_convout_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTailSmem);
  });
  TG_REQUIRE(attr_err == cudaSuccess, (int)attr_err, "convT_convout: cudaFuncSetAttribute: %s",
             cudaGetErrorString(attr_err));
  int sms = 0;
  rc = tg_device_sm_count(&sms);
  if (rc != TG_OK) return rc;
  int grid = d->max_ctas > 0 && d->max_ctas < sms ? d->max_ctas : sms;
  if (grid > p.num_tiles) grid = p.num_tiles;
  const cudaError_t lerr =
      tg_launch(convT_convout_kernel, dim3(grid), dim3(kTailThreads), kTailSmem, (cudaStream_t)stream, p);
  TG_REQUIRE(lerr == cudaSuccess, (int)lerr, "convT_convout: launch failed: %s", cudaGetErrorString(lerr));
  TG_CUDA_LAUNCH_CHECK("convT_convout");
  return TG_OK;
}

}  // extern "C"
