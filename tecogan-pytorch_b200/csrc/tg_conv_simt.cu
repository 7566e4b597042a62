// Weight packing + the CUDA-core cross-check convolution.
//
// tg_conv_simt implements exactly the tg_conv_desc contract of the tcgen05 kernel (same packed
// weights, same epilogues) with one thread per (input pixel, accumulator, 8 output channels) and
// fp32 accumulation.  It exists so the GPU tests can tell a tensor-core descriptor bug from a
// packing / epilogue bug; the hot path never calls it.
#include "tg_common.cuh"
#include "tg_epilogue.cuh"

namespace {

// ------------------------------------------------------------------ weight packing
// conv3x3: w[co][ci][ky][kx] -> tile (g=ky*3+kx, chunk=ci/64), element (row=co, k=ci%64)
// convT  : w[ci][co][ky][kx] -> tile (g per tg_group(TG_CONVT_3X3_S2, g)), same element map
// dgrad  : (kind = TG_CONV_3X3, dgrad = 1) the layer's roles are swapped and the taps flipped: `cout`/`cin`
//          are the dgrad layer's (= the forward layer's cin/cout), source w_fwd[ci'][co'][2-ky][2-kx] with
//          w_fwd laid out [cout_fwd = cin][cin_fwd = cout][3][3]
__global__ void pack_weights_kernel(const float* __restrict__ w, __half* __restrict__ packed,
                                    int kind, int cout, int cin, int cout_pad, int cin_pad, int dgrad) {
  tg_pdl_wait();
  // no early trigger: the weights this kernel writes are loaded by the next conv BEFORE its PDL wait
  const int chunks = cin_pad / 64;
  const size_t total = (size_t)9 * chunks * cout_pad * 64;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % 64);
    const int row = (int)((i / 64) % cout_pad);
    const int tile = (int)(i / ((size_t)64 * cout_pad));
    const int chunk = tile % chunks, g = tile / chunks;
    const int ci = chunk * 64 + k, co = row;
    const TgGroup gr = tg_group(kind, g);
    float v = 0.f;
    if (ci < cin && co < cout) {
      if (dgrad)                        v = w[(((size_t)ci * cout + co) * 3 + (2 - gr.ky)) * 3 + (2 - gr.kx)];
      else if (kind != TG_CONVT_3X3_S2) v = w[(((size_t)co * cin + ci) * 3 + gr.ky) * 3 + gr.kx];
      else                              v = w[(((size_t)ci * cout + co) * 3 + gr.ky) * 3 + gr.kx];
    }
    const size_t tile_bytes = (size_t)cout_pad * 128;
    unsigned char* base = reinterpret_cast<unsigned char*>(packed) + (size_t)tile * tile_bytes;
    *reinterpret_cast<__half*>(base + tg_wtile_off(row, k)) = __float2half(v);
  }
}

// tap-major N layout for thin heads: tile per chunk [48 rows][64 k], row = tap*4 + co
__global__ void pack_weights_tapn_kernel(const float* __restrict__ w, __half* __restrict__ packed,
                                         int cout, int cin, int cin_pad) {
  tg_pdl_wait();
  // no early trigger: the weights this kernel writes are loaded by the next conv BEFORE its PDL wait
  const int chunks = cin_pad / 64;
  const size_t total = (size_t)chunks * TG_TAPN_ROWS * 64;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % 64);
    const int row = (int)((i / 64) % TG_TAPN_ROWS);
    const int chunk = (int)(i / ((size_t)64 * TG_TAPN_ROWS));
    const int tap = row >> 2, co = row & 3, ci = chunk * 64 + k;
    float v = 0.f;
    if (tap < 9 && co < cout && ci < cin) v = w[(((size_t)co * cin + ci) * 3 + tap / 3) * 3 + tap % 3];
    unsigned char* base = reinterpret_cast<unsigned char*>(packed) + (size_t)chunk * TG_TAPN_ROWS * 128;
    *reinterpret_cast<__half*>(base + tg_wtile_off(row, k)) = __float2half(v);
  }
}

// ------------------------------------------------------------------ cross-check conv
__global__ void conv_simt_kernel(tg_conv_desc d) {
  tg_pdl_wait();
  tg_pdl_trigger();
  const int chunks = d.cin / 64;
  const int n_acc = d.kind == TG_CONVT_3X3_S2 ? 4 : 1;
  const bool tapn = d.epilogue != TG_EPI_NHWC_F16;
  const int co_groups = tapn ? 1 : d.cout / 8;
  const size_t total = (size_t)d.n * d.h * d.w * n_acc * co_groups;
  const __half* x = reinterpret_cast<const __half*>(d.x);
  const unsigned char* wp = reinterpret_cast<const unsigned char*>(d.weights);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x) {
    const int cg = (int)(i % co_groups);
    size_t p = i / co_groups;
    const int acc = (int)(p % n_acc); p /= n_acc;
    const int xx = (int)(p % d.w); p /= d.w;
    const int yy = (int)(p % d.h);
    const int nn = (int)(p / d.h);
    float a[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = 0.f;
    for (int g = 0; g < 9; ++g) {
      const TgGroup gr = tg_group(d.kind, g);
      if (gr.acc != acc) continue;
      int iy = yy + gr.dy, ix = xx + gr.dx, IH = d.h, IW = d.w;
      if (d.kind == TG_CONV_3X3_S2) { iy = 2 * yy + gr.ky - 1; ix = 2 * xx + gr.kx - 1; IH = 2 * d.h; IW = 2 * d.w; }
      if (iy < 0 || iy >= IH || ix < 0 || ix >= IW) continue;  // zero padding
      const __half* px = x + (((size_t)nn * IH + iy) * IW + ix) * d.cin;
      for (int ci = 0; ci < d.cin; ++ci) {
        const float xv = __half2float(px[ci]);
        if (tapn) {   // NCHW heads: tile per chunk, row = tap*4 + co, 4 real output channels max
          const unsigned char* tile = wp + (size_t)(ci / 64) * TG_TAPN_ROWS * 128;
#pragma unroll
          for (int j = 0; j < 4; ++j)
            a[j] += xv * __half2float(*reinterpret_cast<const __half*>(
                             tile + tg_wtile_off(g * 4 + j, ci & 63)));
        } else {
          const unsigned char* tile = wp + (size_t)(g * chunks + ci / 64) * d.cout * 128;
#pragma unroll
          for (int j = 0; j < 8; ++j)
            a[j] += xv * __half2float(*reinterpret_cast<const __half*>(
                             tile + tg_wtile_off(cg * 8 + j, ci & 63)));
        }
      }
    }
    // output pixel of this accumulator
    int oy = yy, ox = xx, OH = d.h, OW = d.w;
    if (d.kind == TG_CONVT_3X3_S2) { oy = 2 * yy + (acc >> 1); ox = 2 * xx + (acc & 1); OH = 2 * d.h; OW = 2 * d.w; }
    tg_epilogue_store8(d, nn, oy, ox, OH, OW, cg * 8, a);
  }
}

}  // namespace

extern "C" {

size_t tg_packed_weight_bytes(int cin_pad, int cout_pad) {
  if (cin_pad <= 0 || cout_pad <= 0 || cin_pad % 64 != 0 || cout_pad % 16 != 0) return 0;
  return (size_t)9 * (cin_pad / 64) * cout_pad * 128;
}

static int pack_common(const float* w, int kind, int cout, int cin, void* packed, int cout_pad,
                       int cin_pad, void* stream, int dgrad = 0) {
  TG_REQUIRE(w && packed, TG_E_INVALID, "pack_weights: null pointer");
  TG_REQUIRE(cout > 0 && cin > 0 && cout <= cout_pad && cin <= cin_pad, TG_E_INVALID,
             "pack_weights: cout=%d cin=%d exceed pads %d/%d", cout, cin, cout_pad, cin_pad);
  TG_REQUIRE(cin_pad % 64 == 0 && cout_pad % 16 == 0 && cout_pad <= 512, TG_E_UNSUPPORTED,
             "pack_weights: cin_pad %% 64, cout_pad %% 16, cout_pad <= 512 required");
  const size_t total = (size_t)9 * cin_pad * cout_pad;
  int grid = (int)((total + 255) / 256);
  if (grid > tg_sms() * 16) grid = tg_sms() * 16;
  tg_launch(pack_weights_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, w, (__half*)packed, kind, cout, cin,
            cout_pad, cin_pad, dgrad);
  TG_CUDA_LAUNCH_CHECK("pack_weights");
  return TG_OK;
}

int tg_pack_conv3x3_weights(const float* w_oihw, int cout, int cin, void* packed, int cout_pad,
                            int cin_pad, void* stream) {
  return pack_common(w_oihw, TG_CONV_3X3, cout, cin, packed, cout_pad, cin_pad, stream);
}

int tg_pack_convT3x3s2_weights(const float* w_iohw, int cin, int cout, void* packed, int cout_pad,
                               int cin_pad, void* stream) {
  return pack_common(w_iohw, TG_CONVT_3X3_S2, cout, cin, packed, cout_pad, cin_pad, stream);
}

int tg_pack_conv3x3_weights_dgrad(const float* w_oihw, int cout, int cin, void* packed, int cin_as_cout_pad,
                                  int cout_as_cin_pad, void* stream) {
  // the dgrad layer computes cin outputs from cout inputs
  return pack_common(w_oihw, TG_CONV_3X3, cin, cout, packed, cin_as_cout_pad, cout_as_cin_pad, stream, 1);
}

int tg_pack_conv3x3s2_weights(const float* w_oihw, int cout, int cin, void* packed, int cout_pad, int cin_pad,
                              void* stream) {
  return pack_common(w_oihw, TG_CONV_3X3_S2, cout, cin, packed, cout_pad, cin_pad, stream);
}

size_t tg_packed_weight_bytes_tapn(int cin_pad) {
  if (cin_pad <= 0 || cin_pad % 64 != 0) return 0;
  return (size_t)(cin_pad / 64) * TG_TAPN_ROWS * 128;
}

int tg_pack_conv3x3_weights_tapn(const float* w_oihw, int cout, int cin, void* packed, int cin_pad,
                                 void* stream) {
  TG_REQUIRE(w_oihw && packed, TG_E_INVALID, "pack_weights_tapn: null pointer");
  TG_REQUIRE(cout >= 1 && cout <= 4 && cin > 0 && cin <= cin_pad && cin_pad % 64 == 0, TG_E_UNSUPPORTED,
             "pack_weights_tapn: cout=%d (<=4) cin=%d cin_pad=%d", cout, cin, cin_pad);
  tg_launch(pack_weights_tapn_kernel, dim3((cin_pad / 64) * 12), dim3(256), 0, (cudaStream_t)stream, w_oihw,
            (__half*)packed, cout, cin, cin_pad);
  TG_CUDA_LAUNCH_CHECK("pack_weights_tapn");
  return TG_OK;
}

int tg_conv_validate(const tg_conv_desc* d, const char* who);

int tg_conv_simt(const tg_conv_desc* d, void* stream) {
  int rc = tg_conv_validate(d, "conv_simt");
  if (rc != TG_OK) return rc;
  TG_REQUIRE(d->epilogue != TG_EPI_NHWC_F16_POOL2, TG_E_UNSUPPORTED, "conv_simt: pooled epilogue is tcgen05-only");
  const int n_acc = d->kind == TG_CONVT_3X3_S2 ? 4 : 1;
  const size_t total = (size_t)d->n * d->h * d->w * n_acc *
                       (d->epilogue != TG_EPI_NHWC_F16 ? 1 : d->cout / 8);
  size_t grid = (total + 127) / 128;
  if (grid > (size_t)tg_sms() * 64) grid = (size_t)tg_sms() * 64;
  tg_launch(conv_simt_kernel, dim3((unsigned)grid), dim3(128), 0, (cudaStream_t)stream, *d);
  TG_CUDA_LAUNCH_CHECK("conv_simt");
  return TG_OK;
}

}  // extern "C"
