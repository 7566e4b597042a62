/*
 * tecogan_b200.h -- C ABI of libtecogan_b200.so (sm_90a, H100).  Entry points keep their
 * historical *_tcgen05 names; on sm_90a they run wgmma kernels.
 *
 * The reference (skycrapers/TecoGAN-PyTorch @ 903b070) has NO native / FFI
 * boundary: its generator hot path is Python calling PyTorch library ops
 * (SURVEY.md 2.1, 8-b).  This ABI is therefore new; each entry point cites the
 * reference Python call site whose arithmetic it replaces.  The Python host
 * (tecogan-pytorch_b200/) binds it with ctypes and keeps the reference's
 * nn.Module surface (FRNet / FNet / SRNet / define_generator); INTEGRATION.md
 * shows the stub a reference maintainer would add.
 *
 * Conventions
 *   - every function returns int: 0 = OK, <0 = invalid argument / unsupported
 *     shape (TG_E_*), >0 = cudaError_t.  Nothing throws.
 *   - every pointer is a caller-owned DEVICE pointer unless named host_*;
 *     no ownership transfer, no hidden allocation, no hidden synchronisation.
 *   - all work is enqueued on the cudaStream_t passed last (as void*), so the
 *     calls are CUDA-graph capturable.
 *   - activation layout inside the path: NHWC fp16, channel count a multiple
 *     of 64 ("c64"); module boundaries are NCHW fp32 like the reference.
 *   - tg_last_error_string() describes the most recent failure of this thread.
 */
#ifndef TECOGAN_B200_H_
#define TECOGAN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TG_ABI_VERSION 2   /* 2: tg_conv_desc.mask, backward (training) entry points; tg_conv_desc.reserved became
                              cin_real (0 keeps the old meaning: all stored input channels are used) */
#define TG_TAPN_ROWS 48   /* 9 taps x 4 output channels, padded to a multiple of 16 */
#define TG_TAIL_OUT_ROWS 40   /* the fused tail's conv_out N: 5 x (2 taps x 4 output channels) */

enum {
  TG_OK = 0,
  TG_E_INVALID = -1,      /* null pointer, non-positive size, bad enum       */
  TG_E_UNSUPPORTED = -2,  /* shape / channel count the kernels do not cover  */
  TG_E_DRIVER = -3        /* cuTensorMapEncodeTiled unavailable or failed    */
};

enum {
  TG_ACT_NONE = 0, TG_ACT_RELU = 1, TG_ACT_LRELU02 = 2,
  /* data-gradient epilogues: y = (conv + bias [+ residual]) * act'(mask), the derivative taken from
   * the STORED forward output `mask` of the layer the gradient flows into (sign(out) == sign(pre-act)) */
  TG_ACT_DRELU = 3,     /* * (mask > 0 ? 1 : 0)   */
  TG_ACT_DLRELU02 = 4   /* * (mask > 0 ? 1 : 0.2) */
};
enum {
  TG_CONV_3X3 = 0,
  TG_CONVT_3X3_S2 = 1,
  TG_CONV_3X3_S2 = 2    /* stride-2 conv, pad 1: y[oy,ox] = sum x[2oy+ky-1, 2ox+kx-1] * w[.,.,ky,kx] -- the data
                           gradient of TG_CONVT_3X3_S2 (wgmma: tap mode over the four parity planes of x) */
};
enum { TG_UP_BICUBIC = 0, TG_UP_BILINEAR = 1 };
enum {
  TG_EPI_NHWC_F16 = 0,      /* y = act(conv + bias) [+ residual]  -> NHWC fp16        */
  TG_EPI_FLOW_NCHW_F32 = 1, /* y = 24*tanh(conv + bias)           -> NCHW fp32 [N,2,H,W] */
  TG_EPI_OUT_NCHW_F32 = 2,  /* y = conv + bias                    -> NCHW fp32 [N,C,H,W] */
  TG_EPI_NHWC_F16_POOL2 = 3 /* y = maxpool2x2(act(conv + bias))   -> NHWC fp16 [n,h/2,w/2,cout]: nn.MaxPool2d(2,2)
                               (tecogan_nets.py:28,35,42) folded into the producing conv's epilogue (wgmma kernel,
                               conv3x3 only, no residual); the full-resolution map is never written */
};
enum { TG_AMODE_AUTO = 0, TG_AMODE_HALO = 1, TG_AMODE_TAP = 2 };
/* Flag OR'd into tg_conv_desc.a_mode (wgmma kernel only): walk the tiles last to first.  The output bits do not
 * depend on the walk.  A launch that reads a map the previous launch wrote then starts on the tiles written last,
 * which are the ones still in L2; networks.py alternates the direction along each chain of convs. */
#define TG_AMODE_REVERSE 0x100

int tg_version(void);
const char* tg_last_error_string(void);
/* number of SMs of the current device (132 on H100 SXM) */
int tg_device_sm_count(int* out_sm_count);

/* ------------------------------------------------------------------------
 * Weight packing (run once per optimizer step / checkpoint load).
 * Packed layout = the exact shared-memory image the wgmma kernel consumes:
 * tiles [group g][chunk c][cout_pad rows][64 k] fp16, 128-byte rows with the
 * 128B swizzle (16-byte chunk index XOR (row & 7)); g = ky*3+kx for conv3x3.
 * ---------------------------------------------------------------------- */
size_t tg_packed_weight_bytes(int cin_pad, int cout_pad);
/* nn.Conv2d(cin,cout,3,1,1).weight [cout,cin,3,3] fp32 (tecogan_nets.py:24-65,93-95,112,131) */
int tg_pack_conv3x3_weights(const float* w_oihw, int cout, int cin, void* packed,
                            int cout_pad, int cin_pad, void* stream);
/* nn.ConvTranspose2d(cin,cout,3,2,1,output_padding=1).weight [cin,cout,3,3] fp32
 * (tecogan_nets.py:119-126) -> 9 tiles grouped by output parity (1/2/2/4 taps) */
int tg_pack_convT3x3s2_weights(const float* w_iohw, int cin, int cout, void* packed,
                               int cout_pad, int cin_pad, void* stream);
/* Data-gradient operands (autograd of the above under loss.backward(), vsr_model.py:92):
 *  - conv3x3 dgrad = conv3x3 of dz with the taps flipped and cin/cout swapped: packs
 *    w'[ci][co][ky][kx] = w[co][ci][2-ky][2-kx] from the nn.Conv2d weight [cout,cin,3,3]; run it as a
 *    TG_CONV_3X3 layer with cin_pad(layer) = pad(cout), cout_pad(layer) = pad(cin).
 *  - convT dgrad = TG_CONV_3X3_S2 over dz with w'[ci][co][ky][kx] = wt[ci][co][ky][kx]: the
 *    nn.ConvTranspose2d weight [cin,cout,3,3] read as an OIHW conv weight (out = cin, in = cout). */
int tg_pack_conv3x3_weights_dgrad(const float* w_oihw, int cout, int cin, void* packed, int cin_as_cout_pad,
                                  int cout_as_cin_pad, void* stream);
int tg_pack_conv3x3s2_weights(const float* w_oihw, int cout, int cin, void* packed, int cout_pad, int cin_pad,
                              void* stream);
/* Thin heads (cout <= 4: FNet flow head 32->2, SRNet conv_out 64->3) use the "tap-major N"
 * layout: one tile per 64-ch chunk, [48 rows][64 k], row = tap*4 + co (rows >= 36 zero).  One
 * MMA group then yields all nine tap products of a pixel (N = 48) and the 3x3 shift-add happens
 * in the epilogue -- 4 MMAs per 128 pixels instead of 36.  Used with the two NCHW epilogues. */
size_t tg_packed_weight_bytes_tapn(int cin_pad);
int tg_pack_conv3x3_weights_tapn(const float* w_oihw, int cout, int cin, void* packed, int cin_pad,
                                 void* stream);

/* ------------------------------------------------------------------------
 * 3x3 convolution / stride-2 transposed convolution as wgmma implicit GEMM.
 * Replaces nn.Conv2d+activation (tecogan_nets.py:23-65, 92-98, 111-116, 131),
 * nn.ConvTranspose2d+ReLU (:119-126), torch.tanh(.)*24 (:80) and the add of
 * `out += upsample_func(lr_curr)` (:145): TG_EPI_OUT_NCHW_F32 stores conv+bias and the caller
 * then runs tg_upsample_nchw_f32(lr_curr, accumulate=1) on the same buffer (the epilogue is a pure
 * store: a read-modify-write there exposes a global-load round trip per tile).
 * ---------------------------------------------------------------------- */
typedef struct tg_conv_desc {
  const void* x;        /* NHWC fp16 [n,h,w,cin]  (TG_CONV_3X3_S2: [n,2h,2w,cin])                */
  const void* weights;  /* packed weights (tg_pack_*)                                    */
  const float* bias;    /* fp32 [cout] (zero padded)                                     */
  const void* residual; /* NHWC fp16 [n,h,w,cout] or NULL (TG_EPI_NHWC_F16, conv3x3 only) */
  void* y;              /* see epilogue; convT writes [n,2h,2w,cout]                     */
  int32_t n, h, w;      /* batch and the height / width the kernel tiles over: the input's (= the
                           output's for conv3x3; convT writes 2h x 2w), the OUTPUT's for TG_CONV_3X3_S2 */
  int32_t cin, cout;    /* stored channel counts: cin in {64,128,192,256,384,512}; cout in {64,...,384,512}
                           for TG_EPI_NHWC_F16, 48 (= TG_TAPN_ROWS, tap-major N packing)
                           for the two NCHW epilogues                                    */
  int32_t cout_real;    /* NCHW epilogues: channels actually written (2 resp. 3)         */
  int32_t kind;         /* TG_CONV_3X3 | TG_CONVT_3X3_S2                                 */
  int32_t act;          /* TG_ACT_*                                                      */
  int32_t epilogue;     /* TG_EPI_*                                                      */
  int32_t a_mode;       /* TG_AMODE_* (wgmma kernel only; AUTO = fastest validated), | TG_AMODE_REVERSE */
  int32_t max_ctas;     /* 0 = one persistent CTA per SM                                 */
  int32_t cin_real;     /* input channels that can be non-zero (0 = cin): for cin = 64 the wgmma kernel skips the
                           k-steps of 16 channels at or beyond it -- the packed weights are zero there, so the
                           result is bit-identical (thin layers: FNet 6->32, 32->32, 32->64, 32->2)  */
  const void* mask;     /* TG_ACT_DRELU / TG_ACT_DLRELU02: NHWC fp16, shape of y; else NULL */
} tg_conv_desc;

int tg_conv_tcgen05(const tg_conv_desc* d, void* stream);
/* Same contract on CUDA cores (fp32 accumulate, reads the same packed weights):
 * bring-up / cross-check kernel used by the GPU tests, not by the hot path. */
int tg_conv_simt(const tg_conv_desc* d, void* stream);

/* ------------------------------------------------------------------------
 * SRNet tail in one launch: last nn.ConvTranspose2d(64,64,3,2,1,op=1) + ReLU -> conv_out (64 -> out_nc)
 * -> + upsample_func(lr_curr) (tecogan_nets.py:119-131,143-145), optionally also float32_to_uint8 +
 * CHW->HWC (data_utils.py:80-87, tecogan_nets.py:278-281).  The 64-channel HR map only exists as one
 * 32x16-pixel tile in shared memory (four parity blocks, used directly as conv_out's wgmma operand)
 * instead of a round trip through HBM.  No allocation, no synchronisation.
 * ---------------------------------------------------------------------- */
typedef struct tg_tail_desc {
  const void* x;        /* input of the transposed conv, NHWC fp16 [n,h,w,64]                       */
  const void* w_up;     /* tg_pack_convT3x3s2_weights(cout_pad=64, cin_pad=64)                      */
  const float* b_up;    /* fp32 [64]                                                                */
  const void* w_out;    /* tg_pack_tail_out_weights                                                 */
  const float* b_out;   /* fp32 [cout_real]                                                         */
  const float* lr;      /* lr_curr NCHW fp32 [n,cout_real,2h/lr_scale,2w/lr_scale] or NULL: the residual is
                           evaluated inside the kernel (16 gathers per pixel pair and channel)          */
  float* y;             /* NCHW fp32 [n,cout_real,2h,2w]; accumulate != 0: read-modify-write             */
  uint8_t* y_u8;        /* NHWC uint8 [n,2h,2w,cout_real] (round-half-even, clip) or NULL           */
  int32_t n, h, w;      /* of the transposed conv's input                                           */
  int32_t cout_real;    /* 1..3                                                                     */
  int32_t lr_scale;     /* 2 or 4: output size / lr size                                            */
  int32_t up_mode;      /* TG_UP_*                                                                  */
  int32_t max_ctas;     /* 0 = one persistent CTA per SM                                            */
  int32_t accumulate;   /* != 0: y already holds upsample_func(lr_curr) (tg_upsample_nchw_f32): out = y + conv +
                           bias -- one coalesced read per pixel instead of the in-kernel gathers (lr must be NULL) */
  int32_t reserved;     /* must be 0                                                                */
} tg_tail_desc;
int tg_convT_convout_tcgen05(const tg_tail_desc* d, void* stream);
/* conv_out's weights (nn.Conv2d(cin <= 64, cout <= 3, 3, 1, 1).weight, fp32) as the tail reads them: one
 * [TG_TAIL_OUT_ROWS rows][64 k] tile (TG_TAIL_OUT_ROWS * 128 bytes), tap t of output channel co in row
 * 8*(t>>1) + 2*co + (t&1), so that one thread of the tail's conv_out holds all nine taps of one channel. */
int tg_pack_tail_out_weights(const float* w_oihw, int cout, int cin, void* packed, void* stream);

/* ------------------------------------------------------------------------
 * Fused  backward_warp + space_to_depth + concat  (HBM-bound).
 * Replaces net_utils.backward_warp (net_utils.py:50-82), space_to_depth
 * (:36-47) and torch.cat([lr_curr, hr_prev_tran]) (tecogan_nets.py:141).
 * out NHWC fp16 [n,h,w,cpad]: ch [0,c) = lr_curr, ch c+(sy*s+sx)*c+k =
 * warp(hr_prev)[k, y*s+sy, x*s+sx], remaining channels zero.
 * ---------------------------------------------------------------------- */
/* flow given at HR: hr_flow NCHW fp32 [n,2,s*h,s*w] (FRNet.forward_sequence, :201-212) */
int tg_warp_s2d_concat_hrflow(const float* hr_prev, const float* hr_flow, const float* lr_curr,
                              void* out, int n, int c, int h, int w, int s, int cpad,
                              void* stream);
/* flow given at LR: lr_flow NCHW fp32 [n,2,h8,w8]; reflect pad to (h,w) (:239-241),
 * upsample_func and the *scale (:244) are evaluated inline (FRNet.step, :227-252) */
int tg_warp_s2d_concat_lrflow(const float* hr_prev, const float* lr_flow, const float* lr_curr,
                              void* out, int n, int c, int h, int w, int h8, int w8, int s,
                              int up_mode, int cpad, void* stream);

/* ------------------------------------------------------------------------
 * Small NHWC fp16 helpers of FNet (tecogan_nets.py:28,35,42 and :74-79)
 * ---------------------------------------------------------------------- */
int tg_maxpool2x2_nhwc_f16(const void* x, void* y, int n, int h, int w, int c, void* stream);
int tg_upsample2x_bilinear_nhwc_f16(const void* x, void* y, int n, int h, int w, int c,
                                    void* stream);
/* cat([x1,x2],1) (tecogan_nets.py:71) + NCHW fp32 -> NHWC fp16, zero padded to cpad */
int tg_pack_pair_nhwc_f16(const float* x1, const float* x2, void* y, int n, int c, int h, int w,
                          int cpad, void* stream);

/* ------------------------------------------------------------------------
 * Module-boundary ops on NCHW fp32 (drop-in for codes/utils/net_utils.py)
 * ---------------------------------------------------------------------- */
int tg_backward_warp_nchw_f32(const float* x, const float* flow, float* y, int n, int c, int h,
                              int w, void* stream);                      /* net_utils.py:50-82  */
int tg_space_to_depth_nchw_f32(const float* x, float* y, int n, int c, int h, int w, int s,
                               void* stream);                            /* net_utils.py:36-47  */
/* y = [y +] mul * upsample(reflect_pad(x -> (h,w)))  ; x [n,c,hin,win], hin<=h, win<=w;
 * accumulate != 0 adds into y (fp32).
 * up_mode bicubic = BicubicUpsampler (net_utils.py:101-156), bilinear = F.interpolate
 * (net_utils.py:87-89).  hin==h, win==w, mul==1 gives the plain upsample_func. */
int tg_upsample_nchw_f32(const float* x, float* y, int n, int c, int hin, int win, int h, int w,
                         int s, int up_mode, float mul, int accumulate, void* stream);
int tg_nchw_f32_to_nhwc_f16(const float* x, void* y, int n, int c, int h, int w, int cpad,
                            int c_offset, void* stream);
int tg_nhwc_f16_to_nchw_f32(const void* x, float* y, int n, int c, int h, int w, int cpad,
                            void* stream);
/* float32_to_uint8 (data_utils.py:80-87) + CHW->HWC (tecogan_nets.py:281):
 * x NCHW fp32 [n,c,h,w] -> uint8 [n,h,w,c], round-half-even, clip [0,255] */
int tg_float_to_uint8_nhwc(const float* x, uint8_t* y, int n, int c, int h, int w, void* stream);
/* The same, written as the h x w picture at `win` of each uint8 HWC frame y [n, frame_h, frame_w, c]
 * (struct tg_frame_window, declared with the stream's frame I/O below); nothing outside the picture is written. */
struct tg_frame_window;
int tg_float_to_uint8_nhwc_window(const float* x, uint8_t* y, const struct tg_frame_window* win, int n, int c, int h,
                                  int w, void* stream);

/* Frame input of one streamed step (codes/data/paired_folder_dataset.py:49, tecogan_nets.py:269-276).
 * in_u8 : uint8 [n,h,w,c] HWC frames, or NULL (lr_curr was filled by the caller)
 *         -> lr_curr fp32 NCHW [n,c,h,w] = float(v) / 255 (IEEE division, == numpy float32 / 255.0);
 *            bgr != 0 reverses the channel order (cv2's BGR -> the reference's RGB)
 * reset : int32 [n] in device memory, or NULL; slot k with reset[k] != 0 starts a new video:
 *         lr_prev[k] and hr_prev[k] (fp32, [c,h,w] / [c,s*h,s*w]) are zeroed, as the reference's
 *         infer_sequence does for frame 0 (tecogan_nets.py:269-270); other slots are not touched
 * lr_curr, lr_prev and hr_prev must be non-NULL and 4-byte aligned; c <= 4; s in {2,4}.  The mask is read
 * on the device, so one captured launch serves every pattern of resets. */
int tg_stream_frame_in(const uint8_t* in_u8, const int32_t* reset, float* lr_curr, float* lr_prev,
                       float* hr_prev, int n, int c, int h, int w, int s, int bgr, void* stream);
/* Step input of a temporally padded stream, assembled from a ring of decoded frames (FRNet.stream(pad_front=p)).
 * ring   : fp32 [depth, n, c, h, w], frames decoded ahead of the step (tg_stream_frame_in into ring positions)
 * table  : int32 [3n] in device memory, read on the device (one captured launch serves every schedule):
 *          cur[k] = table[k], mode[k] = table[n + k], prev[k] = table[2n + k]
 *   cur[k] in [0, depth): lr_curr[k] = ring[cur[k]][k]; any other value leaves lr_curr[k] untouched
 *   mode[k] == TG_GATHER_ZERO: lr_prev[k] = hr_prev[k] = 0 (tg_stream_frame_in's reset)
 *   mode[k] == TG_GATHER_LOAD: lr_prev[k] = ring[prev[k]][k] (0 when prev[k] lies outside [0, depth)) and
 *                              hr_prev[k] = warm_hr[k]; with warm_hr NULL the slot is kept
 *   any other mode (TG_GATHER_KEEP): lr_prev[k] and hr_prev[k] are not touched (one read of mode[k])
 * warm_hr: fp32 [n, c, s*h, s*w] (the warm-up steps' HR state), or NULL.  The outputs must not overlap the ring or
 * warm_hr.  Exact copies: no arithmetic, so the result does not depend on the grid.  Pointers 4-byte aligned; 16-byte
 * vectors wherever source and destination share their alignment.
 * TG_E_INVALID: null pointers (warm_hr aside), non-positive sizes, misalignment; TG_E_UNSUPPORTED: s not 2 or 4, a
 * grid too large. */
#define TG_GATHER_KEEP 0
#define TG_GATHER_ZERO 1
#define TG_GATHER_LOAD 2
int tg_stream_gather(const float* ring, int depth, const int32_t* table, const float* warm_hr, float* lr_curr,
                     float* lr_prev, float* hr_prev, int n, int c, int h, int w, int s, void* stream);
/* The same step input from YUV 4:2:0 frames, as video decoders produce them (BT.601 limited range).
 * in    : uint8 [n, 3h/2, w], each frame the h x w Y plane followed by the interleaved (h/2) x w UV plane
 *         (nv12 != 0) or by the (h/2) x (w/2) U and V planes (nv12 == 0: I420 / yuv420p), or NULL
 *         -> lr_curr fp32 NCHW [n,3,h,w] = float(rgb) / 255 with rgb = cv2.cvtColor(frame, COLOR_YUV2RGB_NV12 /
 *            COLOR_YUV2RGB_I420) bit for bit (20-bit fixed point, nearest chroma)
 * reset : as above.  h and w must be even (TG_E_UNSUPPORTED otherwise). */
int tg_stream_frame_in_yuv420(const uint8_t* in, int nv12, const int32_t* reset, float* lr_curr, float* lr_prev,
                              float* hr_prev, int n, int h, int w, int s, void* stream);
/* Encode of the streamed output: rgb uint8 NHWC [n,H,W,3] (the step's out_u8) -> out uint8 [n, 3H/2, W] in
 * NV12 (nv12 != 0) or I420, the layouts above; == cv2.cvtColor(rgb, COLOR_RGB2YUV_I420) bit for bit (U and V
 * of each 2x2 block from its top-left pixel), NV12 with the U and V planes interleaved.  H and W must be even. */
int tg_rgb_u8_to_yuv420(const uint8_t* rgb, uint8_t* out, int nv12, int n, int H, int W, void* stream);

/* YUV frame I/O (4:2:0, 4:2:2, 4:4:4) in any supported layout and colour.
 * layout : TG_YUV_NV12 / TG_YUV_I420 (uint8 words, as above), TG_YUV_P010 (NV12 planes, uint16 words, sample in the
 *          high 10 bits: v << 6; NVDEC / NVENC, ffmpeg p010le), TG_YUV_I420_10 (I420 planes, uint16 words, sample in
 *          the low 10 bits; ffmpeg yuv420p10le).  Frames are [n, 3h/2, w] words; 10-bit frames 2-byte aligned.
 * matrix : 601 (Kr, Kb = 0.299, 0.114) or 709 (0.2126, 0.0722); full_range 0 = limited ("tv"), 1 = full ("pc")
 *          quantisation of ITU-T H.273 at the layout's bit depth; reserved must be 0.
 *          4:2:2 and 4:4:4 (h of any parity):
 *          TG_YUV_YUY2 / TG_YUV_UYVY: packed 4:2:2, uint8 frames [n, h, 2w] (w even; V4L2 YUYV, SDI "2vuy"), each
 *            pixel pair one 4-byte group Y0 U Y1 V (YUY2) or U Y0 V Y1 (UYVY); frames and output 4-byte aligned.
 *          TG_YUV_I444: planar 4:4:4, uint8 frames [n, 3h, w] (the Y, U, V planes of h x w; ffmpeg yuv444p).
 *          TG_YUV_I444_10: as I444 in uint16 words [n, 3h, w], sample in the low 10 bits (ffmpeg yuv444p10le).
 *          Value 7 is not a layout (it stays an unknown one).  oracle/yuv_422_444.py specifies these four.
 * matrix : 601 (Kr, Kb = 0.299, 0.114) or 709 (0.2126, 0.0722); full_range 0 = limited ("tv"), 1 = full ("pc")
 *          quantisation of ITU-T H.273 at the layout's bit depth; reserved must be 0.
 * The fixed-point matrices are tg_yuv_coefficients' table (oracle/yuv_color.py derives the same numbers); matrix
 * 601, limited range, 8 bit is cv2's BT.601 and gives the bytes of the two entry points above.  Decode uses nearest
 * chroma (both pixels of a 4:2:2 pair take its U and V).  The 4:2:2 encode takes U and V of the pair's mean,
 * rounded half up: C = (c . (rgb0 + rgb1) + 2^(s-1) + (128 << s)) >> s with the table row's coefficients and
 * s = 21, except for 601 / limited, where it is cv2's COLOR_RGB2YUV_YUY2 / _UYVY bit for bit, luma included:
 * Y = ((4211 R + 8258 G + 1606 B + 8192) >> 14) + 16, U = ((-1212 SR - 2384 SG + 3596 SB + 8192) >> 14) + 128,
 * V = ((3596 SR - 3015 SG - 582 SB + 8192) >> 14) + 128 with SR = R0 + R1 and so on.
 *
 * 10-bit 4:2:2 (h of any parity, w even; oracle/yuv_422_10.py specifies these three):
 *          TG_YUV_P210: uint16 frames [n, 2h, w], the h x w Y plane then a full-height interleaved UV plane
 *            (U0 V0 U1 V1 ... per row, one (U, V) per pixel pair), each sample in the high 10 bits (v << 6), as P010.
 *          TG_YUV_I422_10: uint16 frames [n, 2h, w], the Y plane then the U and V planes of h x w/2, each sample in
 *            the low 10 bits, read as min(v, 1023) (ffmpeg yuv422p10le).
 *          TG_YUV_V210: uint8 frames [n, h, S], S = 128 * ceil(w / 48) bytes a row (SDI capture / playout, ffmpeg
 *            v210).  Each 16-byte group holds 6 pixels as four little-endian 32-bit words
 *              Cb0 Y0 Cr0 | Y1 Cb2 Y2 | Cr2 Y3 Cb4 | Y4 Cr4 Y5
 *            with the 10-bit fields at bits 0, 10 and 20 and bits 30-31 zero.  Row r starts at byte r * S; the
 *            ceil(w / 6) groups of a row hold its pixels, the fields past pixel w - 1 of a partial last group and
 *            the row padding up to S are 0 in encoded frames (ignored on decode).  Frames and output 16-byte aligned.
 *            A v210 window's picture starts on a group (left % 6 == 0) and ends on one unless it reaches the frame's
 *            right edge; a windowed encode writes its picture's groups only, a whole-frame encode every byte of
 *            each row.  The frame width is not implied by S: every call passes it (w or frame_w).
 *          Decode: the 10-bit row per pixel, nearest chroma.  Encode from rgb_f32 (10 bit): Y per pixel as
 *          I444_10, C = clip((c . (q0 + q1) + 2^18 + (512 << 19)) >> 19) from the pair's sum of 10-bit codes (the
 *          10-bit row's coefficients, one more fraction bit). */
enum { TG_YUV_NV12 = 0, TG_YUV_I420 = 1, TG_YUV_P010 = 2, TG_YUV_I420_10 = 3, TG_YUV_YUY2 = 4, TG_YUV_UYVY = 5,
       TG_YUV_I444 = 6, TG_YUV_I444_10 = 8 };
enum { TG_YUV_P210 = 9, TG_YUV_I422_10 = 10, TG_YUV_V210 = 11 };
typedef struct tg_yuv_format {
  int32_t layout;       /* TG_YUV_*                   */
  int32_t matrix;       /* 601 or 709                 */
  int32_t full_range;   /* 0 limited, 1 full          */
  int32_t reserved;     /* must be 0                  */
} tg_yuv_format;
/* tg_stream_frame_in_yuv420 for any format: lr_curr = float(rgb) / 255 (8 bit) or / 1023 (10 bit, P010 read as
 * v >> 6, I420_10 and I444_10 as min(v, 1023)), rgb decoded with nearest chroma; reset as in tg_stream_frame_in. */
int tg_stream_frame_in_yuv(const void* in, const tg_yuv_format* fmt, const int32_t* reset, float* lr_curr,
                           float* lr_prev, float* hr_prev, int n, int h, int w, int s, void* stream);
/* Encode of the streamed output into any format.  8-bit layouts read rgb_u8 (uint8 NHWC [n,H,W,3], the step's
 * out_u8; rgb_f32 must be NULL), 10-bit layouts read rgb_f32 (fp32 NCHW [n,3,H,W], the step's HR frame, quantised as
 * clip(rint(x * 1023), 0, 1023); rgb_u8 must be NULL).  4:2:0: chroma of each 2x2 block from its top-left pixel;
 * 4:2:2: of each pixel pair's mean (above); 4:4:4: per pixel.  Output [n, 3H/2, W], [n, H, 2W] or [n, 3H, W] words;
 * P210 / I422_10 [n, 2H, W] uint16 and v210 [n, H, 128 * ceil(W / 48)] bytes, all three from rgb_f32.
 * TG_E_INVALID: null pointers, the wrong source for the bit depth, a non-zero reserved, misaligned buffers;
 * TG_E_UNSUPPORTED: odd sizes (H and W for 4:2:0, W for 4:2:2), unknown layout or matrix. */
int tg_rgb_to_yuv(const uint8_t* rgb_u8, const float* rgb_f32, void* out, const tg_yuv_format* fmt, int n, int H,
                  int W, void* stream);
/* Host only: the 16 int32 of the kernels' table row for fmt (its bit depth and colour): encode cRY cGY cBY cRU cGU
 * cBU cRV cGV cBV, decode CY CUB CUG CVG CVR, then the fraction bits and the luma offset. */
int tg_yuv_coefficients(const tg_yuv_format* fmt, int32_t* out16);

/* A picture inside a stored frame: the frames in memory are frame_h x frame_w pixels in their layout (a uint8 HWC
 * frame [frame_h, frame_w, c], or that layout's YUV words of a frame_h x frame_w frame), and the picture is the
 * h x w pixels at row `top`, column `left`.  The plain entry points are the window {h, w, 0, 0}.  Used on the input
 * side (crop a letterboxed picture out of its frame; read a decoder surface of pitch P words and R rows as a frame
 * of R x P) and on the output side (put the picture into a larger, black-padded delivery frame).  Only the picture
 * is read or written.
 * TG_E_INVALID: a NULL window, a frame of non-positive size, a picture outside the frame;
 * TG_E_UNSUPPORTED: a window off the layout's chroma grid (4:2:0: frame_h, frame_w, top and left even; 4:2:2:
 * frame_w and left even; v210 in addition left % 6 == 0 and left + w % 6 == 0 or left + w == frame_w). */
typedef struct tg_frame_window {
  int32_t frame_h, frame_w;   /* the stored frame, in pixels */
  int32_t top, left;          /* the picture's first row and column in it */
} tg_frame_window;
/* tg_stream_frame_in / tg_stream_frame_in_yuv reading the h x w picture at `win` of each stored frame (in_u8 / in
 * point at the first frame; frames follow each other at the frame's size).  lr_curr, lr_prev, hr_prev, reset and the
 * other arguments are those of the picture, as in the plain entry points. */
int tg_stream_frame_in_window(const uint8_t* in_u8, const tg_frame_window* win, const int32_t* reset, float* lr_curr,
                              float* lr_prev, float* hr_prev, int n, int c, int h, int w, int s, int bgr,
                              void* stream);
int tg_stream_frame_in_yuv_window(const void* in, const tg_yuv_format* fmt, const tg_frame_window* win,
                                  const int32_t* reset, float* lr_curr, float* lr_prev, float* hr_prev, int n, int h,
                                  int w, int s, void* stream);
/* tg_rgb_to_yuv writing the encoded H x W picture at `win` of each output frame (out [n, frame words]).  The words
 * outside the picture are not touched: fill them once with tg_fill_black. */
int tg_rgb_to_yuv_window(const uint8_t* rgb_u8, const float* rgb_f32, void* out, const tg_yuv_format* fmt,
                         const tg_frame_window* win, int n, int H, int W, void* stream);
/* Every word of n frames of frame_h x frame_w set to the format's black: fmt NULL -> uint8 HWC [n,frame_h,frame_w,c]
 * all 0; else the YUV layout's frames (c must be 3) with Y = the luma offset of the colour (16 << (depth - 8) for
 * limited range, 0 for full) and U = V = 128 << (depth - 8), stored as the layout stores samples (P010: << 6).
 * TG_E_INVALID: null pointers, non-positive sizes, misalignment; TG_E_UNSUPPORTED: sizes off the chroma grid. */
int tg_fill_black(void* out, const tg_yuv_format* fmt, int n, int c, int frame_h, int frame_w, void* stream);
/* Per-row and per-column sums of the 8-bit luma of n frames of h x w: Y for YUV frames (10-bit samples >> 2), and
 * for uint8 HWC RGB frames (fmt NULL, c == 3; bgr != 0 for BGR order) the gray of tg_metrics_frames_in,
 * (9798 R + 19235 G + 3735 B + 16384) >> 15.  rows uint64 [n,h], cols uint64 [n,w], zeroed by the call (memsets on
 * the stream), 8-byte aligned.  Exact integers: the result does not depend on the grid.  detect_bars' input. */
int tg_luma_line_sums(const void* in, const tg_yuv_format* fmt, int bgr, int n, int c, int h, int w,
                      unsigned long long* rows, unsigned long long* cols, void* stream);

/* Resize of the streamed output: Pillow's antialiased bicubic (a = -0.5, support 2) or Lanczos-3 (support 3)
 * filters, as Image.resize on 'F' images (oracle/resample.py restates them).  A downscale widens the filter by the
 * ratio.  Each axis needs in/4 <= out <= 2*in, so an axis has at most 17 (bicubic) or 25 (Lanczos) taps.
 * Per axis the kernel reads a caller-owned table: first[out] int32 (window start) and weights[out * taps] fp32 (the
 * window's normalised weights, zero for padding taps).  The window ends inside the axis where it fits: first =
 * max(0, min(xmin, in - taps)); on an axis shorter than taps the kernel clamps the index. */
enum { TG_RESAMPLE_BICUBIC = 0, TG_RESAMPLE_LANCZOS3 = 1 };
/* Host only: *taps = 2 * ceil(support * max(in / out, 1)) + 1.  TG_E_INVALID: null taps, non-positive sizes;
 * TG_E_UNSUPPORTED: unknown filter, ratio outside [1/4, 2]. */
int tg_resample_taps(int in, int out, int filter, int* taps);
/* Host only: fills first[out] and weights[out * taps] (host memory; float64 weights rounded to fp32).  taps must be
 * tg_resample_taps' value (TG_E_INVALID otherwise); other errors as tg_resample_taps. */
int tg_resample_table(int in, int out, int filter, int taps, int32_t* first, float* weights);
/* x fp32 NCHW [n,c,H,W] (the step's HR frame) -> exactly one of
 *   y_u8  uint8 NHWC [n,Ho,Wo,c] = clip(rint(y * 255), 0, 255), round half to even (float32_to_uint8), or
 *   y_f32 fp32 NCHW [n,c,Ho,Wo].
 * Vertical pass (row tables, H -> Ho) then horizontal (column tables, W -> Wo), fp32 sums in tap order: the result
 * does not depend on the grid.  Tables in device memory; x, the tables and y_f32 4-byte aligned.
 * TG_E_INVALID: null pointers, both or neither output, non-positive sizes or taps, c > 4, misalignment;
 * TG_E_UNSUPPORTED: a ratio outside [1/4, 2] on either axis, taps above 25, a grid too large. */
int tg_resample_nchw_f32(const float* x, int n, int c, int H, int W, const int32_t* row_first, const float* row_w,
                         int row_taps, const int32_t* col_first, const float* col_w, int col_taps, int Ho, int Wo,
                         uint8_t* y_u8, float* y_f32, void* stream);
/* tg_resample_nchw_f32 with the uint8 output written as the Ho x Wo picture at `win` of each uint8 HWC frame
 * y_u8 [n, frame_h, frame_w, c] (tg_frame_window above); nothing outside the picture is written. */
int tg_resample_nchw_f32_window(const float* x, int n, int c, int H, int W, const int32_t* row_first,
                                const float* row_w, int row_taps, const int32_t* col_first, const float* col_w,
                                int col_taps, int Ho, int Wo, uint8_t* y_u8, const tg_frame_window* win,
                                void* stream);
/* Frame input of a streamed step at another LR size: the h x w source picture resized to hn x wn in one launch.
 * in    : the source frames, uint8 HWC [n, frame_h, frame_w, c] (fmt NULL; bgr != 0 reverses the channel order) or
 *         any tg_yuv_format layout and colour (c must be 3, bgr 0), read through `win` as tg_stream_frame_in_window /
 *         tg_stream_frame_in_yuv_window read them (NULL: the whole h x w frame)
 *      -> lr_curr fp32 NCHW [n,c,hn,wn] = the resize (tg_resample_nchw_f32, fp32 output) of the fp32 picture those
 *         entry points would write, with the row tables (h -> hn) and the column tables (w -> wn) of
 *         tg_resample_table, bit for bit: the same decode per source pixel and the same fmaf sums in tap order.
 *         Nothing is re-quantised, and no source-size fp32 frame exists.
 * reset : int32 [n] in device memory, or NULL: lr_prev[k] ([c,hn,wn]) and hr_prev[k] ([c,s*hn,s*wn]) of the flagged
 *         slots are zeroed in the same launch, as tg_stream_frame_in does.
 * Each axis needs in/4 <= out <= 2*in, and its table's taps must be the bicubic or the Lanczos-3 count of that axis
 * (tg_resample_taps).  Tables in device memory, 4-byte aligned like the fp32 buffers.
 * TG_E_INVALID: null pointers (reset aside; in too), non-positive sizes, misalignment, c != 3 or bgr with a YUV
 * format, a non-zero reserved, a picture outside its frame, tap counts that do not belong to the sizes;
 * TG_E_UNSUPPORTED: c > 4, s not 2 or 4, odd sizes or windows off the layout's chroma grid, an unknown layout or
 * matrix, a ratio outside [1/4, 2], a grid too large. */
int tg_stream_frame_in_resample(const void* in, const tg_yuv_format* fmt, int bgr, const tg_frame_window* win, int h,
                                int w, const int32_t* row_first, const float* row_w, int row_taps,
                                const int32_t* col_first, const float* col_w, int col_taps, const int32_t* reset,
                                float* lr_curr, float* lr_prev, float* hr_prev, int n, int c, int hn, int wn, int s,
                                void* stream);

/* Scene-cut detection of a streamed step (oracle/scene_cut.py is the specification).  Per slot k, with a = lr_curr[k]
 * and b = lr_prev[k] (fp32 [c,h,w], as the step sees them: decoded, and zeroed by a reset of this step):
 *   q(x) = clip(rint(x * 255), 0, 255) (fp32 product, round half to even; NaN counts as 0),
 *   SAD  = sum |q(a) - q(b)| (exact integer), mafd = float64(SAD) * 100 / (c*h*w) / 255 (float64, in that order);
 *   reset[k] != 0     : score 0, cut 0, prev_mafd[k] = -1
 *   prev_mafd[k] < 0  : score 0, cut 0, prev_mafd[k] = mafd
 *   otherwise         : score = min(max(min(mafd, |mafd - prev_mafd[k]|), 0), 100), cut = score >= threshold,
 *                       prev_mafd[k] = cut ? -1 : mafd.
 * score[n] (float64) and cut[n] (int32 0 / 1) are written for every slot on every launch; with cut as the reset mask
 * of tg_stream_frame_in (in_u8 = NULL) a detected cut restarts the slot exactly as a reset at that frame would.
 * reset : int32 [n] in device memory (tg_stream_frame_in's mask), or NULL (no caller resets).
 * work  : caller-owned device workspace of n * TG_SCENE_CUT_WORK_BYTES bytes, zeroed once by the caller; every launch
 *         leaves it zeroed again, so a captured launch replays without a memset.
 * Every sum is an integer, so the result does not depend on the grid.  lr_curr, lr_prev, reset and cut 4-byte aligned;
 * prev_mafd, work and score 8-byte aligned.
 * TG_E_INVALID: null pointers (reset aside), non-positive sizes, misalignment, a threshold that is not finite or lies
 * outside (0, 100]; TG_E_UNSUPPORTED: c > 4, a grid too large. */
#define TG_SCENE_CUT_WORK_BYTES 16
int tg_scene_cut(const float* lr_curr, const float* lr_prev, int n, int c, int h, int w, const int32_t* reset,
                 double threshold, double* prev_mafd, void* work, double* score, int32_t* cut, void* stream);

/* ------------------------------------------------------------------------
 * Video quality metrics: PSNR and tOF as TecoGAN's MetricCalculator computes them (oracle/metrics_oracle.py and
 * oracle/farneback.py are the specification).
 * ---------------------------------------------------------------------- */
enum { TG_PSNR_NONE = 0, TG_PSNR_RGB = 1, TG_PSNR_Y = 2 };
/* One read of t uint8 RGB frames true_u8 [t,ht,wt,3] and pred_u8 [t,hp,wp,3], both cropped to h = min(ht, hp),
 * w = min(wt, wp) (their top-left corner):
 *   gray [2,t,h,w] uint8 (true then pred) = (9798 R + 19235 G + 3735 B + 16384) >> 15, cv2 COLOR_RGB2GRAY bit for
 *        bit; NULL when not wanted.  With pred_u8 NULL (psnr TG_PSNR_NONE) only the true frames: gray [t,ht,wt].
 *   sse  [t] uint64 = the exact integer sum of squared differences per frame over R, G, B (TG_PSNR_RGB) or over the
 *        Y of data_utils.rgb_to_ycbcr (TG_PSNR_Y: float64 r*T0 + g*T1 + b*T2 + 16 left to right without FMA, rounded
 *        half to even, and one lower for the three colours (1,173,225), (12,174,191), (24,46,73) whose numpy matmul
 *        rounds the other way).  Zeroed by the call (a memset on the stream); NULL exactly when psnr is
 *        TG_PSNR_NONE.  PSNR = 20 log10(255 / sqrt(sse / count)) then equals the reference's numpy result.
 * TG_E_INVALID: null true frames, non-positive sizes, bad psnr mode, sse given or missing against the mode, nothing
 * requested, sse not 8-byte aligned; TG_E_UNSUPPORTED: t > 65535. */
int tg_metrics_frames_in(const uint8_t* true_u8, int ht, int wt, const uint8_t* pred_u8, int hp, int wp, int t,
                         int psnr, uint8_t* gray, unsigned long long* sse, void* stream);

/* Farneback dense optical flow, cv2.calcOpticalFlowFarneback(prev, next, None, pyr_scale, levels, winsize,
 * iterations, poly_n, poly_sigma, flags=0), in fp32.  (pyr_scale, poly_sigma float64.) */
typedef struct tg_farneback_params {
  double pyr_scale;     /* (0, 1) */
  int32_t levels;       /* >= 0 */
  int32_t winsize;      /* box window, [1, 63] */
  int32_t iterations;   /* >= 1 */
  int32_t poly_n;       /* 5 or 7 */
  double poly_sigma;    /* > 0 */
  int32_t flags;        /* 0: OPTFLOW_USE_INITIAL_FLOW and OPTFLOW_FARNEBACK_GAUSSIAN are not implemented */
  int32_t reserved;
} tg_farneback_params;
/* Bytes of the workspace of tg_farneback for `groups` groups of t frames of h x w (0 for bad sizes). */
size_t tg_farneback_workspace_bytes(int groups, int t, int h, int w);
/* gray uint8 [groups * t, h, w]: every group of t consecutive frames gives the t - 1 flows of its consecutive pairs,
 * flow[g (t-1) + j] = farneback(gray[g t + j], gray[g t + j + 1]), fp32 [groups * (t-1), h, w, 2] (dx, dy).  Each
 * frame's polynomial expansion is computed once per pyramid level however many pairs use it.  Per level: blur +
 * resize (2 launches), polynomial expansion (2), the level's first flow and matrices (1), then one launch per
 * iteration (box mean + solve + matrix update on 32 x 16 tiles with a winsize/2 halo).  flow and work 16-byte
 * aligned; work_bytes >= tg_farneback_workspace_bytes.  The result does not depend on the grid.
 * TG_E_INVALID: null pointers, bad sizes (t < 2), bad parameters, misalignment, a short workspace;
 * TG_E_UNSUPPORTED: frames below 2 x 2, more than 65535 frames, a coarsest blur above 63 taps. */
int tg_farneback(const uint8_t* gray, int groups, int t, int h, int w, const tg_farneback_params* params,
                 float* flow, void* work, size_t work_bytes, void* stream);
/* sums[q] = sum over the h*w pixels of |a[q] - b[q]| (the end-point error of two fp32 flows [n,h,w,2]), accumulated
 * in float64; sums is zeroed by the call.  a, b and sums 8-byte aligned.  TG_E_INVALID: null pointers, non-positive
 * sizes, misalignment; TG_E_UNSUPPORTED: n > 65535. */
int tg_flow_epe_sum(const float* a, const float* b, int n, int h, int w, double* sums, void* stream);
/* Bytes of tg_flow_epe_sum_window's workspace for n pairs and a window of hc rows (0 for bad sizes). */
size_t tg_flow_epe_sum_window_workspace_bytes(int n, int hc);
/* tg_flow_epe_sum over the window rows y0 .. y0+hc-1, columns x0 .. x0+wc-1 of the h x w flows, with the per-CTA
 * sums added in a fixed order through the workspace (work 8-byte aligned, work_bytes >=
 * tg_flow_epe_sum_window_workspace_bytes): the same inputs give the same bits.  tg_flow_epe_sum is the same kernel
 * over the whole frame with float64 atomics in place of the workspace.  TG_E_INVALID also for a window outside the
 * flows, a null or short workspace. */
int tg_flow_epe_sum_window(const float* a, const float* b, int n, int h, int w, int y0, int x0, int hc, int wc,
                           double* sums, void* work, size_t work_bytes, void* stream);

/* The official metric script (codes/official_metrics/metrics.py, oracle/official_metrics.py) scores the Y of
 * _rgb2ycbcr, Y = float64 r*T0 + g*T1 + b*T2 + 16 left to right without FMA and without rounding, over the window
 * rows y0 .. y0+hc-1, columns x0 .. x0+wc-1 of t pairs of uint8 RGB frames true_u8 [t,ht,wt,3] / pred_u8
 * [t,hp,wp,3].  The window lies in the common size min(ht, hp) x min(wt, wp) (the frames' top-left corner).
 * Sums are reduced in a fixed order through the caller's workspace: the same inputs give the same bits.
 * TG_E_INVALID: null or misaligned (8 bytes) pointers, non-positive sizes, a window outside the common size, a short
 * workspace; TG_E_UNSUPPORTED: t > 65535.  Two launches each. */
size_t tg_official_frames_stats_workspace_bytes(int t, int hc, int wc);
/* stats [t,3] float64 = {sum over the window of (Yt - Yp)^2, min Yp, max Yp} per frame. */
int tg_official_frames_stats(const uint8_t* true_u8, int ht, int wt, const uint8_t* pred_u8, int hp, int wp, int t,
                             int y0, int x0, int hc, int wc, double* stats, void* work, size_t work_bytes,
                             void* stream);
/* Bytes of tg_ssim_y's workspace (0 for bad sizes or a window below 7 x 7). */
size_t tg_ssim_y_workspace_bytes(int t, int hc, int wc);
/* ssim [t] float64 = skimage.measure.compare_ssim(Yt, Yp, data_range=R) of the window: 7x7 box means of Yt, Yp,
 * Yt^2, Yp^2, Yt Yp, covariances scaled by 49/48, C1 = (0.01 R)^2, C2 = (0.03 R)^2, and the mean of the SSIM map
 * over the (hc-6) x (wc-6) windows inside the crop.  R = stats[3f+2] - stats[3f+1] (tg_official_frames_stats's
 * output, read on the device).  Plain IEEE division: R = 0 gives numpy's nan where a 7x7 window is flat in both
 * frames.  TG_E_INVALID also for a window below 7 x 7. */
int tg_ssim_y(const uint8_t* true_u8, int ht, int wt, const uint8_t* pred_u8, int hp, int wp, int t, int y0, int x0,
              int hc, int wc, const double* stats, double* ssim, void* work, size_t work_bytes, void* stream);

/* ------------------------------------------------------------------------
 * LPIPS (net-lin, AlexNet, v0.1) as both of TecoGAN's copies compute it (codes/metrics/LPIPS,
 * codes/official_metrics/LPIPSmodels; oracle/lpips.py is the specification of every layout below).  AlexNet's five
 * convs run on tg_conv_tcgen05 as pad-1 3x3 convs:
 *   conv1 (11x11, stride 4, pad 2, 3 -> 64): a 3x3 conv over the space-to-depth(4) picture, zero-padded by 2 at the
 *         top and left, on an (oh+2) x (ow+2) grid (oh = (h-7)/4 + 1, ow likewise) with cin = 64, cin_real = 48
 *         (channel (py*4 + px)*3 + c) and the 11x11 kernel zero-padded to 12x12 and split the same way; its output
 *         is the grid's interior at (1, 1).
 *   conv2 (5x5, pad 2, 64 -> 192): a 3x3 conv over four copies of the pooled map (cin = 256, copy b = (by, bx)
 *         shifted by (3by - 1, 3bx - 1), zero fill) with the kernel padded to 6x6 and split into four 3x3 blocks, on
 *         a (ph+2) x (pw+2) grid; its output is the interior at (1, 1).
 *   conv3 .. conv5 (192 -> 384 -> 256 -> 256): plain pad-1 3x3 convs.
 * Each layer's feature (after its ReLU) feeds a head; a picture needs at least TG_LPIPS_MIN_SIDE pixels per side.
 * ---------------------------------------------------------------------- */
#define TG_LPIPS_MIN_SIDE 31   /* below it the second pool is empty */
enum { TG_LPIPS_NORM_CALC = 0,      /* MetricCalculator: float32 x * 2 / 255 - 1 */
       TG_LPIPS_NORM_OFFICIAL = 1   /* the official script's util.im2tensor: float64 x / 127.5 - 1, then float32 */ };
/* t uint8 RGB frames [t, frame_h, frame_w, 3] read through `win` (the h x w picture at (top, left)) -> out fp16 NHWC
 * [t, oh+2, ow+2, 64] in conv1's layout: channel (py*4 + px)*3 + c of grid pixel (Y, X) holds the normalised
 * (norm: TG_LPIPS_NORM_*) and scaled ((v - shift[c]) / scale[c], PNetLin's ScalingLayer, fp32) value of picture pixel
 * (4Y + py - 2, 4X + px - 2), 0 outside the picture; channels 48..63 are 0.  One read of the frames.
 * TG_E_INVALID: null pointers, non-positive sizes, a picture outside its frame, a bad norm, out not 16-byte aligned;
 * TG_E_UNSUPPORTED: h or w below TG_LPIPS_MIN_SIDE. */
int tg_lpips_frames_in(const uint8_t* frames, const tg_frame_window* win, int t, int h, int w, int norm, void* out,
                       void* stream);
/* MaxPool2d(3, 2) (floor) of the h x w interior at (y0, x0) of x fp16 NHWC [n, xh, xw, c] (c a multiple of 8), with
 * ph = (h-3)/2 + 1, pw = (w-3)/2 + 1:
 *   shifts == 0: y [n, ph, pw, c]
 *   shifts != 0: conv2's input, y [n, ph+2, pw+2, 4c]: channel block b = by*2 + bx of pixel (i, j) holds the pooled
 *                pixel (i + 3by - 2, j + 3bx - 2), 0 outside the pooled map.
 * Every output element is written.  TG_E_INVALID: null or misaligned (16 bytes) pointers, bad sizes, an interior below
 * 3x3 or outside x. */
int tg_maxpool3x3s2_nhwc_f16(const void* x, int n, int xh, int xw, int c, int y0, int x0, int h, int w, void* y,
                             int shifts, void* stream);
/* Bytes of tg_lpips_head's workspace for npairs pairs and an h x w interior (0 for bad sizes). */
size_t tg_lpips_head_workspace_bytes(int npairs, int h, int w);
/* One LPIPS layer for npairs pairs of images of a batch of features feat fp16 NHWC [n, xh, xw, c] (c <= 512, a
 * multiple of 8), over the h x w interior at (y0, x0): pair k = (pairs[2k], pairs[2k+1]) (int32, device memory; an
 * index outside [0, n) scores NaN) gives
 *   d = mean over the interior of sum_c weights[c] (f0_c / (|f0| + 1e-10) - f1_c / (|f1| + 1e-10))^2,
 * |f| the pixel's channel norm.  Per pixel in fp32; the pixels are summed in float64 per CTA and the CTA sums per pair
 * in a fixed order through the workspace, so the same inputs give the same bits.  out [npairs] float64: out = d, or
 * out += d with accumulate != 0 (the five layers of LPIPS summed in layer order).  weights fp32 [c].
 * TG_E_INVALID: null or misaligned pointers (feat 16 bytes, pairs / weights 4, out / work 8), bad sizes, an interior
 * outside the map, a short workspace; TG_E_UNSUPPORTED: c, more than 65535 pairs.  Two launches. */
int tg_lpips_head(const void* feat, int n, int xh, int xw, int c, int y0, int x0, int h, int w, const int32_t* pairs,
                  int npairs, const float* weights, int accumulate, double* out, void* work, size_t work_bytes,
                  void* stream);

/* BD degradation of the data side (codes/utils/data_utils.py:30-53, called on GT frames by
 * base_model.py:75,115): optional reflect pad by (k-1)/2 | k-1-(k-1)/2, then a depthwise valid
 * correlation with the k x k kernel `k2d` (device, fp32, = create_kernel(sigma)[0,0]) and stride s.
 * x NCHW fp32 [n,c,H,W] -> y [n,c,h,w] with h = (Hp-k)/s+1, Hp = H (+k-1 when pad_data). */
int tg_downsample_bd_nchw_f32(const float* x, const float* k2d, float* y, int n, int c, int H, int W,
                              int k, int s, int pad_data, void* stream);

/* ========================================================================
 * Training: the generator backward (SURVEY.md 8-f1).  Replaces autograd through
 * FRNet.forward_sequence (tecogan_nets.py:174-225) under loss_G.backward() (vsr_model.py:92,
 * vsrgan_model.py:273) and through backward_warp / upsample_func / fnet at the module boundary
 * (vsr_model.py:86, vsrgan_model.py:106-108,214-222, tecogan_nets.py:419-453).
 *
 * fp16 gradients between conv layers carry a power-of-two LOSS SCALE held in device memory:
 * `scale` points at two floats {scale, 1/scale} (tg_grad_scale_from_amax / tg_flow_head_bwd write
 * them); kernels producing fp32 results multiply by 1/scale.  scale == NULL means 1.
 * ====================================================================== */
size_t tg_grad_scale_workspace_bytes(void);   /* 16: {scale, 1/scale} fp32 + amax scratch (zero it once) */
/* scale = 2^floor(log2(target / max(|a|,|b|))) clamped to 2^+-24, the exponent computed exactly (1 when all-zero
 * or when the maximum is inf / NaN); b may be NULL */
int tg_grad_scale_from_amax(const float* a, size_t na, const float* b, size_t nb, float target, void* ws,
                            void* stream);
/* (a [+ b]) * scale : NCHW fp32 [n,c,h,w] -> NHWC fp16 [n,h,w,cpad] (pad channels zero) */
int tg_grad_pack_nhwc_f16(const float* a, const float* b, const float* scale, void* y, int n, int c, int h, int w,
                          int cpad, void* stream);
/* channels [c_offset, c_offset+c) of NHWC fp16 -> NCHW fp32 * 1/scale ; accumulate != 0 adds into y */
int tg_grad_unpack_nchw_f32(const void* x, const float* scale, float* y, int n, int c, int h, int w, int cpad,
                            int c_offset, int accumulate, void* stream);
/* The amax step of tg_grad_scale_from_amax alone: folds max |a| into the workspace, so that the next
 * tg_grad_scale_from_amax on the same ws chooses one scale for several tensors (the VGG extractor's taps). */
int tg_grad_amax_f32(const float* a, size_t na, void* ws, void* stream);
/* tg_grad_pack_nhwc_f16 of one tensor a, with each of these steps where its operand is non-NULL, in this order:
 *   v = (a - sub[ch]) / div[ch]     per-channel normalisation in fp32 (sub and div fp32 [c], given together)
 *   v = v * scale                   (scale NULL: 1)
 *   v = v + add                     add NHWC fp16 [n,h,w,cpad], every channel
 *   v = v * act'(mask)              mask NHWC fp16 [n,h,w,cpad], the stored forward output; act TG_ACT_DRELU /
 *                                   TG_ACT_DLRELU02 with a mask, TG_ACT_NONE without
 * -> NHWC fp16 y [n,h,w,cpad] (channels >= c of a count as 0).  VGG19 perceptual loss: the input normalisation
 * (vgg_nets.py:30) and each feature tap's loss gradient joined to the running gradient.  y, add, mask 16-byte aligned. */
int tg_grad_pack_ex_nhwc_f16(const float* a, const float* sub, const float* div, const float* scale, const void* add,
                             const void* mask, int act, void* y, int n, int c, int h, int w, int cpad, void* stream);
/* tg_grad_unpack_nchw_f32 with a per-channel divisor: y = x * 1/scale / div[ch] (div fp32 [c], non-NULL; the input
 * gradient of the VGG extractor through its normalisation (x - mean) / std) */
int tg_grad_unpack_ex_nchw_f32(const void* x, const float* scale, const float* div, float* y, int n, int c, int h,
                               int w, int cpad, int c_offset, int accumulate, void* stream);
/* db[ch] += 1/scale * sum_pixels dz[p][ch], ch < c_real  (bias gradient of any conv layer) */
int tg_bias_grad_nhwc_f16(const void* dz, size_t npix, int c, int c_real, const float* scale, float* db,
                          void* stream);

/* Weight gradient of a conv3x3 / convT3x3s2 layer: dw += 1/scale * sum_p x[p+tap] (x) dz[p], written in
 * the parameter's own layout (nn.Conv2d [cout_real,cin_real,3,3]; nn.ConvTranspose2d
 * [cin_real,cout_real,3,3]) with fp32 atomics -- the caller zeroes dw (or accumulates on purpose).
 * wgmma: GEMM over pixels (K), x and dz both channel-contiguous ("MN-major") operands. */
typedef struct tg_wgrad_desc {
  const void* x;        /* layer input,  NHWC fp16 [n,h,w,cin]                              */
  const void* dz;       /* gradient of the pre-activation output, NHWC fp16 [n,h,w,cout]
                           (convT: [n,2h,2w,cout]), loss-scaled                           */
  float* dw;            /* fp32 gradient, parameter layout                                  */
  const float* scale;   /* {scale, 1/scale} or NULL                                         */
  float* db;            /* conv3x3 only, may be NULL: bias gradient db[co] += 1/scale * sum_p dz[p][co]
                           (tg_bias_grad_nhwc_f16 after the GEMM)                          */
  int32_t n, h, w;      /* of the layer INPUT                                               */
  int32_t cin, cout;    /* stored channel counts (64/128/256)                               */
  int32_t cin_real, cout_real;
  int32_t kind;         /* TG_CONV_3X3 | TG_CONVT_3X3_S2                                    */
  int32_t max_ctas;     /* 0 = all SMs                                                      */
  int32_t reserved;     /* must be 0                                                        */
} tg_wgrad_desc;
int tg_wgrad_tcgen05(const tg_wgrad_desc* d, void* stream);
int tg_wgrad_simt(const tg_wgrad_desc* d, void* stream);    /* CUDA-core cross-check (tests only) */

/* grid_sample(bilinear, border, align_corners) backward = autograd of net_utils.backward_warp
 * (net_utils.py:50-82): gx += scatter(gy) (fp32 atomics, caller zeroes gx), gflow = gather; either
 * output may be NULL. */
int tg_backward_warp_bwd_nchw_f32(const float* x, const float* flow, const float* gy, float* gx, float* gflow,
                                  int n, int c, int h, int w, void* stream);
/* gradient of tg_warp_s2d_concat_hrflow w.r.t. hr_prev (atomic accumulate) and hr_flow (store), from the
 * loss-scaled NHWC fp16 gradient `gx` of the SRNet input; either output may be NULL */
int tg_warp_s2d_concat_bwd(const void* gx, const float* hr_prev, const float* hr_flow, const float* scale,
                           float* d_hr_prev, float* d_hr_flow, int n, int c, int h, int w, int s, int cpad,
                           void* stream);
/* gradient of y = mul * upsample_func(x): gy [n,c,s*h,s*w] -> gx [n,c,h,w] (net_utils.py:85-156) */
int tg_upsample_bwd_nchw_f32(const float* gy, float* gx, int n, int c, int h, int w, int s, int up_mode, float mul,
                             int accumulate, void* stream);
/* FNet helpers (tecogan_nets.py:28,35,42,74-79), each fused with the activation derivative of the conv
 * layer whose stored output is `x` / `m` (act = that layer's TG_ACT_*):
 *   maxpool:  gx[n,h,w,c] = route(gy[n,h/2,w/2,c]) * act'(x)      upsample2x: gx[n,h,w,c] = T(gy[n,2h,2w,c]) * act'(m) */
int tg_maxpool2x2_bwd_nhwc_f16(const void* x, const void* gy, void* gx, int n, int h, int w, int c, int act,
                               void* stream);
int tg_upsample2x_bilinear_bwd_nhwc_f16(const void* gy, const void* m, void* gx, int n, int h, int w, int c,
                                        int act, void* stream);
/* flow head: flow = 24*tanh(z) (tecogan_nets.py:80): dz = (gflow [+ gflow2]) * (24 - flow^2/24) * scale as NHWC
 * fp16 [n,h,w,cpad]; chooses the loss scale of the FNet backward from the amax of that product (scale_ws as
 * in tg_grad_scale_from_amax) */
int tg_flow_head_bwd(const float* gflow, const float* gflow2, const float* flow, void* scale_ws, float target,
                     void* dz, int n, int h, int w, int cpad, void* stream);
/* Input builder of the spatio-temporal discriminator (SURVEY.md 8-f3; tecogan_nets.py:438-463): the three
 * backward_warps of every 3-frame clip + centre crop / zero pad + "rrrgggbbb" permutes + 27-channel concat
 * in one kernel.  data, bi: [n,t_full,c,h,w] fp32 (frames >= t are ignored, t % 3 == 0); flow:
 * hr_flow_merge [n*t,2,h,w] (clip-major, 3 per clip); out: [n*t/3, 9*c, h, w] = [orig | warp | cond].
 * pad = (spatial_size - c_size)/2, csize = c_size = int(spatial_size * crop_border_ratio). */
int tg_st_disc_input_nchw_f32(const float* data, const float* bi, const float* flow, float* out, int n, int t_full,
                              int t, int c, int h, int w, int pad, int csize, void* stream);
/* its gradient w.r.t. data: gdata [n,t_full,c,h,w] (zeroed by the caller) += orig part + warp scatter */
int tg_st_disc_input_bwd_nchw_f32(const float* gout, const float* flow, float* gdata, int n, int t_full, int t, int c,
                                  int h, int w, int pad, int csize, void* stream);
/* space_to_depth backward (net_utils.py:36-47): gy [n,c*s*s,h/s,w/s] -> gx [n,c,h,w] */
int tg_depth_to_space_nchw_f32(const float* gy, float* gx, int n, int c, int h, int w, int s, void* stream);

/* ------------------------------------------------------------------------
 * Diagnostics: per-CTA role timers.  The sm_90a kernels record none: NULL is
 * accepted (and is the default), a buffer returns TG_E_UNSUPPORTED.
 * ---------------------------------------------------------------------- */
int tg_debug_set_conv_timers(void* device_buffer);

#ifdef __cplusplus
}
#endif
#endif /* TECOGAN_B200_H_ */
