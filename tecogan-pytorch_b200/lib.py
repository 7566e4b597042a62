"""ctypes binding of libtecogan_b200.so (the C ABI declared in include/tecogan_b200.h).

There is NO fallback: if the shared library is missing or a call fails, this module raises.
The library is built in-tree by ``__graft_entry__.build()`` (``make -C csrc``).
"""
import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_int32, c_size_t, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libtecogan_b200.so')
HEADER_PATH = os.path.join(os.path.dirname(_HERE), 'include', 'tecogan_b200.h')

# enums of include/tecogan_b200.h
TG_OK = 0
ACT_NONE, ACT_RELU, ACT_LRELU02, ACT_DRELU, ACT_DLRELU02 = 0, 1, 2, 3, 4
CONV_3X3, CONVT_3X3_S2, CONV_3X3_S2 = 0, 1, 2
UP_BICUBIC, UP_BILINEAR = 0, 1
EPI_NHWC_F16, EPI_FLOW_NCHW_F32, EPI_OUT_NCHW_F32, EPI_NHWC_F16_POOL2 = 0, 1, 2, 3
AMODE_AUTO, AMODE_HALO, AMODE_TAP = 0, 1, 2
YUV_NV12, YUV_I420, YUV_P010, YUV_I420_10 = 0, 1, 2, 3
YUV_YUY2, YUV_UYVY, YUV_I444, YUV_I444_10 = 4, 5, 6, 8      # 7 is not a layout
RESAMPLE_BICUBIC, RESAMPLE_LANCZOS3 = 0, 1
SCENE_CUT_WORK_BYTES = 16            # TG_SCENE_CUT_WORK_BYTES: workspace of tg_scene_cut per slot
TAIL_OUT_ROWS = 40                   # TG_TAIL_OUT_ROWS: rows of tg_pack_tail_out_weights' tile (128 bytes each)
PSNR_NONE, PSNR_RGB, PSNR_Y = 0, 1, 2
GATHER_KEEP, GATHER_ZERO, GATHER_LOAD = 0, 1, 2    # TG_GATHER_*: per-slot state modes of tg_stream_gather
LPIPS_NORM_CALC, LPIPS_NORM_OFFICIAL = 0, 1          # TG_LPIPS_NORM_*: the input normalisation of tg_lpips_frames_in
LPIPS_MIN_SIDE = 31                                  # TG_LPIPS_MIN_SIDE


class ConvDesc(ctypes.Structure):
    """struct tg_conv_desc"""
    _fields_ = [
        ('x', c_void_p), ('weights', c_void_p), ('bias', c_void_p), ('residual', c_void_p),
        ('y', c_void_p),
        ('n', c_int32), ('h', c_int32), ('w', c_int32),
        ('cin', c_int32), ('cout', c_int32), ('cout_real', c_int32),
        ('kind', c_int32), ('act', c_int32), ('epilogue', c_int32),
        ('a_mode', c_int32), ('max_ctas', c_int32), ('cin_real', c_int32),
        ('mask', c_void_p),
    ]


class WgradDesc(ctypes.Structure):
    """struct tg_wgrad_desc"""
    _fields_ = [
        ('x', c_void_p), ('dz', c_void_p), ('dw', c_void_p), ('scale', c_void_p), ('db', c_void_p),
        ('n', c_int32), ('h', c_int32), ('w', c_int32),
        ('cin', c_int32), ('cout', c_int32), ('cin_real', c_int32), ('cout_real', c_int32),
        ('kind', c_int32), ('max_ctas', c_int32), ('reserved', c_int32),
    ]


class TailDesc(ctypes.Structure):
    """struct tg_tail_desc"""
    _fields_ = [
        ('x', c_void_p), ('w_up', c_void_p), ('b_up', c_void_p), ('w_out', c_void_p), ('b_out', c_void_p),
        ('lr', c_void_p), ('y', c_void_p), ('y_u8', c_void_p),
        ('n', c_int32), ('h', c_int32), ('w', c_int32), ('cout_real', c_int32),
        ('lr_scale', c_int32), ('up_mode', c_int32), ('max_ctas', c_int32), ('accumulate', c_int32),
        ('reserved', c_int32),
    ]


class YuvFormat(ctypes.Structure):
    """struct tg_yuv_format"""
    _fields_ = [('layout', c_int32), ('matrix', c_int32), ('full_range', c_int32), ('reserved', c_int32)]


class FrameWindow(ctypes.Structure):
    """struct tg_frame_window"""
    _fields_ = [('frame_h', c_int32), ('frame_w', c_int32), ('top', c_int32), ('left', c_int32)]


class FarnebackParams(ctypes.Structure):
    """struct tg_farneback_params"""
    _fields_ = [('pyr_scale', c_double), ('levels', c_int32), ('winsize', c_int32), ('iterations', c_int32),
                ('poly_n', c_int32), ('poly_sigma', c_double), ('flags', c_int32), ('reserved', c_int32)]


_P = c_void_p
_SIGNATURES = {
    'tg_version': (c_int, []),
    'tg_last_error_string': (c_char_p, []),
    'tg_device_sm_count': (c_int, [ctypes.POINTER(c_int)]),
    'tg_packed_weight_bytes': (c_size_t, [c_int, c_int]),
    'tg_pack_conv3x3_weights': (c_int, [_P, c_int, c_int, _P, c_int, c_int, _P]),
    'tg_pack_convT3x3s2_weights': (c_int, [_P, c_int, c_int, _P, c_int, c_int, _P]),
    'tg_packed_weight_bytes_tapn': (c_size_t, [c_int]),
    'tg_pack_conv3x3_weights_tapn': (c_int, [_P, c_int, c_int, _P, c_int, _P]),
    'tg_conv_tcgen05': (c_int, [ctypes.POINTER(ConvDesc), _P]),
    'tg_conv_simt': (c_int, [ctypes.POINTER(ConvDesc), _P]),
    'tg_convT_convout_tcgen05': (c_int, [ctypes.POINTER(TailDesc), _P]),
    'tg_pack_tail_out_weights': (c_int, [_P, c_int, c_int, _P, _P]),
    'tg_warp_s2d_concat_hrflow': (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    'tg_warp_s2d_concat_lrflow': (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int,
                                          c_int, c_int, c_int, _P]),
    'tg_maxpool2x2_nhwc_f16': (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
    'tg_upsample2x_bilinear_nhwc_f16': (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
    'tg_pack_pair_nhwc_f16': (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    'tg_backward_warp_nchw_f32': (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, _P]),
    'tg_space_to_depth_nchw_f32': (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    'tg_upsample_nchw_f32': (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                     c_float, c_int, _P]),
    'tg_nchw_f32_to_nhwc_f16': (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    'tg_nhwc_f16_to_nchw_f32': (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    'tg_float_to_uint8_nhwc': (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
    'tg_float_to_uint8_nhwc_window': (c_int, [_P, _P, ctypes.POINTER(FrameWindow), c_int, c_int, c_int, c_int, _P]),
    'tg_stream_frame_in': (c_int, [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    'tg_stream_gather': (c_int, [_P, c_int, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    'tg_stream_frame_in_yuv420': (c_int, [_P, c_int, _P, _P, _P, _P, c_int, c_int, c_int, c_int, _P]),
    'tg_rgb_u8_to_yuv420': (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P]),
    'tg_stream_frame_in_yuv': (c_int, [_P, ctypes.POINTER(YuvFormat), _P, _P, _P, _P, c_int, c_int, c_int, c_int, _P]),
    'tg_rgb_to_yuv': (c_int, [_P, _P, _P, ctypes.POINTER(YuvFormat), c_int, c_int, c_int, _P]),
    'tg_yuv_coefficients': (c_int, [ctypes.POINTER(YuvFormat), ctypes.POINTER(c_int32)]),
    'tg_stream_frame_in_window': (c_int, [_P, ctypes.POINTER(FrameWindow), _P, _P, _P, _P, c_int, c_int, c_int, c_int,
                                          c_int, c_int, _P]),
    'tg_stream_frame_in_yuv_window': (c_int, [_P, ctypes.POINTER(YuvFormat), ctypes.POINTER(FrameWindow), _P, _P, _P,
                                              _P, c_int, c_int, c_int, c_int, _P]),
    'tg_rgb_to_yuv_window': (c_int, [_P, _P, _P, ctypes.POINTER(YuvFormat), ctypes.POINTER(FrameWindow), c_int, c_int,
                                     c_int, _P]),
    'tg_fill_black': (c_int, [_P, ctypes.POINTER(YuvFormat), c_int, c_int, c_int, c_int, _P]),
    'tg_luma_line_sums': (c_int, [_P, ctypes.POINTER(YuvFormat), c_int, c_int, c_int, c_int, c_int, _P, _P, _P]),
    'tg_resample_taps': (c_int, [c_int, c_int, c_int, ctypes.POINTER(c_int)]),
    'tg_resample_table': (c_int, [c_int, c_int, c_int, c_int, _P, _P]),
    'tg_resample_nchw_f32': (c_int, [_P, c_int, c_int, c_int, c_int, _P, _P, c_int, _P, _P, c_int, c_int, c_int,
                                     _P, _P, _P]),
    'tg_resample_nchw_f32_window': (c_int, [_P, c_int, c_int, c_int, c_int, _P, _P, c_int, _P, _P, c_int, c_int, c_int,
                                            _P, ctypes.POINTER(FrameWindow), _P]),
    'tg_stream_frame_in_resample': (c_int, [_P, ctypes.POINTER(YuvFormat), c_int, ctypes.POINTER(FrameWindow), c_int,
                                            c_int, _P, _P, c_int, _P, _P, c_int, _P, _P, _P, _P, c_int, c_int, c_int,
                                            c_int, c_int, _P]),
    'tg_scene_cut': (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P, c_double, _P, _P, _P, _P, _P]),
    'tg_metrics_frames_in': (c_int, [_P, c_int, c_int, _P, c_int, c_int, c_int, c_int, _P, _P, _P]),
    'tg_farneback_workspace_bytes': (c_size_t, [c_int, c_int, c_int, c_int]),
    'tg_farneback': (c_int, [_P, c_int, c_int, c_int, c_int, ctypes.POINTER(FarnebackParams), _P, _P, c_size_t, _P]),
    'tg_flow_epe_sum': (c_int, [_P, _P, c_int, c_int, c_int, _P, _P]),
    'tg_flow_epe_sum_window_workspace_bytes': (c_size_t, [c_int, c_int]),
    'tg_flow_epe_sum_window': (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, c_size_t, _P]),
    'tg_official_frames_stats_workspace_bytes': (c_size_t, [c_int, c_int, c_int]),
    'tg_official_frames_stats': (c_int, [_P, c_int, c_int, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P,
                                         _P, c_size_t, _P]),
    'tg_ssim_y_workspace_bytes': (c_size_t, [c_int, c_int, c_int]),
    'tg_ssim_y': (c_int, [_P, c_int, c_int, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P, _P, _P, c_size_t,
                          _P]),
    'tg_lpips_frames_in': (c_int, [_P, ctypes.POINTER(FrameWindow), c_int, c_int, c_int, c_int, _P, _P]),
    'tg_maxpool3x3s2_nhwc_f16': (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P, c_int, _P]),
    'tg_lpips_head_workspace_bytes': (c_size_t, [c_int, c_int, c_int]),
    'tg_lpips_head': (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P, c_int, _P, c_int, _P, _P,
                              c_size_t, _P]),
    'tg_downsample_bd_nchw_f32': (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    'tg_debug_set_conv_timers': (c_int, [_P]),
    # ---- training (generator backward)
    'tg_pack_conv3x3_weights_dgrad': (c_int, [_P, c_int, c_int, _P, c_int, c_int, _P]),
    'tg_pack_conv3x3s2_weights': (c_int, [_P, c_int, c_int, _P, c_int, c_int, _P]),
    'tg_grad_scale_workspace_bytes': (c_size_t, []),
    'tg_grad_scale_from_amax': (c_int, [_P, c_size_t, _P, c_size_t, c_float, _P, _P]),
    'tg_grad_pack_nhwc_f16': (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    'tg_grad_unpack_nchw_f32': (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    'tg_bias_grad_nhwc_f16': (c_int, [_P, c_size_t, c_int, c_int, _P, _P, _P]),
    'tg_wgrad_tcgen05': (c_int, [ctypes.POINTER(WgradDesc), _P]),
    'tg_wgrad_simt': (c_int, [ctypes.POINTER(WgradDesc), _P]),
    'tg_backward_warp_bwd_nchw_f32': (c_int, [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, _P]),
    'tg_warp_s2d_concat_bwd': (c_int, [_P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    'tg_upsample_bwd_nchw_f32': (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_int, _P]),
    'tg_maxpool2x2_bwd_nhwc_f16': (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    'tg_upsample2x_bilinear_bwd_nhwc_f16': (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
    'tg_flow_head_bwd': (c_int, [_P, _P, _P, _P, c_float, _P, c_int, c_int, c_int, c_int, _P]),
    'tg_st_disc_input_nchw_f32': (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    'tg_st_disc_input_bwd_nchw_f32': (c_int, [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    'tg_depth_to_space_nchw_f32': (c_int, [_P, _P, c_int, c_int, c_int, c_int, c_int, _P]),
}

_lib = None


class TecoganB200Error(RuntimeError):
    pass


def exported_symbols():
    return sorted(_SIGNATURES)


def load():
    """Load the CUDA library (once). Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise TecoganB200Error(
            f'{LIB_PATH} is missing: the sm_90a CUDA library has not been built. Run '
            f'`python -c "import __graft_entry__ as g; g.build()"` (or `make -C '
            f'{os.path.join(_HERE, "csrc")}`). There is no CPU / PyTorch fallback.')
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the .so does not export it
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what):
    if rc != TG_OK:
        msg = load().tg_last_error_string()
        raise TecoganB200Error(f'{what} failed (rc={rc}): {msg.decode() if msg else ""}')
