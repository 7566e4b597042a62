"""Torch-tensor front end of the C ABI (include/tecogan_b200.h).

PyTorch is plumbing here: it owns device memory and the CUDA stream; every operation below is
one call into libtecogan_b200.so on ``torch.cuda.current_stream()``.  No op has a torch/CPU
fallback -- a tensor that is not on a CUDA device is an error.
"""
import collections
import ctypes
import os

import torch

from . import lib as L


LAUNCH_COUNT = 0   # kernels enqueued through the C ABI by this process (each call = 1 launch)


def _stream():
    global LAUNCH_COUNT
    LAUNCH_COUNT += 1
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _req(t, dtype, name, ndim=None):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise L.TecoganB200Error(f'{name}: expected a CUDA tensor (no CPU fallback exists)')
    if t.dtype != dtype:
        raise L.TecoganB200Error(f'{name}: expected dtype {dtype}, got {t.dtype}')
    if ndim is not None and t.dim() != ndim:
        raise L.TecoganB200Error(f'{name}: expected {ndim} dims, got {tuple(t.shape)}')
    if not t.is_contiguous():
        raise L.TecoganB200Error(f'{name}: tensor must be contiguous')
    return t


def sm_count():
    out = ctypes.c_int(0)
    L.check(L.load().tg_device_sm_count(ctypes.byref(out)), 'tg_device_sm_count')
    return out.value


def pad64(c):
    return (c + 63) // 64 * 64


# ---------------------------------------------------------------------------- conv layers
class PackedConv:
    """One 3x3 conv / stride-2 transposed conv of the path with device-packed fp16 weights.

    weight: nn.Conv2d layout [cout,cin,3,3] or nn.ConvTranspose2d layout [cin,cout,3,3] (fp32).
    Stored channel counts are padded to multiples of 64 (cin) and to 64/128/192/256/384 or 16 (cout).
    """

    def __init__(self, weight, bias, kind=L.CONV_3X3, act=L.ACT_NONE, epilogue=L.EPI_NHWC_F16):
        self.kind, self.act, self.epilogue = kind, act, epilogue
        if kind == L.CONV_3X3:
            self.cout_real, self.cin_real = weight.shape[0], weight.shape[1]
        else:
            self.cin_real, self.cout_real = weight.shape[0], weight.shape[1]
        self.cin = pad64(self.cin_real)
        self.tapn = epilogue != L.EPI_NHWC_F16      # thin NCHW heads: tap-major N packing
        self.cout = pad64(self.cout_real) if not self.tapn else 48
        # Walk the tiles last to first (TG_AMODE_REVERSE); same output bits.  The networks set it so that each conv
        # walks opposite to the launch that wrote its input and starts on what is still in L2.
        self.reverse = False
        self.packed = None
        self.tail_packed = None
        self.bias = None
        self._ver = None
        self.refresh(weight, bias)

    def refresh(self, weight, bias, force=False):
        """(Re)pack when the parameters changed (optimizer step / load_state_dict).  Change detection
        is the tensors' version counters + storage pointers; writes through ``param.data`` do not
        bump the counter -- call with force=True (FRNet.refresh_packed_weights(force=True)) after such
        an update."""
        ver = (weight._version, bias._version, weight.data_ptr(), bias.data_ptr())
        if ver == self._ver and not force:
            return
        lib = L.load()
        w = _req(weight.detach(), torch.float32, 'weight', 4)
        nbytes = (lib.tg_packed_weight_bytes_tapn(self.cin) if self.tapn
                  else lib.tg_packed_weight_bytes(self.cin, self.cout))
        if self.packed is None:
            self.packed = torch.empty(nbytes, dtype=torch.uint8, device=w.device)
            self.bias = torch.zeros(self.cout, dtype=torch.float32, device=w.device)
        if self.tapn:
            rc = lib.tg_pack_conv3x3_weights_tapn(_ptr(w), self.cout_real, self.cin_real, _ptr(self.packed),
                                                  self.cin, _stream())
        elif self.kind == L.CONV_3X3:
            rc = lib.tg_pack_conv3x3_weights(_ptr(w), self.cout_real, self.cin_real, _ptr(self.packed),
                                             self.cout, self.cin, _stream())
        else:
            rc = lib.tg_pack_convT3x3s2_weights(_ptr(w), self.cin_real, self.cout_real,
                                                _ptr(self.packed), self.cout, self.cin, _stream())
        L.check(rc, 'tg_pack_weights')
        if self.epilogue == L.EPI_OUT_NCHW_F32 and self.cin == 64 and self.cout_real <= 3:
            # conv_out: the fused SRNet tail (fused_tail) reads its own N packing of the same weights
            if self.tail_packed is None:
                self.tail_packed = torch.empty(L.TAIL_OUT_ROWS * 128, dtype=torch.uint8, device=w.device)
            L.check(lib.tg_pack_tail_out_weights(_ptr(w), self.cout_real, self.cin_real, _ptr(self.tail_packed),
                                                 _stream()), 'tg_pack_tail_out_weights')
        self.bias[:self.cout_real].copy_(bias.detach())
        self._ver = ver

    def out_shape(self, n, h, w):
        if self.epilogue == L.EPI_NHWC_F16:
            if self.kind == L.CONVT_3X3_S2:
                return (n, 2 * h, 2 * w, self.cout), torch.float16
            return (n, h, w, self.cout), torch.float16
        return (n, self.cout_real, h, w), torch.float32

    def __call__(self, x, y=None, residual=None, impl=None, a_mode=None, max_ctas=0, pool=False):
        """x NHWC fp16 [n,h,w,cin] -> y (allocated when None).  pool=True: nn.MaxPool2d(2,2) folded into the
        epilogue, y = [n,h//2,w//2,cout] (conv3x3 layers with the NHWC epilogue, wgmma path only)."""
        _req(x, torch.float16, 'conv input', 4)
        n, h, w, cin = x.shape
        if cin != self.cin:
            raise L.TecoganB200Error(f'conv input has {cin} channels, layer expects {self.cin}')
        shape, dtype = self.out_shape(n, h, w)
        if pool:
            if self.epilogue != L.EPI_NHWC_F16 or self.kind != L.CONV_3X3 or residual is not None:
                raise L.TecoganB200Error('pooled epilogue: conv3x3 with the NHWC epilogue and no residual only')
            shape = (n, h // 2, w // 2, self.cout)
        if y is None:
            y = torch.empty(shape, dtype=dtype, device=x.device)
        else:
            _req(y, dtype, 'conv output')
            if tuple(y.shape) != shape:
                raise L.TecoganB200Error(f'conv output shape {tuple(y.shape)} != {shape}')
        if residual is not None:
            _req(residual, torch.float16, 'residual', 4)
            if tuple(residual.shape) != (n, h, w, self.cout):
                raise L.TecoganB200Error('residual shape mismatch')
        d = L.ConvDesc()
        d.x, d.weights, d.bias = x.data_ptr(), self.packed.data_ptr(), self.bias.data_ptr()
        d.residual = residual.data_ptr() if residual is not None else None
        d.y = y.data_ptr()
        d.n, d.h, d.w, d.cin, d.cout, d.cout_real = n, h, w, self.cin, self.cout, self.cout_real
        d.kind, d.act, d.epilogue = self.kind, self.act, (L.EPI_NHWC_F16_POOL2 if pool else self.epilogue)
        d.a_mode = (default_a_mode() if a_mode is None else a_mode) | (L.AMODE_REVERSE if self.reverse else 0)
        d.max_ctas = max_ctas
        d.cin_real = self.cin_real
        impl = impl or default_conv_impl()
        lib = L.load()
        if impl == 'tcgen05':
            L.check(lib.tg_conv_tcgen05(ctypes.byref(d), _stream()), 'tg_conv_tcgen05')
        elif impl == 'simt':
            L.check(lib.tg_conv_simt(ctypes.byref(d), _stream()), 'tg_conv_simt')
        else:
            raise L.TecoganB200Error(f'unknown conv impl {impl!r}')
        return y


def fused_tail(up, outc, x, lr_curr, lr_scale, up_mode, y=None, y_u8=None, max_ctas=0, accumulate=False):
    """SRNet tail in one launch (tg_convT_convout_tcgen05): y = conv_out(relu(convT(x))) + upsample_func(lr_curr)
    [, y_u8 = float32_to_uint8(y) as NHWC].  `up` / `outc` are the PackedConv objects of the last transposed
    conv and of conv_out (the transposed conv's packed weights and conv_out's tail packing are used as they are)."""
    _req(x, torch.float16, 'tail input', 4)
    n, h, w, c = x.shape
    if (up.kind != L.CONVT_3X3_S2 or up.cin != 64 or up.cout != 64 or c != 64 or outc.tail_packed is None):
        raise L.TecoganB200Error('fused tail: needs a 64->64 transposed conv and a 64->(<=3) conv_out')
    co = outc.cout_real
    if y is None:
        y = torch.empty((n, co, 2 * h, 2 * w), dtype=torch.float32, device=x.device)
    _req(y, torch.float32, 'tail output', 4)
    if tuple(y.shape) != (n, co, 2 * h, 2 * w):
        raise L.TecoganB200Error(f'fused tail: output shape {tuple(y.shape)}')
    d = L.TailDesc()
    d.x, d.w_up, d.b_up = x.data_ptr(), up.packed.data_ptr(), up.bias.data_ptr()
    d.w_out, d.b_out, d.y = outc.tail_packed.data_ptr(), outc.bias.data_ptr(), y.data_ptr()
    if lr_curr is not None:
        _req(lr_curr, torch.float32, 'lr_curr', 4)
        if tuple(lr_curr.shape) != (n, co, 2 * h // lr_scale, 2 * w // lr_scale):
            raise L.TecoganB200Error(f'fused tail: lr_curr shape {tuple(lr_curr.shape)}')
        d.lr = lr_curr.data_ptr()
    if y_u8 is not None:
        _req(y_u8, torch.uint8, 'uint8 output', 4)
        if tuple(y_u8.shape) != (n, 2 * h, 2 * w, co):
            raise L.TecoganB200Error(f'fused tail: uint8 output shape {tuple(y_u8.shape)}')
        d.y_u8 = y_u8.data_ptr()
    d.n, d.h, d.w, d.cout_real, d.lr_scale, d.up_mode, d.max_ctas, d.reserved = n, h, w, co, lr_scale, up_mode, max_ctas, 0
    d.accumulate = 1 if accumulate else 0
    L.check(L.load().tg_convT_convout_tcgen05(ctypes.byref(d), _stream()), 'tg_convT_convout_tcgen05')
    return y


def tail_mode():
    """TECOGAN_B200_TAIL: '0' = last transposed conv, conv_out, residual upsample and uint8 as four launches;
    'acc' = tg_convT_convout_tcgen05 accumulating onto a pre-written residual (default: one coalesced read per
    pixel instead of the in-kernel 4x4 LR gathers); 'fused' = residual and uint8 evaluated inside the tail
    kernel."""
    v = os.environ.get('TECOGAN_B200_TAIL', 'acc')
    return {'0': None, '': None, '1': 'fused', 'fused': 'fused', '2': 'acc', 'acc': 'acc'}[v]


def pool_fused():
    """TECOGAN_B200_POOL=0 runs FNet's three max-pools as their own kernels instead of in the epilogue of the
    conv that feeds them (A/B measurements; bit-identical output)."""
    return os.environ.get('TECOGAN_B200_POOL', '1') != '0'


def chain_enabled():
    # bench.py asks; the persistent conv-chain kernel was removed (DESIGN.md)
    return False


def default_conv_impl():
    """'tcgen05' (the product path: the wgmma kernels; the name is historical) unless TECOGAN_B200_CONV=simt selects the CUDA-core
    cross-check kernel (bring-up / debugging only)."""
    return os.environ.get('TECOGAN_B200_CONV', 'tcgen05')


def default_a_mode():
    return {'auto': L.AMODE_AUTO, 'halo': L.AMODE_HALO, 'tap': L.AMODE_TAP}[
        os.environ.get('TECOGAN_B200_AMODE', 'auto')]


# ---------------------------------------------------------------------------- fused warp
def warp_s2d_concat_hrflow(hr_prev, hr_flow, lr_curr, scale, out=None, cpad=64):
    _req(hr_prev, torch.float32, 'hr_prev', 4)
    _req(hr_flow, torch.float32, 'hr_flow', 4)
    _req(lr_curr, torch.float32, 'lr_curr', 4)
    n, c, h, w = lr_curr.shape
    if tuple(hr_prev.shape) != (n, c, scale * h, scale * w) or tuple(hr_flow.shape) != (n, 2, scale * h, scale * w):
        raise L.TecoganB200Error('warp_s2d_concat: shape mismatch')
    if out is None:
        out = torch.empty((n, h, w, cpad), dtype=torch.float16, device=lr_curr.device)
    L.check(L.load().tg_warp_s2d_concat_hrflow(_ptr(hr_prev), _ptr(hr_flow), _ptr(lr_curr), _ptr(out),
                                               n, c, h, w, scale, cpad, _stream()),
            'tg_warp_s2d_concat_hrflow')
    return out


def warp_s2d_concat_lrflow(hr_prev, lr_flow, lr_curr, scale, up_mode, out=None, cpad=64):
    _req(hr_prev, torch.float32, 'hr_prev', 4)
    _req(lr_flow, torch.float32, 'lr_flow', 4)
    _req(lr_curr, torch.float32, 'lr_curr', 4)
    n, c, h, w = lr_curr.shape
    h8, w8 = lr_flow.shape[2], lr_flow.shape[3]
    if tuple(hr_prev.shape) != (n, c, scale * h, scale * w) or lr_flow.shape[0] != n or lr_flow.shape[1] != 2:
        raise L.TecoganB200Error('warp_s2d_concat: shape mismatch')
    if out is None:
        out = torch.empty((n, h, w, cpad), dtype=torch.float16, device=lr_curr.device)
    L.check(L.load().tg_warp_s2d_concat_lrflow(_ptr(hr_prev), _ptr(lr_flow), _ptr(lr_curr), _ptr(out),
                                               n, c, h, w, h8, w8, scale, up_mode, cpad, _stream()),
            'tg_warp_s2d_concat_lrflow')
    return out


# ---------------------------------------------------------------------------- NHWC fp16 helpers
def maxpool2x2(x, y=None):
    _req(x, torch.float16, 'maxpool input', 4)
    n, h, w, c = x.shape
    if y is None:
        y = torch.empty((n, h // 2, w // 2, c), dtype=torch.float16, device=x.device)
    L.check(L.load().tg_maxpool2x2_nhwc_f16(_ptr(x), _ptr(y), n, h, w, c, _stream()), 'tg_maxpool2x2')
    return y


def upsample2x(x, y=None):
    _req(x, torch.float16, 'upsample2x input', 4)
    n, h, w, c = x.shape
    if y is None:
        y = torch.empty((n, 2 * h, 2 * w, c), dtype=torch.float16, device=x.device)
    L.check(L.load().tg_upsample2x_bilinear_nhwc_f16(_ptr(x), _ptr(y), n, h, w, c, _stream()),
            'tg_upsample2x')
    return y


def pack_pair(x1, x2, y=None, cpad=64):
    _req(x1, torch.float32, 'x1', 4)
    _req(x2, torch.float32, 'x2', 4)
    n, c, h, w = x1.shape
    if y is None:
        y = torch.empty((n, h, w, cpad), dtype=torch.float16, device=x1.device)
    L.check(L.load().tg_pack_pair_nhwc_f16(_ptr(x1), _ptr(x2), _ptr(y), n, c, h, w, cpad, _stream()),
            'tg_pack_pair')
    return y


def nchw_to_nhwc(x, cpad=None, y=None):
    _req(x, torch.float32, 'x', 4)
    n, c, h, w = x.shape
    cpad = cpad or pad64(c)
    if y is None:
        y = torch.empty((n, h, w, cpad), dtype=torch.float16, device=x.device)
    L.check(L.load().tg_nchw_f32_to_nhwc_f16(_ptr(x), _ptr(y), n, c, h, w, cpad, 0, _stream()),
            'tg_nchw_to_nhwc')
    return y


def nhwc_to_nchw(x, c, y=None):
    _req(x, torch.float16, 'x', 4)
    n, h, w, cpad = x.shape
    if y is None:
        y = torch.empty((n, c, h, w), dtype=torch.float32, device=x.device)
    L.check(L.load().tg_nhwc_f16_to_nchw_f32(_ptr(x), _ptr(y), n, c, h, w, cpad, _stream()),
            'tg_nhwc_to_nchw')
    return y


# ---------------------------------------------------------------------------- NCHW fp32 module ops
def backward_warp(x, flow, y=None):
    _req(x, torch.float32, 'x', 4)
    _req(flow, torch.float32, 'flow', 4)
    n, c, h, w = x.shape
    if tuple(flow.shape) != (n, 2, h, w):
        raise L.TecoganB200Error('backward_warp: flow shape mismatch')
    if y is None:
        y = torch.empty_like(x)
    L.check(L.load().tg_backward_warp_nchw_f32(_ptr(x), _ptr(flow), _ptr(y), n, c, h, w, _stream()),
            'tg_backward_warp')
    return y


def space_to_depth(x, scale, y=None):
    _req(x, torch.float32, 'x', 4)
    n, c, h, w = x.shape
    if y is None:
        y = torch.empty((n, c * scale * scale, h // scale, w // scale), dtype=torch.float32, device=x.device)
    L.check(L.load().tg_space_to_depth_nchw_f32(_ptr(x), _ptr(y), n, c, h, w, scale, _stream()),
            'tg_space_to_depth')
    return y


def upsample(x, scale, up_mode, out_hw=None, mul=1.0, y=None, accumulate=False):
    """[y +] mul * upsample_func(reflect_pad(x -> out_hw)); out_hw defaults to x's own size."""
    _req(x, torch.float32, 'x', 4)
    n, c, hin, win = x.shape
    h, w = out_hw if out_hw is not None else (hin, win)
    if y is None:
        y = torch.empty((n, c, h * scale, w * scale), dtype=torch.float32, device=x.device)
    L.check(L.load().tg_upsample_nchw_f32(_ptr(x), _ptr(y), n, c, hin, win, h, w, scale, up_mode,
                                          ctypes.c_float(mul), int(accumulate), _stream()), 'tg_upsample')
    return y


def downsample_bd(x, k2d, scale, pad_data, y=None):
    """x NCHW fp32, k2d [k,k] fp32 (device) -> blurred + subsampled NCHW fp32 (tg_downsample_bd_nchw_f32)."""
    _req(x, torch.float32, 'data', 4)
    _req(k2d, torch.float32, 'kernel', 2)
    n, c, H, W = x.shape
    k = k2d.shape[0]
    if k2d.shape[1] != k:
        raise L.TecoganB200Error('downsample_bd: kernel must be square')
    Hp, Wp = (H + k - 1, W + k - 1) if pad_data else (H, W)
    oh, ow = (Hp - k) // scale + 1, (Wp - k) // scale + 1
    if y is None:
        y = torch.empty((n, c, oh, ow), dtype=torch.float32, device=x.device)
    L.check(L.load().tg_downsample_bd_nchw_f32(_ptr(x), _ptr(k2d), _ptr(y), n, c, H, W, k, scale,
                                               1 if pad_data else 0, _stream()), 'tg_downsample_bd')
    return y


def float_to_uint8_nhwc(x, y=None):
    _req(x, torch.float32, 'x', 4)
    n, c, h, w = x.shape
    if y is None:
        y = torch.empty((n, h, w, c), dtype=torch.uint8, device=x.device)
    L.check(L.load().tg_float_to_uint8_nhwc(_ptr(x), _ptr(y), n, c, h, w, _stream()),
            'tg_float_to_uint8')
    return y


def float_to_uint8_nhwc_window(x, y, window):
    """tg_float_to_uint8_nhwc_window: float_to_uint8_nhwc of x fp32 NCHW [n,c,h,w] written as the h x w picture at
    window = (top, left) of each uint8 NHWC frame of y [n,Hf,Wf,c]; nothing else of y is written."""
    _req(x, torch.float32, 'x', 4)
    n, c, h, w = x.shape
    _req(y, torch.uint8, 'y', 4)
    if y.shape[0] != n or y.shape[3] != c or y.device != x.device:
        raise L.TecoganB200Error(f'float_to_uint8_nhwc: y {tuple(y.shape)} does not hold [n={n},Hf,Wf,c={c}] frames')
    win = frame_window(y.shape[1], y.shape[2], *window)
    L.check(L.load().tg_float_to_uint8_nhwc_window(_ptr(x), _ptr(y), ctypes.byref(win), n, c, h, w, _stream()),
            'tg_float_to_uint8_nhwc_window')
    return y


def frame_window(frame_h, frame_w, top, left):
    """struct tg_frame_window: the picture at (top, left) of a frame_h x frame_w stored frame."""
    return L.FrameWindow(int(frame_h), int(frame_w), int(top), int(left))


def _step_state(name, reset, lr_curr, lr_prev, hr_prev, scale):
    """Checks the step state a frame input writes: lr_curr / lr_prev fp32 [n,c,h,w], hr_prev fp32 [n,c,scale*h,scale*w]
    and reset int32 [n] or None.  -> (n, c, h, w)"""
    for t, nm in ((lr_curr, 'lr_curr'), (lr_prev, 'lr_prev'), (hr_prev, 'hr_prev')):
        _req(t, torch.float32, nm, 4)
    n, c, h, w = lr_curr.shape
    if tuple(lr_prev.shape) != (n, c, h, w) or tuple(hr_prev.shape) != (n, c, scale * h, scale * w):
        raise L.TecoganB200Error(f'{name}: lr_prev / hr_prev shape mismatch')
    if reset is not None:
        _req(reset, torch.int32, 'reset', 1)
        if reset.shape[0] != n:
            raise L.TecoganB200Error(f'{name}: reset has {reset.shape[0]} entries, expected {n}')
    return n, c, h, w


def _split_window(name, layout, window):
    """window -> ((top, left) or None, the frame width it names or None).  A v210 frame's padded rows do not give its
    width, so a v210 window is (top, left, frame_w); every other window is (top, left)."""
    if window is None:
        return None, None
    window = tuple(window)
    if layout is not None and YUV_LAYOUT_TABLE[layout].needs_width:
        if len(window) != 3:
            raise L.TecoganB200Error(f'{name}: a {layout} window is (top, left, frame_w), got {window!r}')
        return window[:2], window[2]
    return window, None


def _frames(name, frames, layout, n, c, h, w, window, frame_w=None):
    """Checks the frames an h x w picture of n slots is read from: uint8 HWC [n,Hf,Wf,c] (layout None) or a YUV
    layout's words [n,*yuv_frame_shape(layout, Hf, Wf)] (yuv_word_dtype), or None (no frames).  Hf x Wf is h x w, or
    any size when the picture is read at window = (top, left); a windowed v210 frame's width Wf is frame_w, which its
    padded rows do not give.  -> (Hf, Wf)"""
    if layout is not None:
        if c != 3:
            raise L.TecoganB200Error(f'{name}: lr_curr has {c} channels, YUV frames decode to 3')
        err = yuv_size_error(layout, h, w)
        if err:
            raise L.TecoganB200Error(f'{name}: {err}')
    if frames is None:
        return h, w
    if layout is None:
        _req(frames, torch.uint8, 'frames', 4)
        fh, fw = (h, w) if window is None else frames.shape[1:3]
        want = (n, fh, fw, c)
    else:
        _req(frames, yuv_word_dtype(layout), 'frames', 3)
        fh, fw = (h, w) if window is None else yuv_frame_size(layout, frames.shape[1:], frame_w)
        want = (n, *yuv_frame_shape(layout, fh, fw))
    if tuple(frames.shape) != want:
        raise L.TecoganB200Error(f'{name}: frames {tuple(frames.shape)} != {want} ({layout or "uint8 HWC"} frames of '
                                 f'{fh}x{fw})')
    return fh, fw


def _same_device(name, x, *tensors):
    for t in tensors:
        if t is not None and t.device != x.device:
            raise L.TecoganB200Error(f'{name}: tensors on different devices')


def stream_frame_in(u8, reset, lr_curr, lr_prev, hr_prev, scale, bgr=False, window=None):
    """Frame input of a streamed step (tg_stream_frame_in): u8 uint8 [n,h,w,c] (or None) -> lr_curr fp32
    [n,c,h,w] = u8 / 255, channels reversed when bgr; slots k with reset[k] != 0 (int32 [n] on the device,
    or None) get lr_prev[k] = hr_prev[k] = 0 ([n,c,h,w] / [n,c,scale*h,scale*w] fp32).  With window = (top, left),
    u8 is [n,Hf,Wf,c] and the h x w picture at (top, left) of each frame is read (tg_stream_frame_in_window)."""
    name = 'stream_frame_in'
    n, c, h, w = _step_state(name, reset, lr_curr, lr_prev, hr_prev, scale)
    fh, fw = _frames(name, u8, None, n, c, h, w, window)
    _same_device(name, lr_curr, lr_prev, hr_prev, u8, reset)
    if window is not None:
        win = frame_window(fh, fw, *window) if u8 is not None else frame_window(h, w, 0, 0)
        L.check(L.load().tg_stream_frame_in_window(_ptr(u8), ctypes.byref(win), _ptr(reset), _ptr(lr_curr),
                                                   _ptr(lr_prev), _ptr(hr_prev), n, c, h, w, scale, int(bool(bgr)),
                                                   _stream()), 'tg_stream_frame_in_window')
        return lr_curr
    L.check(L.load().tg_stream_frame_in(_ptr(u8), _ptr(reset), _ptr(lr_curr), _ptr(lr_prev), _ptr(hr_prev),
                                        n, c, h, w, scale, int(bool(bgr)), _stream()), 'tg_stream_frame_in')
    return lr_curr


def stream_gather(ring, table, warm_hr, lr_curr, lr_prev, hr_prev, scale):
    """Step input of a padded stream from the ring of decoded frames (tg_stream_gather): ring fp32 [depth,n,c,h,w],
    table int32 [3n] on the device (cur, mode, prev per slot; modes L.GATHER_KEEP / _ZERO / _LOAD), warm_hr fp32
    [n,c,scale*h,scale*w] or None -> lr_curr[k] = ring[cur[k]][k]; zero: lr_prev[k] = hr_prev[k] = 0; load:
    lr_prev[k] = ring[prev[k]][k] (0 for prev[k] < 0), hr_prev[k] = warm_hr[k]."""
    name = 'stream_gather'
    _req(ring, torch.float32, 'ring', 5)
    depth, n, c, h, w = ring.shape
    _step_state(name, None, lr_curr, lr_prev, hr_prev, scale)
    if tuple(lr_curr.shape) != (n, c, h, w):
        raise L.TecoganB200Error(f'{name}: lr_curr {tuple(lr_curr.shape)} is not [n={n},c={c},h={h},w={w}]')
    if warm_hr is not None:
        _req(warm_hr, torch.float32, 'warm_hr', 4)
        if warm_hr.shape != hr_prev.shape:
            raise L.TecoganB200Error(f'{name}: warm_hr {tuple(warm_hr.shape)} != hr_prev {tuple(hr_prev.shape)}')
    _req(table, torch.int32, 'table', 1)
    if table.shape[0] != 3 * n:
        raise L.TecoganB200Error(f'{name}: table has {table.shape[0]} entries, expected {3 * n}')
    _same_device(name, ring, table, warm_hr, lr_curr, lr_prev, hr_prev)
    L.check(L.load().tg_stream_gather(_ptr(ring), depth, _ptr(table), _ptr(warm_hr), _ptr(lr_curr), _ptr(lr_prev),
                                      _ptr(hr_prev), n, c, h, w, scale, _stream()), 'tg_stream_gather')
    return lr_curr


def _yuv_layout(layout, name):
    if layout not in YUV420_LAYOUTS:
        raise L.TecoganB200Error(f'{name}: layout must be one of {YUV420_LAYOUTS}, got {layout!r}')
    return int(layout == 'nv12')


def stream_frame_in_yuv420(yuv, layout, reset, lr_curr, lr_prev, hr_prev, scale):
    """stream_frame_in from YUV 4:2:0 frames (tg_stream_frame_in_yuv420): yuv uint8 [n,3h/2,w] in layout 'nv12' or
    'i420' (or None) -> lr_curr fp32 [n,3,h,w] = cv2.cvtColor(frame, COLOR_YUV2RGB_<layout>) / 255; reset as in
    stream_frame_in."""
    name = 'stream_frame_in_yuv420'
    nv12 = _yuv_layout(layout, name)
    n, c, h, w = _step_state(name, reset, lr_curr, lr_prev, hr_prev, scale)
    _frames(name, yuv, layout, n, c, h, w, None)
    _same_device(name, lr_curr, lr_prev, hr_prev, yuv, reset)
    L.check(L.load().tg_stream_frame_in_yuv420(_ptr(yuv), nv12, _ptr(reset), _ptr(lr_curr), _ptr(lr_prev),
                                               _ptr(hr_prev), n, h, w, scale, _stream()), 'tg_stream_frame_in_yuv420')
    return lr_curr


def rgb_u8_to_yuv420(rgb, layout, out=None):
    """tg_rgb_u8_to_yuv420: uint8 NHWC RGB [n,H,W,3] -> uint8 [n,3H/2,W] in layout 'nv12' or 'i420'
    (== cv2.cvtColor(rgb, COLOR_RGB2YUV_I420), U and V interleaved for 'nv12')."""
    nv12 = _yuv_layout(layout, 'rgb_u8_to_yuv420')
    _req(rgb, torch.uint8, 'rgb', 4)
    n, H, W, c = rgb.shape
    if c != 3:
        raise L.TecoganB200Error(f'rgb_u8_to_yuv420: expected [n,H,W,3] RGB, got {tuple(rgb.shape)}')
    if H % 2 or W % 2:
        raise L.TecoganB200Error(f'rgb_u8_to_yuv420: YUV 4:2:0 needs an even height and width, got {H}x{W}')
    if out is None:
        out = torch.empty((n, 3 * H // 2, W), dtype=torch.uint8, device=rgb.device)
    _req(out, torch.uint8, 'out', 3)
    if tuple(out.shape) != (n, 3 * H // 2, W):
        raise L.TecoganB200Error(f'rgb_u8_to_yuv420: out {tuple(out.shape)} != {(n, 3 * H // 2, W)}')
    if out.device != rgb.device:
        raise L.TecoganB200Error('rgb_u8_to_yuv420: tensors on different devices')
    L.check(L.load().tg_rgb_u8_to_yuv420(_ptr(rgb), _ptr(out), nv12, n, H, W, _stream()), 'tg_rgb_u8_to_yuv420')
    return out


def v210_stride(w):
    """Bytes per row of a v210 frame w pixels wide: 128 * ceil(w / 48) (ceil(w / 6) 16-byte groups of 6 pixels,
    padded to 128 bytes)."""
    return 128 * (-(-w // 48))


# What a YUV layout is, on the host: C code, bit depth, word dtype, the words (a, b) of an h x w frame (shape) and
# its inverse (size; v210 rows do not give w, which needs_width says must be passed), the (row, column) steps of a
# picture's origin (grid) and size (size_grid), and the shape text of a stack of its frames.
_Layout = collections.namedtuple('_Layout', 'code depth dtype shape size grid size_grid needs_width text')
_420, _422, _444 = (2, 2), (1, 2), (1, 1)
_P420 = (lambda h, w: (3 * h // 2, w), lambda a, b: (2 * a // 3, b), _420, _420, False, '3h/2,w')
_PACKED422 = (lambda h, w: (h, 2 * w), lambda a, b: (a, b // 2), _422, _422, False, 'h,2w')
_P444 = (lambda h, w: (3 * h, w), lambda a, b: (a // 3, b), _444, _444, False, '3h,w')
_P422 = (lambda h, w: (2 * h, w), lambda a, b: (a // 2, b), _422, _422, False, '2h,w')
# a v210 picture starts on a 6-pixel group and has an even width; it ends on a group or at the frame's right edge
_V210 = (lambda h, w: (h, v210_stride(w)), None, (1, 6), _422, True, 'h,128*ceil(w/48)')
YUV_LAYOUT_TABLE = {
    'nv12': _Layout(L.YUV_NV12, 8, torch.uint8, *_P420),
    'i420': _Layout(L.YUV_I420, 8, torch.uint8, *_P420),
    'p010': _Layout(L.YUV_P010, 10, torch.uint16, *_P420),
    'i420_10': _Layout(L.YUV_I420_10, 10, torch.uint16, *_P420),
    'yuy2': _Layout(L.YUV_YUY2, 8, torch.uint8, *_PACKED422),
    'uyvy': _Layout(L.YUV_UYVY, 8, torch.uint8, *_PACKED422),
    'i444': _Layout(L.YUV_I444, 8, torch.uint8, *_P444),
    'i444_10': _Layout(L.YUV_I444_10, 10, torch.uint16, *_P444),
    # P210 / I422_10: the Y plane, then the interleaved UV plane / the U and V planes of h x w/2; v210: 6 pixels
    # per 16-byte group, rows padded to 128 bytes
    'p210': _Layout(L.YUV_P210, 10, torch.uint16, *_P422),
    'i422_10': _Layout(L.YUV_I422_10, 10, torch.uint16, *_P422),
    'v210': _Layout(L.YUV_V210, 10, torch.uint8, *_V210),
}
YUV_LAYOUTS = tuple(YUV_LAYOUT_TABLE)          # 4:2:0, then 4:2:2 and 4:4:4, then 10-bit 4:2:2
_LAYOUT_CODE = {k: v.code for k, v in YUV_LAYOUT_TABLE.items()}
YUV420_LAYOUTS = tuple(k for k, v in YUV_LAYOUT_TABLE.items() if v.grid == _420 and v.depth == 8)
YUV422_LAYOUTS = tuple(k for k, v in YUV_LAYOUT_TABLE.items() if v.grid == _422 and v.depth == 8)   # packed
YUV444_LAYOUTS = tuple(k for k, v in YUV_LAYOUT_TABLE.items() if v.grid == _444)
YUV422_10_LAYOUTS = tuple(k for k, v in YUV_LAYOUT_TABLE.items() if v.size_grid == _422 and v.depth == 10)
YUV_COLORS = ('bt601', 'bt709', 'bt601-full', 'bt709-full')


def yuv_depth(layout):
    """Bit depth of a YUV layout: 8 or 10."""
    return YUV_LAYOUT_TABLE[layout].depth


def yuv_word_dtype(layout):
    """The dtype of a YUV layout's frames: uint16 for the 10-bit layouts, uint8 for the 8-bit ones and for v210,
    whose 10-bit samples are packed into bytes."""
    return YUV_LAYOUT_TABLE[layout].dtype


def yuv_frame_shape(layout, h, w):
    """The words of one h x w frame: (3h/2, w) for 4:2:0, (h, 2w) for packed 4:2:2, (3h, w) for planar 4:4:4,
    (2h, w) for P210 / I422_10 and (h, v210_stride(w)) bytes for v210."""
    return YUV_LAYOUT_TABLE[layout].shape(h, w)


def yuv_size_error(layout, h, w):
    """None if an h x w frame fits the layout's chroma subsampling, else why not: 4:2:0 needs an even height and
    width, 4:2:2 an even width, 4:4:4 any size."""
    sy, sx = YUV_LAYOUT_TABLE[layout].size_grid
    if sy == 2:
        return None if h % 2 == 0 and w % 2 == 0 else f'YUV 4:2:0 needs an even height and width, got {h}x{w}'
    return None if w % sx == 0 else f'YUV 4:2:2 needs an even width, got {w}'


def yuv_format(layout, color, name='yuv_format'):
    """(layout, colour) names -> struct tg_yuv_format."""
    if layout not in YUV_LAYOUTS:
        raise L.TecoganB200Error(f'{name}: layout must be one of {YUV_LAYOUTS}, got {layout!r}')
    if color not in YUV_COLORS:
        raise L.TecoganB200Error(f'{name}: colour must be one of {YUV_COLORS}, got {color!r}')
    return L.YuvFormat(_LAYOUT_CODE[layout], 709 if color.startswith('bt709') else 601,
                       int(color.endswith('-full')), 0)


def yuv_coefficients(layout, color):
    """tg_yuv_coefficients: the 16 int32 of the kernels' colour table row (host only, no GPU needed)."""
    out = (ctypes.c_int32 * 16)()
    L.check(L.load().tg_yuv_coefficients(ctypes.byref(yuv_format(layout, color, 'yuv_coefficients')), out),
            'tg_yuv_coefficients')
    return list(out)


def yuv_frame_size(layout, shape, w=None):
    """(h, w) of a frame whose words have the 2-d shape `shape` in a YUV layout (yuv_frame_shape's inverse).  A v210
    row's bytes do not give its width (rows are padded to 128 bytes): w must be given; for the other layouts a w
    that is given must be the shape's."""
    a, b = shape
    lay = YUV_LAYOUT_TABLE[layout]
    if lay.needs_width:
        if w is None:
            raise L.TecoganB200Error(f'{layout} frames do not give their width (rows are padded to 128 bytes): pass it '
                                     '(frame_w)')
        return a, int(w)
    hw = lay.size(a, b)
    if w is not None and int(w) != hw[1]:
        raise L.TecoganB200Error(f'{layout} frames of shape {tuple(shape)} are {hw[1]} wide, not {w}')
    return hw


def stream_frame_in_yuv(frames, layout, color, reset, lr_curr, lr_prev, hr_prev, scale, window=None):
    """tg_stream_frame_in_yuv: frames [n,*yuv_frame_shape(layout, h, w)] (uint8 for the 8-bit layouts, uint16 for
    'p010' / 'i420_10' / 'i444_10'; or None) in colour `color` -> lr_curr fp32 [n,3,h,w] = RGB / 255 (8 bit) or
    RGB / 1023 (10 bit), as oracle/yuv_color.py (4:2:0) and oracle/yuv_422_444.py (4:2:2, 4:4:4) specify; reset as
    in stream_frame_in.  With window = (top, left), frames hold Hf x Wf frames (frames.shape[1:] ==
    yuv_frame_shape(layout, Hf, Wf)) and the h x w picture at (top, left) is read (tg_stream_frame_in_yuv_window);
    a v210 window is (top, left, Wf): its frames' rows do not give Wf."""
    name = 'stream_frame_in_yuv' if window is None else 'stream_frame_in_yuv_window'
    fmt = yuv_format(layout, color, name)
    window, frame_w = _split_window(name, layout, window)
    n, c, h, w = _step_state(name, reset, lr_curr, lr_prev, hr_prev, scale)
    fh, fw = _frames(name, frames, layout, n, c, h, w, window, frame_w)
    _same_device(name, lr_curr, lr_prev, hr_prev, frames, reset)
    if window is not None:
        win = frame_window(fh, fw, *window) if frames is not None else frame_window(h, w, 0, 0)
        L.check(L.load().tg_stream_frame_in_yuv_window(_ptr(frames), ctypes.byref(fmt), ctypes.byref(win),
                                                       _ptr(reset), _ptr(lr_curr), _ptr(lr_prev), _ptr(hr_prev), n,
                                                       h, w, scale, _stream()), 'tg_stream_frame_in_yuv_window')
        return lr_curr
    L.check(L.load().tg_stream_frame_in_yuv(_ptr(frames), ctypes.byref(fmt), _ptr(reset), _ptr(lr_curr),
                                            _ptr(lr_prev), _ptr(hr_prev), n, h, w, scale, _stream()),
            'tg_stream_frame_in_yuv')
    return lr_curr


def rgb_to_yuv(layout, color, rgb_u8=None, rgb_f32=None, out=None, window=None):
    """tg_rgb_to_yuv: 8-bit layouts encode rgb_u8 (uint8 NHWC [n,H,W,3]) into uint8 [n,*yuv_frame_shape]; 10-bit
    layouts encode rgb_f32 (fp32 NCHW [n,3,H,W], quantised as clip(rint(x * 1023), 0, 1023)) into uint16
    [n,*yuv_frame_shape] ([n,3H/2,W] for 4:2:0, [n,H,2W] for 4:2:2, [n,3H,W] for 4:4:4).  With window = (top, left),
    out holds larger Hf x Wf frames and the H x W picture is written at (top, left) of each (tg_rgb_to_yuv_window);
    the words around it are left as they are.  'p210' / 'i422_10' are [n,2H,W] uint16 and 'v210' [n,H,v210_stride(W)]
    uint8, all three 10-bit (from rgb_f32); a v210 window is (top, left, Wf).  A whole-frame v210 encode writes every
    byte of each row (the fields past the last pixel and the row padding 0), a windowed one the picture's groups."""
    name = 'rgb_to_yuv' if window is None else 'rgb_to_yuv_window'
    fmt = yuv_format(layout, color, name)
    window, frame_w = _split_window(name, layout, window)
    ten = yuv_depth(layout) == 10
    if ten:
        if rgb_f32 is None or rgb_u8 is not None:
            raise L.TecoganB200Error(f'{name}: 10-bit {layout} is encoded from rgb_f32 (fp32 NCHW) only')
        src = _req(rgb_f32, torch.float32, 'rgb_f32', 4)
        n, c, H, W = src.shape
    else:
        if rgb_u8 is None or rgb_f32 is not None:
            raise L.TecoganB200Error(f'{name}: 8-bit {layout} is encoded from rgb_u8 (uint8 NHWC) only')
        src = _req(rgb_u8, torch.uint8, 'rgb_u8', 4)
        n, H, W, c = src.shape
    if c != 3:
        raise L.TecoganB200Error(f'{name}: expected 3 colour channels, got {tuple(src.shape)}')
    err = yuv_size_error(layout, H, W)
    if err:
        raise L.TecoganB200Error(f'{name}: {err}')
    dtype = yuv_word_dtype(layout)
    if window is not None and out is None:
        raise L.TecoganB200Error(f'{name}: a window needs the output frames (out)')
    fh, fw = (H, W) if window is None else yuv_frame_size(layout, out.shape[1:], frame_w)
    shape = (n, *yuv_frame_shape(layout, fh, fw))
    if out is None:
        out = torch.empty(shape, dtype=dtype, device=src.device)
    _req(out, dtype, 'out', 3)
    if tuple(out.shape) != shape:
        raise L.TecoganB200Error(f'{name}: out {tuple(out.shape)} != {shape}')
    if out.device != src.device:
        raise L.TecoganB200Error(f'{name}: tensors on different devices')
    if window is not None:
        win = frame_window(fh, fw, *window)
        L.check(L.load().tg_rgb_to_yuv_window(_ptr(rgb_u8), _ptr(rgb_f32), _ptr(out), ctypes.byref(fmt),
                                              ctypes.byref(win), n, H, W, _stream()), 'tg_rgb_to_yuv_window')
        return out
    L.check(L.load().tg_rgb_to_yuv(_ptr(rgb_u8), _ptr(rgb_f32), _ptr(out), ctypes.byref(fmt), n, H, W, _stream()),
            'tg_rgb_to_yuv')
    return out


def fill_black(out, layout=None, color='bt601'):
    """tg_fill_black: every word of out := the format's black.  layout None: uint8 HWC [n,Hf,Wf,c], all 0; else the
    YUV layout's frames [n,*yuv_frame_shape(layout, Hf, Wf)] with Y = the colour's black level (16 << (depth - 8)
    limited range, 0 full) and U = V = 128 << (depth - 8), P010 / P210 words << 6.  v210: fill_black_v210."""
    if layout == 'v210':
        raise L.TecoganB200Error('fill_black: v210 frames do not give their width: use fill_black_v210(out, color, '
                                 'frame_w)')
    return _fill_black(out, layout, color, None)


def fill_black_v210(out, color, frame_w):
    """tg_fill_black of v210 frames out [n,Hf,v210_stride(frame_w)] (uint8), whose rows do not give their width:
    Y = the colour's black level (64 limited range, 0 full) and U = V = 512 in the fields of the frame_w pixels, 0 in
    the rest of each row."""
    return _fill_black(out, 'v210', color, frame_w)


def _yuv_stack(name, t, arg, layout, frame_w):
    """(fh, fw) of the frames of t, a stack [n,*yuv_frame_shape(layout, fh, fw)] of a YUV layout's frames."""
    _req(t, yuv_word_dtype(layout), arg, 3)
    fh, fw = yuv_frame_size(layout, t.shape[1:], frame_w)
    if tuple(t.shape[1:]) != yuv_frame_shape(layout, fh, fw):
        raise L.TecoganB200Error(f'{name}: {tuple(t.shape)} is not a stack of {layout} frames')
    return fh, fw


def _fill_black(out, layout, color, frame_w):
    fmt = None
    if layout is None:
        _req(out, torch.uint8, 'out', 4)
        n, fh, fw, c = out.shape
    else:
        fmt = yuv_format(layout, color, 'fill_black')
        (fh, fw), n, c = _yuv_stack('fill_black', out, 'out', layout, frame_w), out.shape[0], 3
    L.check(L.load().tg_fill_black(_ptr(out), ctypes.byref(fmt) if fmt is not None else None, n, c, fh, fw,
                                   _stream()), 'tg_fill_black')
    return out


def luma_line_sums(frames, layout=None, bgr=False, frame_w=None):
    """tg_luma_line_sums: the per-row and per-column sums of the 8-bit luma of frames (uint8 HWC RGB [n,h,w,3], or a
    YUV layout's [n,*yuv_frame_shape]; v210 frames are frame_w wide) as int64 tensors rows [n,h], cols [n,w] on the
    frames' device."""
    fmt = None
    if layout is None:
        _req(frames, torch.uint8, 'frames', 4)
        n, h, w, c = frames.shape
    else:
        fmt = yuv_format(layout, 'bt601', 'luma_line_sums')
        (h, w), n, c = _yuv_stack('luma_line_sums', frames, 'frames', layout, frame_w), frames.shape[0], 3
    rows = torch.empty((n, h), dtype=torch.int64, device=frames.device)
    cols = torch.empty((n, w), dtype=torch.int64, device=frames.device)
    L.check(L.load().tg_luma_line_sums(_ptr(frames), ctypes.byref(fmt) if fmt is not None else None, int(bool(bgr)),
                                       n, c, h, w, _ptr(rows), _ptr(cols), _stream()), 'tg_luma_line_sums')
    return rows, cols


RESIZE_FILTERS = ('bicubic', 'lanczos')
_FILTER_CODE = {'bicubic': L.RESAMPLE_BICUBIC, 'lanczos': L.RESAMPLE_LANCZOS3}


def resample_ratio_ok(n_in, n_out):
    """The resize supports in/4 <= out <= 2*in on each axis."""
    return n_in > 0 and n_out > 0 and 4 * n_out >= n_in and n_out <= 2 * n_in


def resample_table(n_in, n_out, filt='bicubic'):
    """tg_resample_table (host only, no GPU needed): the kernel's table of one axis, (first int32 [out],
    weights fp32 [out, taps]) as CPU tensors; oracle/resample.py's table rounded to fp32."""
    if filt not in _FILTER_CODE:
        raise L.TecoganB200Error(f'resample_table: filter must be one of {RESIZE_FILTERS}, got {filt!r}')
    lib = L.load()
    taps = ctypes.c_int(0)
    L.check(lib.tg_resample_taps(int(n_in), int(n_out), _FILTER_CODE[filt], ctypes.byref(taps)), 'tg_resample_taps')
    first = torch.empty(n_out, dtype=torch.int32)
    weights = torch.empty(n_out, taps.value, dtype=torch.float32)
    L.check(lib.tg_resample_table(int(n_in), int(n_out), _FILTER_CODE[filt], taps.value, _ptr(first), _ptr(weights)),
            'tg_resample_table')
    return first, weights


def resample(x, rows, cols, out_u8=None, out_f32=None, window=None):
    """tg_resample_nchw_f32: x fp32 NCHW [n,c,H,W] resized with the device tables rows = (first [Ho], weights
    [Ho, taps]) and cols = (first [Wo], weights [Wo, taps]) into exactly one of out_u8 (uint8 NHWC [n,Ho,Wo,c],
    float32_to_uint8 of the result) or out_f32 (fp32 NCHW [n,c,Ho,Wo]).  With neither given, a new uint8 tensor.
    With window = (top, left), out_u8 is [n,Hf,Wf,c] and the picture is written at (top, left) of each frame."""
    name = 'resample'
    _req(x, torch.float32, 'x', 4)
    n, c, H, W = x.shape
    tabs = []
    for axis, (first, weights), n_in in (('rows', rows, H), ('cols', cols, W)):
        _req(first, torch.int32, f'{axis} first', 1)
        _req(weights, torch.float32, f'{axis} weights', 2)
        if weights.shape[0] != first.shape[0]:
            raise L.TecoganB200Error(f'{name}: {axis} first {tuple(first.shape)} and weights '
                                     f'{tuple(weights.shape)} disagree')
        if first.device != x.device or weights.device != x.device:
            raise L.TecoganB200Error(f'{name}: tensors on different devices')
        if not resample_ratio_ok(n_in, first.shape[0]):
            raise L.TecoganB200Error(f'{name}: {axis} {n_in} -> {first.shape[0]} outside in/4 <= out <= 2*in')
        tabs.append((first, weights, weights.shape[1]))
    Ho, Wo = rows[0].shape[0], cols[0].shape[0]
    if out_u8 is not None and out_f32 is not None:
        raise L.TecoganB200Error(f'{name}: give out_u8 or out_f32, not both')
    if out_f32 is None and out_u8 is None:
        out_u8 = torch.empty((n, Ho, Wo, c), dtype=torch.uint8, device=x.device)
    if window is not None and out_u8 is None:
        raise L.TecoganB200Error(f'{name}: a window applies to the uint8 output (out_u8)')
    if out_u8 is not None:
        out, want = _req(out_u8, torch.uint8, 'out_u8', 4), (n, Ho, Wo, c)
        if window is not None:
            want = (n, out.shape[1], out.shape[2], c)
    else:
        out, want = _req(out_f32, torch.float32, 'out_f32', 4), (n, c, Ho, Wo)
    if tuple(out.shape) != want:
        raise L.TecoganB200Error(f'{name}: out {tuple(out.shape)} != {want}')
    if out.device != x.device:
        raise L.TecoganB200Error(f'{name}: tensors on different devices')
    (rf, rw, rt), (cf, cw, ct) = tabs
    if window is not None:
        win = frame_window(out.shape[1], out.shape[2], *window)
        L.check(L.load().tg_resample_nchw_f32_window(_ptr(x), n, c, H, W, _ptr(rf), _ptr(rw), rt, _ptr(cf), _ptr(cw),
                                                     ct, Ho, Wo, _ptr(out_u8), ctypes.byref(win), _stream()),
                'tg_resample_nchw_f32_window')
        return out
    L.check(L.load().tg_resample_nchw_f32(_ptr(x), n, c, H, W, _ptr(rf), _ptr(rw), rt, _ptr(cf), _ptr(cw), ct, Ho, Wo,
                                          _ptr(out_u8), _ptr(out_f32), _stream()), 'tg_resample_nchw_f32')
    return out


def stream_frame_in_resample(frames, layout, color, reset, lr_curr, lr_prev, hr_prev, scale, rows, cols, size,
                             bgr=False, window=None):
    """tg_stream_frame_in_resample: the frame input (stream_frame_in / stream_frame_in_yuv) of the size = (h, w)
    source picture, resized on the device with the device tables rows = (first [hn], weights [hn, taps]) (h -> hn)
    and cols = (first [wn], weights [wn, taps]) (w -> wn) into lr_curr fp32 [n,c,hn,wn], in one launch; bit for bit
    the frame input at h x w followed by resample(..., out_f32=lr_curr).  frames: uint8 HWC [n,Hf,Wf,c] (layout None,
    channels reversed when bgr) or a YUV layout's [n,*yuv_frame_shape(layout, Hf, Wf)] in colour `color`; the picture
    is the whole frame, or the h x w one at window = (top, left) ((top, left, Wf) for v210).  reset as in
    stream_frame_in (lr_prev [n,c,hn,wn], hr_prev [n,c,scale*hn,scale*wn])."""
    name = 'stream_frame_in_resample'
    fmt = None if layout is None else yuv_format(layout, color, name)
    n, c, hn, wn = _step_state(name, reset, lr_curr, lr_prev, hr_prev, scale)
    h, w = (int(v) for v in size)
    window, frame_w = _split_window(name, layout, window)
    fh, fw = _frames(name, frames, layout, n, c, h, w, window, frame_w)
    tabs = []
    for axis, (first, weights), n_in, n_out in (('rows', rows, h, hn), ('cols', cols, w, wn)):
        _req(first, torch.int32, f'{axis} first', 1)
        _req(weights, torch.float32, f'{axis} weights', 2)
        if first.shape[0] != n_out or weights.shape[0] != n_out:
            raise L.TecoganB200Error(f'{name}: {axis} tables {tuple(first.shape)} / {tuple(weights.shape)} do not '
                                     f'give {n_out} outputs')
        if not resample_ratio_ok(n_in, n_out):
            raise L.TecoganB200Error(f'{name}: {axis} {n_in} -> {n_out} outside in/4 <= out <= 2*in')
        tabs.append((first, weights, weights.shape[1]))
    _same_device(name, lr_curr, lr_prev, hr_prev, frames, reset, *rows, *cols)
    win = frame_window(fh, fw, *(window or (0, 0)))
    (rf, rw, rt), (cf, cw, ct) = tabs
    L.check(L.load().tg_stream_frame_in_resample(_ptr(frames), ctypes.byref(fmt) if fmt is not None else None,
                                                 int(bool(bgr)), ctypes.byref(win), h, w, _ptr(rf), _ptr(rw), rt,
                                                 _ptr(cf), _ptr(cw), ct, _ptr(reset), _ptr(lr_curr), _ptr(lr_prev),
                                                 _ptr(hr_prev), n, c, hn, wn, scale, _stream()),
            'tg_stream_frame_in_resample')
    return lr_curr


def scene_cut_threshold_ok(threshold):
    """tg_scene_cut takes a finite threshold in (0, 100]."""
    return 0.0 < threshold <= 100.0


def scene_cut_work(n, device):
    """The zeroed workspace of tg_scene_cut for n slots (each launch leaves it zeroed again)."""
    return torch.zeros(n * L.SCENE_CUT_WORK_BYTES // 8, dtype=torch.int64, device=device)


def scene_cut(lr_curr, lr_prev, reset, threshold, prev_mafd, work, score, cut):
    """tg_scene_cut: per slot k of lr_curr / lr_prev (fp32 [n,c,h,w]), score[k] (float64) and cut[k] (int32 0 / 1)
    of oracle/scene_cut.py, with prev_mafd (float64 [n]) the state it updates and reset (int32 [n], or None) the
    caller's resets of this step.  work: scene_cut_work(n) (int64 tensor of n * SCENE_CUT_WORK_BYTES bytes)."""
    name = 'scene_cut'
    _req(lr_curr, torch.float32, 'lr_curr', 4)
    _req(lr_prev, torch.float32, 'lr_prev', 4)
    n, c, h, w = lr_curr.shape
    if tuple(lr_prev.shape) != (n, c, h, w):
        raise L.TecoganB200Error(f'{name}: lr_prev {tuple(lr_prev.shape)} != lr_curr {(n, c, h, w)}')
    for t, dtype, nm in ((prev_mafd, torch.float64, 'prev_mafd'), (score, torch.float64, 'score'),
                         (cut, torch.int32, 'cut'), (reset, torch.int32, 'reset')):
        if t is None and nm == 'reset':
            continue
        _req(t, dtype, nm, 1)
        if t.shape[0] != n:
            raise L.TecoganB200Error(f'{name}: {nm} has {t.shape[0]} entries, expected {n}')
    _req(work, torch.int64, 'work', 1)
    if work.numel() * 8 != n * L.SCENE_CUT_WORK_BYTES:
        raise L.TecoganB200Error(f'{name}: work has {work.numel() * 8} bytes, expected {n * L.SCENE_CUT_WORK_BYTES}')
    _same_device(name, lr_curr, lr_prev, reset, prev_mafd, work, score, cut)
    L.check(L.load().tg_scene_cut(_ptr(lr_curr), _ptr(lr_prev), n, c, h, w, _ptr(reset), float(threshold),
                                  _ptr(prev_mafd), _ptr(work), _ptr(score), _ptr(cut), _stream()), 'tg_scene_cut')
    return score, cut


def metrics_frames_in(true_u8, pred_u8, psnr, gray):
    """tg_metrics_frames_in: true_u8 [t,ht,wt,3] / pred_u8 [t,hp,wp,3] uint8 (pred_u8 None: gray of true_u8 only),
    psnr one of L.PSNR_NONE / PSNR_RGB / PSNR_Y, gray uint8 [2,t,h,w] ([t,h,w] without pred_u8) or None.
    -> the per-frame integer SSE (int64 [t] holding the uint64 sums), or None without PSNR."""
    name = 'metrics_frames_in'
    _req(true_u8, torch.uint8, 'true_u8', 4)
    t, ht, wt, c = true_u8.shape
    hp = wp = 0
    if pred_u8 is not None:
        _req(pred_u8, torch.uint8, 'pred_u8', 4)
        if pred_u8.shape[0] != t or pred_u8.shape[3] != 3:
            raise L.TecoganB200Error(f'{name}: pred {tuple(pred_u8.shape)} does not match true {tuple(true_u8.shape)}')
        hp, wp = pred_u8.shape[1:3]
    if c != 3:
        raise L.TecoganB200Error(f'{name}: expected RGB frames [t,h,w,3], got {tuple(true_u8.shape)}')
    h, w = (min(ht, hp), min(wt, wp)) if pred_u8 is not None else (ht, wt)
    if gray is not None:
        _req(gray, torch.uint8, 'gray')
        want = (2, t, h, w) if pred_u8 is not None else (t, h, w)
        if tuple(gray.shape) != want:
            raise L.TecoganB200Error(f'{name}: gray {tuple(gray.shape)}, expected {want}')
    sse = torch.empty(t, dtype=torch.int64, device=true_u8.device) if psnr != L.PSNR_NONE else None
    for x in (pred_u8, gray):
        if x is not None and x.device != true_u8.device:
            raise L.TecoganB200Error(f'{name}: tensors on different devices')
    L.check(L.load().tg_metrics_frames_in(_ptr(true_u8), ht, wt, _ptr(pred_u8), hp, wp, t, psnr, _ptr(gray),
                                          _ptr(sse), _stream()), 'tg_metrics_frames_in')
    return sse


def farneback_params(pyr_scale, levels, winsize, iterations, poly_n, poly_sigma, flags):
    return L.FarnebackParams(float(pyr_scale), int(levels), int(winsize), int(iterations), int(poly_n),
                             float(poly_sigma), int(flags), 0)


def farneback_workspace_bytes(groups, t, h, w):
    """bytes of tg_farneback's workspace for `groups` groups of t frames of h x w"""
    return int(L.load().tg_farneback_workspace_bytes(groups, t, h, w))


def farneback(gray, groups, params, work=None):
    """tg_farneback: gray uint8 [groups*t, h, w] -> fp32 flows [groups*(t-1), h, w, 2] of the consecutive pairs of
    each group of t frames.  work: a uint8 CUDA tensor of at least farneback_workspace_bytes (allocated if None)."""
    _req(gray, torch.uint8, 'gray', 3)
    n, h, w = gray.shape
    if groups <= 0 or n % groups or n // groups < 2:
        raise L.TecoganB200Error(f'farneback: {n} frames do not make {groups} groups of at least 2')
    t = n // groups
    need = farneback_workspace_bytes(groups, t, h, w)
    if work is None:
        work = torch.empty(need, dtype=torch.uint8, device=gray.device)
    _req(work, torch.uint8, 'work', 1)
    flow = torch.empty(groups * (t - 1), h, w, 2, dtype=torch.float32, device=gray.device)
    L.check(L.load().tg_farneback(_ptr(gray), groups, t, h, w, ctypes.byref(params), _ptr(flow), _ptr(work),
                                  work.numel(), _stream()), 'tg_farneback')
    return flow


def flow_epe_sum(a, b, window=None):
    """tg_flow_epe_sum: fp32 flows a, b [n,h,w,2] -> float64 [n], the per-pair sum of |a - b| over the pixels, or
    (tg_flow_epe_sum_window) over the window (y0, x0, hc, wc) of them, summed in a fixed order"""
    _req(a, torch.float32, 'a', 4)
    _req(b, torch.float32, 'b', 4)
    if a.shape != b.shape or a.shape[3] != 2:
        raise L.TecoganB200Error(f'flow_epe_sum: shapes {tuple(a.shape)} / {tuple(b.shape)}')
    n, h, w, _ = a.shape
    sums = torch.empty(n, dtype=torch.float64, device=a.device)
    if window is None:
        L.check(L.load().tg_flow_epe_sum(_ptr(a), _ptr(b), n, h, w, _ptr(sums), _stream()), 'tg_flow_epe_sum')
    else:
        need = int(L.load().tg_flow_epe_sum_window_workspace_bytes(n, window[2]))
        work = torch.empty(max(need, 8) // 8, dtype=torch.float64, device=a.device)
        L.check(L.load().tg_flow_epe_sum_window(_ptr(a), _ptr(b), n, h, w, *window, _ptr(sums), _ptr(work), need,
                                                _stream()), 'tg_flow_epe_sum_window')
    return sums


def _official_frames(name, true_u8, pred_u8):
    _req(true_u8, torch.uint8, 'true_u8', 4)
    _req(pred_u8, torch.uint8, 'pred_u8', 4)
    if true_u8.shape[0] != pred_u8.shape[0] or true_u8.shape[3] != 3 or pred_u8.shape[3] != 3:
        raise L.TecoganB200Error(f'{name}: expected RGB frames [t,h,w,3] of one length, got {tuple(true_u8.shape)} / '
                                 f'{tuple(pred_u8.shape)}')
    _same_device(name, true_u8, pred_u8)
    t, ht, wt, _ = true_u8.shape
    return (t, ht, wt) + tuple(pred_u8.shape[1:3])


def official_frames_stats_workspace_bytes(t, hc, wc):
    return int(L.load().tg_official_frames_stats_workspace_bytes(t, hc, wc))


def ssim_y_workspace_bytes(t, hc, wc):
    return int(L.load().tg_ssim_y_workspace_bytes(t, hc, wc))


def official_frames_stats(true_u8, pred_u8, window):
    """tg_official_frames_stats: uint8 RGB true_u8 [t,ht,wt,3] / pred_u8 [t,hp,wp,3], window (y0, x0, hc, wc) of the
    common size -> float64 [t, 3]: {sum (Yt - Yp)^2, min Yp, max Yp} per frame"""
    t, ht, wt, hp, wp = _official_frames('official_frames_stats', true_u8, pred_u8)
    stats = torch.empty(t, 3, dtype=torch.float64, device=true_u8.device)
    need = official_frames_stats_workspace_bytes(t, *window[2:])
    work = torch.empty(max(need, 8) // 8, dtype=torch.float64, device=true_u8.device)
    L.check(L.load().tg_official_frames_stats(_ptr(true_u8), ht, wt, _ptr(pred_u8), hp, wp, t, *window, _ptr(stats),
                                              _ptr(work), need, _stream()), 'tg_official_frames_stats')
    return stats


def ssim_y(true_u8, pred_u8, window, stats):
    """tg_ssim_y: SSIM of the Y over the window (y0, x0, hc, wc) -> float64 [t], with data_range from stats
    (official_frames_stats's output, float64 [t, 3] on the device)"""
    t, ht, wt, hp, wp = _official_frames('ssim_y', true_u8, pred_u8)
    _req(stats, torch.float64, 'stats', 2)
    if tuple(stats.shape) != (t, 3):
        raise L.TecoganB200Error(f'ssim_y: stats {tuple(stats.shape)}, expected {(t, 3)}')
    _same_device('ssim_y', true_u8, stats)
    out = torch.empty(t, dtype=torch.float64, device=true_u8.device)
    need = ssim_y_workspace_bytes(t, *window[2:])
    work = torch.empty(max(need, 8) // 8, dtype=torch.float64, device=true_u8.device)
    L.check(L.load().tg_ssim_y(_ptr(true_u8), ht, wt, _ptr(pred_u8), hp, wp, t, *window, _ptr(stats), _ptr(out),
                               _ptr(work), need, _stream()), 'tg_ssim_y')
    return out


def lpips_frames_in(frames, window, norm, out):
    """tg_lpips_frames_in: uint8 RGB frames [t, H, W, 3], window (y0, x0, h, w) of them, norm L.LPIPS_NORM_* ->
    out fp16 [t, (h-7)//4 + 3, (w-7)//4 + 3, 64], conv1's space-to-depth input"""
    _req(frames, torch.uint8, 'frames', 4)
    t, fh, fw, c = frames.shape
    y0, x0, h, w = window
    _req(out, torch.float16, 'out', 4)
    if c != 3 or tuple(out.shape) != (t, (h - 7) // 4 + 3, (w - 7) // 4 + 3, 64):
        raise L.TecoganB200Error(f'lpips_frames_in: frames {tuple(frames.shape)}, out {tuple(out.shape)}')
    _same_device('lpips_frames_in', frames, out)
    win = L.FrameWindow(fh, fw, y0, x0)
    L.check(L.load().tg_lpips_frames_in(_ptr(frames), ctypes.byref(win), t, h, w, norm, _ptr(out), _stream()),
            'tg_lpips_frames_in')
    return out


def maxpool3x3s2(x, interior, shifts, y=None):
    """tg_maxpool3x3s2_nhwc_f16: MaxPool2d(3, 2) of the interior (y0, x0, h, w) of x fp16 [n, xh, xw, c] -> y
    [n, ph, pw, c], or with shifts conv2's four-shift input [n, ph+2, pw+2, 4c]"""
    _req(x, torch.float16, 'maxpool3x3s2 input', 4)
    n, xh, xw, c = x.shape
    y0, x0, h, w = interior
    ph, pw = (h - 3) // 2 + 1, (w - 3) // 2 + 1
    shape = (n, ph + 2, pw + 2, 4 * c) if shifts else (n, ph, pw, c)
    if y is None:
        y = torch.empty(shape, dtype=torch.float16, device=x.device)
    _req(y, torch.float16, 'maxpool3x3s2 output', 4)
    if tuple(y.shape) != shape:
        raise L.TecoganB200Error(f'maxpool3x3s2: output {tuple(y.shape)}, expected {shape}')
    _same_device('maxpool3x3s2', x, y)
    L.check(L.load().tg_maxpool3x3s2_nhwc_f16(_ptr(x), n, xh, xw, c, y0, x0, h, w, _ptr(y), 1 if shifts else 0,
                                             _stream()), 'tg_maxpool3x3s2_nhwc_f16')
    return y


def lpips_head_workspace_bytes(npairs, h, w):
    return int(L.load().tg_lpips_head_workspace_bytes(npairs, h, w))


def lpips_head(feat, interior, pairs, weights, out, accumulate):
    """tg_lpips_head: one LPIPS layer of the image pairs `pairs` (int32 [P, 2] on the device) of the features feat
    fp16 [n, xh, xw, c] over their interior (y0, x0, h, w), with the head weights fp32 [c]; out float64 [P] = (or +=,
    with accumulate) the layer's distance"""
    _req(feat, torch.float16, 'feat', 4)
    _req(pairs, torch.int32, 'pairs', 2)
    _req(weights, torch.float32, 'weights', 1)
    _req(out, torch.float64, 'out', 1)
    n, xh, xw, c = feat.shape
    P = pairs.shape[0]
    if pairs.shape[1] != 2 or out.shape[0] != P or weights.shape[0] != c:
        raise L.TecoganB200Error(f'lpips_head: pairs {tuple(pairs.shape)}, out {tuple(out.shape)}, weights '
                                 f'{tuple(weights.shape)} for {c} channels')
    _same_device('lpips_head', feat, pairs, weights, out)
    need = lpips_head_workspace_bytes(P, *interior[2:])
    work = torch.empty(max(need, 8) // 8, dtype=torch.float64, device=feat.device)
    L.check(L.load().tg_lpips_head(_ptr(feat), n, xh, xw, c, *interior, _ptr(pairs), P, _ptr(weights),
                                   1 if accumulate else 0, _ptr(out), _ptr(work), need, _stream()), 'tg_lpips_head')
    return out


# ============================================================================ training (backward) ops
class GradScale:
    """Device-resident loss scale {scale, 1/scale} of the fp16 gradient path (tg_grad_scale_from_amax /
    tg_flow_head_bwd choose it on the device -- no host round trip)."""

    TARGET = 256.0      # amax of the incoming gradient is scaled to ~2^8: 2^8 of headroom below fp16 max

    def __init__(self, device):
        self.ws = torch.zeros(4, dtype=torch.float32, device=device)       # 16 bytes, zeroed once

    def from_amax(self, a, b=None, target=None):
        _req(a, torch.float32, 'grad')
        if b is not None:
            _req(b, torch.float32, 'grad')
        L.check(L.load().tg_grad_scale_from_amax(_ptr(a), a.numel(), _ptr(b), b.numel() if b is not None else 0,
                                                 ctypes.c_float(target or self.TARGET), _ptr(self.ws), _stream()),
                'tg_grad_scale_from_amax')
        global LAUNCH_COUNT
        LAUNCH_COUNT += 1            # two kernels per call
        return self

    def from_amax_of(self, tensors, target=None):
        """one scale for several fp32 tensors: from the amax over all of them"""
        for t in tensors[:-1]:
            _req(t, torch.float32, 'grad')
            L.check(L.load().tg_grad_amax_f32(_ptr(t), t.numel(), _ptr(self.ws), _stream()), 'tg_grad_amax')
        return self.from_amax(tensors[-1], target=target)

    @property
    def ptr(self):
        return ctypes.c_void_p(self.ws.data_ptr())


def _scale_ptr(scale):
    return scale.ptr if scale is not None else ctypes.c_void_p(0)


class PackedDgrad:
    """Data-gradient operand of a conv layer: the same wgmma implicit GEMM with the roles of the
    channel dimensions swapped -- conv3x3: taps flipped (tg_pack_conv3x3_weights_dgrad); convT3x3s2: a
    stride-2 conv over the output gradient (TG_CONV_3X3_S2).  Built from the forward PackedConv."""

    def __init__(self, fwd, weight):
        self.fwd = fwd
        self.kind = L.CONV_3X3 if fwd.kind == L.CONV_3X3 else L.CONV_3X3_S2
        self.cin = pad64(fwd.cout_real)        # channels of dz
        self.cout = fwd.cin                    # channels of the input gradient (stored)
        self.packed = None
        self._ver = None
        self.refresh(weight)

    def refresh(self, weight, force=False):
        ver = (weight._version, weight.data_ptr())
        if ver == self._ver and not force:
            return
        lib = L.load()
        w = _req(weight.detach(), torch.float32, 'weight', 4)
        if self.packed is None:
            self.packed = torch.empty(lib.tg_packed_weight_bytes(self.cin, self.cout), dtype=torch.uint8, device=w.device)
            self.bias = torch.zeros(self.cout, dtype=torch.float32, device=w.device)
        f = self.fwd
        if self.kind == L.CONV_3X3:
            rc = lib.tg_pack_conv3x3_weights_dgrad(_ptr(w), f.cout_real, f.cin_real, _ptr(self.packed), self.cout,
                                                   self.cin, _stream())
        else:   # nn.ConvTranspose2d weight [cin,cout,3,3] read as OIHW with out = cin, in = cout
            rc = lib.tg_pack_conv3x3s2_weights(_ptr(w), f.cin_real, f.cout_real, _ptr(self.packed), self.cout,
                                               self.cin, _stream())
        L.check(rc, 'tg_pack_weights (dgrad)')
        self._ver = ver

    def __call__(self, dz, y=None, residual=None, mask=None, mask_act=L.ACT_NONE, impl=None):
        """dz NHWC fp16 [n,oh,ow,cin] -> gradient w.r.t. the layer input [n,h,w,cout];
        y = (conv [+ residual]) * act'(mask)."""
        _req(dz, torch.float16, 'dz', 4)
        n, oh, ow, c = dz.shape
        if c != self.cin:
            raise L.TecoganB200Error(f'dgrad: dz has {c} channels, expected {self.cin}')
        if self.kind == L.CONV_3X3_S2:
            if oh % 2 or ow % 2:
                raise L.TecoganB200Error('dgrad of the transposed conv needs even output sizes')
            h, w = oh // 2, ow // 2
        else:
            h, w = oh, ow
        if y is None:
            y = torch.empty((n, h, w, self.cout), dtype=torch.float16, device=dz.device)
        for t, nm in ((y, 'dx'), (residual, 'residual'), (mask, 'mask')):
            if t is not None:
                _req(t, torch.float16, nm, 4)
                if tuple(t.shape) != (n, h, w, self.cout):
                    raise L.TecoganB200Error(f'dgrad: {nm} shape {tuple(t.shape)} != {(n, h, w, self.cout)}')
        if (mask is not None) != (mask_act in (L.ACT_RELU, L.ACT_LRELU02)):
            raise L.TecoganB200Error('dgrad: mask and mask_act (RELU / LRELU02) go together')
        d = L.ConvDesc()
        d.x, d.weights, d.bias = dz.data_ptr(), self.packed.data_ptr(), self.bias.data_ptr()
        d.residual = residual.data_ptr() if residual is not None else None
        d.mask = mask.data_ptr() if mask is not None else None
        d.y = y.data_ptr()
        d.n, d.h, d.w, d.cin, d.cout, d.cout_real = n, h, w, self.cin, self.cout, self.cout
        d.kind, d.epilogue = self.kind, L.EPI_NHWC_F16
        d.act = {L.ACT_NONE: L.ACT_NONE, L.ACT_RELU: L.ACT_DRELU, L.ACT_LRELU02: L.ACT_DLRELU02}[mask_act]
        d.a_mode = L.AMODE_AUTO
        d.cin_real = self.fwd.cout_real          # dz channels beyond the layer's real outputs are zero
        impl = impl or default_conv_impl()
        lib = L.load()
        if impl == 'tcgen05':
            L.check(lib.tg_conv_tcgen05(ctypes.byref(d), _stream()), 'tg_conv_tcgen05 (dgrad)')
        else:
            L.check(lib.tg_conv_simt(ctypes.byref(d), _stream()), 'tg_conv_simt (dgrad)')
        return y


def wgrad(fwd, x, dz, dw, scale=None, impl=None, max_ctas=0, db=None):
    """dw (fp32, the parameter's layout, pre-zeroed or accumulating) += 1/scale * x (*) dz for the
    forward layer `fwd` (PackedConv): x = its NHWC fp16 input, dz = gradient of its pre-activation
    output (NHWC fp16, pad64(cout_real) channels)."""
    _req(x, torch.float16, 'x', 4)
    _req(dz, torch.float16, 'dz', 4)
    _req(dw, torch.float32, 'dw', 4)
    n, h, w, cin = x.shape
    up = 2 if fwd.kind == L.CONVT_3X3_S2 else 1
    cout = pad64(fwd.cout_real)
    if cin != fwd.cin or tuple(dz.shape) != (n, up * h, up * w, cout):
        raise L.TecoganB200Error(f'wgrad: shapes x {tuple(x.shape)} dz {tuple(dz.shape)} do not fit the layer')
    want = (fwd.cout_real, fwd.cin_real, 3, 3) if fwd.kind == L.CONV_3X3 else (fwd.cin_real, fwd.cout_real, 3, 3)
    if tuple(dw.shape) != want:
        raise L.TecoganB200Error(f'wgrad: dw shape {tuple(dw.shape)} != {want}')
    d = L.WgradDesc()
    d.x, d.dz, d.dw = x.data_ptr(), dz.data_ptr(), dw.data_ptr()
    d.scale = scale.ws.data_ptr() if scale is not None else None
    fuse_db = db is not None and fwd.kind == L.CONV_3X3 and (impl or default_conv_impl()) == 'tcgen05'
    if db is not None:
        _req(db, torch.float32, 'db', 1)
        if db.numel() != fwd.cout_real:
            raise L.TecoganB200Error('wgrad: db must have cout_real elements')
        if fuse_db:
            d.db = db.data_ptr()            # bias gradient from the same MMAs
    d.n, d.h, d.w, d.cin, d.cout = n, h, w, cin, cout
    d.cin_real, d.cout_real, d.kind, d.max_ctas, d.reserved = fwd.cin_real, fwd.cout_real, fwd.kind, max_ctas, 0
    lib = L.load()
    impl = impl or default_conv_impl()
    if impl == 'tcgen05':
        L.check(lib.tg_wgrad_tcgen05(ctypes.byref(d), _stream()), 'tg_wgrad_tcgen05')
    else:
        L.check(lib.tg_wgrad_simt(ctypes.byref(d), _stream()), 'tg_wgrad_simt')
    if db is not None and not fuse_db:
        bias_grad(dz, db, scale)            # transposed conv / cross-check path: separate reduction kernel
    return dw


def bias_grad(dz, db, scale=None):
    """db (fp32 [c_real]) += 1/scale * sum over pixels of dz[..., :c_real]"""
    _req(dz, torch.float16, 'dz', 4)
    _req(db, torch.float32, 'db', 1)
    c = dz.shape[-1]
    L.check(L.load().tg_bias_grad_nhwc_f16(_ptr(dz), dz.numel() // c, c, db.numel(), _scale_ptr(scale), _ptr(db),
                                           _stream()), 'tg_bias_grad')
    return db


def grad_pack(a, b=None, scale=None, cpad=64, y=None):
    """(a [+ b]) * scale : NCHW fp32 -> NHWC fp16 (cpad channels)"""
    _req(a, torch.float32, 'grad', 4)
    if b is not None:
        _req(b, torch.float32, 'grad', 4)
    n, c, h, w = a.shape
    if y is None:
        y = torch.empty((n, h, w, cpad), dtype=torch.float16, device=a.device)
    L.check(L.load().tg_grad_pack_nhwc_f16(_ptr(a), _ptr(b), _scale_ptr(scale), _ptr(y), n, c, h, w, cpad, _stream()),
            'tg_grad_pack')
    return y


def grad_unpack(x, c, scale=None, c_offset=0, y=None, accumulate=False):
    """channels [c_offset, c_offset+c) of NHWC fp16 -> NCHW fp32 / scale"""
    _req(x, torch.float16, 'x', 4)
    n, h, w, cpad = x.shape
    if y is None:
        y = torch.empty((n, c, h, w), dtype=torch.float32, device=x.device)
    L.check(L.load().tg_grad_unpack_nchw_f32(_ptr(x), _scale_ptr(scale), _ptr(y), n, c, h, w, cpad, c_offset,
                                             int(accumulate), _stream()), 'tg_grad_unpack')
    return y


def grad_pack_ex(a, sub=None, div=None, scale=None, add=None, mask=None, mask_act=L.ACT_NONE, cpad=64, y=None):
    """NCHW fp32 a -> NHWC fp16 y (cpad channels): ((a - sub[c]) / div[c] * scale + add) * act'(mask), each step only
    where its operand is given (tg_grad_pack_ex_nhwc_f16).  mask_act: the activation (RELU / LRELU02) whose stored
    output is `mask`."""
    _req(a, torch.float32, 'grad', 4)
    n, c, h, w = a.shape
    if (sub is None) != (div is None):
        raise L.TecoganB200Error('grad_pack_ex: sub and div go together')
    for t, nm in ((sub, 'sub'), (div, 'div')):
        if t is not None:
            _req(t, torch.float32, nm)
            if t.numel() != c:
                raise L.TecoganB200Error(f'grad_pack_ex: {nm} must have {c} elements')
    if y is None:
        y = torch.empty((n, h, w, cpad), dtype=torch.float16, device=a.device)
    for t, nm in ((y, 'y'), (add, 'add'), (mask, 'mask')):
        if t is not None:
            _req(t, torch.float16, nm, 4)
            if tuple(t.shape) != (n, h, w, cpad):
                raise L.TecoganB200Error(f'grad_pack_ex: {nm} shape {tuple(t.shape)} != {(n, h, w, cpad)}')
    if (mask is not None) != (mask_act in (L.ACT_RELU, L.ACT_LRELU02)):
        raise L.TecoganB200Error('grad_pack_ex: mask and mask_act (RELU / LRELU02) go together')
    act = {L.ACT_NONE: L.ACT_NONE, L.ACT_RELU: L.ACT_DRELU, L.ACT_LRELU02: L.ACT_DLRELU02}[mask_act]
    L.check(L.load().tg_grad_pack_ex_nhwc_f16(_ptr(a), _ptr(sub), _ptr(div), _scale_ptr(scale), _ptr(add), _ptr(mask),
                                              act, _ptr(y), n, c, h, w, cpad, _stream()), 'tg_grad_pack_ex')
    return y


def grad_unpack_ex(x, c, div, scale=None, y=None):
    """channels [0, c) of NHWC fp16 -> NCHW fp32 / scale / div[ch] (tg_grad_unpack_ex_nchw_f32)"""
    _req(x, torch.float16, 'x', 4)
    _req(div, torch.float32, 'div')
    if div.numel() != c:
        raise L.TecoganB200Error(f'grad_unpack_ex: div must have {c} elements')
    n, h, w, cpad = x.shape
    if y is None:
        y = torch.empty((n, c, h, w), dtype=torch.float32, device=x.device)
    _req(y, torch.float32, 'y', 4)
    L.check(L.load().tg_grad_unpack_ex_nchw_f32(_ptr(x), _scale_ptr(scale), _ptr(div), _ptr(y), n, c, h, w, cpad, 0, 0,
                                                _stream()), 'tg_grad_unpack_ex')
    return y


def backward_warp_bwd(x, flow, gy, need_x=True, need_flow=True):
    """-> (gx, gflow) of backward_warp(x, flow) given gy; outputs not needed are None"""
    _req(x, torch.float32, 'x', 4)
    _req(flow, torch.float32, 'flow', 4)
    _req(gy, torch.float32, 'gy', 4)
    n, c, h, w = x.shape
    gx = torch.zeros_like(x) if need_x else None              # scatter-add target
    gf = torch.empty_like(flow) if need_flow else None
    L.check(L.load().tg_backward_warp_bwd_nchw_f32(_ptr(x), _ptr(flow), _ptr(gy), _ptr(gx), _ptr(gf), n, c, h, w,
                                                   _stream()), 'tg_backward_warp_bwd')
    return gx, gf


def warp_s2d_concat_bwd(gx, hr_prev, hr_flow, scale_factor, d_hr_prev=None, d_hr_flow=None, scale=None):
    """gradient of warp_s2d_concat_hrflow: accumulates into d_hr_prev (fp32 NCHW), stores d_hr_flow"""
    _req(gx, torch.float16, 'gx', 4)
    _req(hr_prev, torch.float32, 'hr_prev', 4)
    _req(hr_flow, torch.float32, 'hr_flow', 4)
    n, h, w, cpad = gx.shape
    c = hr_prev.shape[1]
    L.check(L.load().tg_warp_s2d_concat_bwd(_ptr(gx), _ptr(hr_prev), _ptr(hr_flow), _scale_ptr(scale), _ptr(d_hr_prev),
                                            _ptr(d_hr_flow), n, c, h, w, scale_factor, cpad, _stream()),
            'tg_warp_s2d_concat_bwd')


def upsample_bwd(gy, scale_factor, up_mode, mul=1.0, gx=None, accumulate=False):
    _req(gy, torch.float32, 'gy', 4)
    n, c, H, W = gy.shape
    h, w = H // scale_factor, W // scale_factor
    if gx is None:
        gx = torch.empty((n, c, h, w), dtype=torch.float32, device=gy.device)
    L.check(L.load().tg_upsample_bwd_nchw_f32(_ptr(gy), _ptr(gx), n, c, h, w, scale_factor, up_mode, ctypes.c_float(mul),
                                              int(accumulate), _stream()), 'tg_upsample_bwd')
    return gx


def maxpool2x2_bwd(x, gy, act, gx=None):
    _req(x, torch.float16, 'x', 4)
    _req(gy, torch.float16, 'gy', 4)
    n, h, w, c = x.shape
    if gx is None:
        gx = torch.empty_like(x)
    L.check(L.load().tg_maxpool2x2_bwd_nhwc_f16(_ptr(x), _ptr(gy), _ptr(gx), n, h, w, c, act, _stream()),
            'tg_maxpool2x2_bwd')
    return gx


def upsample2x_bwd(gy, m, act, gx=None):
    _req(gy, torch.float16, 'gy', 4)
    _req(m, torch.float16, 'm', 4)
    n, h, w, c = m.shape
    if gx is None:
        gx = torch.empty_like(m)
    L.check(L.load().tg_upsample2x_bilinear_bwd_nhwc_f16(_ptr(gy), _ptr(m), _ptr(gx), n, h, w, c, act, _stream()),
            'tg_upsample2x_bwd')
    return gx


def flow_head_bwd(gflow, flow, scale, gflow2=None, cpad=64, dz=None):
    """dz (NHWC fp16) of the 24*tanh flow head; also chooses `scale` (GradScale) for the FNet backward"""
    _req(gflow, torch.float32, 'gflow', 4)
    _req(flow, torch.float32, 'flow', 4)
    n, _, h, w = flow.shape
    if dz is None:
        dz = torch.empty((n, h, w, cpad), dtype=torch.float16, device=flow.device)
    L.check(L.load().tg_flow_head_bwd(_ptr(gflow), _ptr(gflow2), _ptr(flow), scale.ptr, ctypes.c_float(scale.TARGET),
                                      _ptr(dz), n, h, w, cpad, _stream()), 'tg_flow_head_bwd')
    global LAUNCH_COUNT
    LAUNCH_COUNT += 2
    return dz


def depth_to_space(gy, scale_factor):
    _req(gy, torch.float32, 'gy', 4)
    n, cs, oh, ow = gy.shape
    c = cs // (scale_factor * scale_factor)
    gx = torch.empty((n, c, oh * scale_factor, ow * scale_factor), dtype=torch.float32, device=gy.device)
    L.check(L.load().tg_depth_to_space_nchw_f32(_ptr(gy), _ptr(gx), n, c, oh * scale_factor, ow * scale_factor,
                                                scale_factor, _stream()), 'tg_depth_to_space')
    return gx


def st_disc_input(data, bi, flow, t, pad, csize, out=None):
    """[orig | crop_pad(warp) | cond] input of the spatio-temporal discriminator (tg_st_disc_input_nchw_f32)"""
    _req(data, torch.float32, 'data', 5)
    _req(bi, torch.float32, 'bi_data', 5)
    _req(flow, torch.float32, 'hr_flow_merge', 4)
    n, t_full, c, h, w = data.shape
    if bi.shape[0] != n or bi.shape[1] < t or tuple(bi.shape[2:]) != (c, h, w) or bi.shape[1] != t_full:
        raise L.TecoganB200Error(f'st_disc_input: bi_data shape {tuple(bi.shape)} does not match data {tuple(data.shape)}')
    if tuple(flow.shape) != (n * t, 2, h, w):
        raise L.TecoganB200Error(f'st_disc_input: flow shape {tuple(flow.shape)} != {(n * t, 2, h, w)}')
    if out is None:
        out = torch.empty((n * t // 3, 9 * c, h, w), dtype=torch.float32, device=data.device)
    L.check(L.load().tg_st_disc_input_nchw_f32(_ptr(data), _ptr(bi), _ptr(flow), _ptr(out), n, t_full, t, c, h, w, pad,
                                               csize, _stream()), 'tg_st_disc_input')
    return out


def st_disc_input_bwd(gout, flow, shape, t, pad, csize):
    _req(gout, torch.float32, 'gout', 4)
    n, t_full, c, h, w = shape
    gdata = torch.zeros(shape, dtype=torch.float32, device=gout.device)
    L.check(L.load().tg_st_disc_input_bwd_nchw_f32(_ptr(gout), _ptr(flow), _ptr(gdata), n, t_full, t, c, h, w, pad, csize,
                                                   _stream()), 'tg_st_disc_input_bwd')
    return gdata
