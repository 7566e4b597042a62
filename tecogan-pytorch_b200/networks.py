"""FRNet / FNet / SRNet with the reference's module surface, running on libtecogan_b200.

Drop-in for the generator half of codes/models/networks/tecogan_nets.py (reference lines
16-314): same constructor arguments, same method names (forward / forward_sequence / step /
infer_sequence / generate_dummy_data / profile), same attributes (fnet, srnet, upsample_func,
scale) and the same state_dict keys and shapes (strict load of reference ``G_iter*.pth`` works).

The nn.Conv2d / nn.ConvTranspose2d objects below are PARAMETER HOLDERS ONLY -- their forward is
never called.  All arithmetic goes through ``ops`` (hand-written sm_90a kernels); a CPU tensor
raises, there is no PyTorch fallback.
"""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn

from . import lib as L
from . import ops
from .net_utils import get_upsampling_func, up_mode_of, no_autograd, needs_grad

_LRELU, _RELU = L.ACT_LRELU02, L.ACT_RELU


def _pair(cin, mid, cout, tail=None):
    """[conv, act-slot, conv, act-slot(, tail)] -- conv modules sit at indices 0 and 2 exactly
    like the reference Sequentials, so state_dict keys read '<block>.0.*' / '<block>.2.*'."""
    mods = [nn.Conv2d(cin, mid, 3, 1, 1, bias=True), nn.Identity(),
            nn.Conv2d(mid, cout, 3, 1, 1, bias=True), nn.Identity()]
    if tail is not None:
        mods.append(tail)
    return nn.Sequential(*mods)


def _cuda_f32(t, name):
    if not t.is_cuda:
        raise L.TecoganB200Error(f'{name} must be a CUDA tensor: tecogan-b200 has no CPU path')
    return t.detach().float().contiguous()


class _ConvCache:
    """Lazily built PackedConv objects, refreshed when parameters change."""

    def __init__(self):
        self._layers = {}
        self._dgrads = {}

    def get(self, key, module, kind, act, epilogue=L.EPI_NHWC_F16):
        ent = self._layers.get(key)
        if ent is None or ent[0].packed.device != module.weight.device:
            pc = ops.PackedConv(module.weight, module.bias, kind, act, epilogue)
            self._layers[key] = (pc, module)
        else:
            pc = ent[0]
            pc.refresh(module.weight, module.bias)
        return pc

    def dgrad(self, key, module, pc=None):
        """The data-gradient operand (ops.PackedDgrad) of the forward layer cached under `key`."""
        if pc is None:
            pc = self._layers[key][0]
        ent = self._dgrads.get(key)
        if ent is None or ent.fwd is not pc:
            ent = self._dgrads[key] = ops.PackedDgrad(pc, module.weight)
        else:
            ent.refresh(module.weight)
        return ent

    def refresh_all(self, force=False):
        """Re-pack (in place) every layer whose parameters changed -- captured CUDA graphs read
        the same packed buffers, so this is all that is needed after an optimizer step or a
        load_state_dict.  force=True repacks unconditionally (needed after ``param.data`` writes,
        which do not bump the version counter)."""
        for pc, module in self._layers.values():
            pc.refresh(module.weight, module.bias, force=force)


class FNet(nn.Module):
    """Optical-flow estimator (reference tecogan_nets.py:16-82): 14 conv3x3, LeakyReLU(0.2)
    after all but the last, 3x maxpool(2), 3x bilinear x2, tanh*24."""

    ENC = (('encoder1', None, 32), ('encoder2', 32, 64), ('encoder3', 64, 128))
    DEC = (('decoder1', 128, 256), ('decoder2', 256, 128), ('decoder3', 128, 64))
    # Position of each conv from the input to the flow head.  The convs alternate their tile walk along it, odd
    # positions walking last to first (PackedConv.reverse), so that each starts on the tiles its producer wrote
    # last, which are still in L2.  pack_pair and upsample2x walk last to first, so encoder1[0] and flow[0], which
    # read their full-resolution maps, walk forward.
    CHAIN = {k: i for i, k in enumerate([(b, j) for b, _, _ in ENC + DEC for j in (0, 2)] + [('flow', 0), ('flow', 2)])}

    def __init__(self, in_nc):
        super().__init__()
        self.in_nc = in_nc
        for name, cin, cout in self.ENC:
            setattr(self, name, _pair(2 * in_nc if cin is None else cin, cout, cout, nn.Identity()))
        for name, cin, cout in self.DEC:
            setattr(self, name, _pair(cin, cout, cout))
        self.flow = nn.Sequential(nn.Conv2d(64, 32, 3, 1, 1, bias=True), nn.Identity(),
                                  nn.Conv2d(32, 2, 3, 1, 1, bias=True))
        self._cache = _ConvCache()

    def _conv(self, block, idx, act, epilogue=L.EPI_NHWC_F16):
        pc = self._cache.get((block, idx), getattr(self, block)[idx], L.CONV_3X3, act, epilogue)
        pc.reverse = self.CHAIN[(block, idx)] % 2 == 1
        return pc

    def forward(self, x1, x2):
        """flow from x1 to x2, NCHW fp32 [n,2,8*(h//8),8*(w//8)]"""
        g1, g2 = x1, x2
        x1, x2 = _cuda_f32(x1, 'x1'), _cuda_f32(x2, 'x2')
        no_autograd('FNet.forward (input gradient)', g1, g2)
        if self.training and needs_grad(*self.parameters()):
            # trained through (FRNet.forward_sequence has its own fused path; this is the bare call the
            # ST-discriminator makes, tecogan_nets.py:420): forward + backward on the library's kernels
            from .autograd import FNetFunction
            return FNetFunction.apply(self, x1, x2, *self.parameters())
        a = ops.pack_pair(x1, x2)                       # cat + NHWC fp16 (c64)
        fuse_pool = ops.default_conv_impl() == 'tcgen05' and ops.pool_fused()
        for name, _, _ in self.ENC:
            a = self._conv(name, 0, _LRELU)(a)
            if fuse_pool:                               # MaxPool2d(2,2) in the conv's epilogue (inference only:
                a = self._conv(name, 2, _LRELU)(a, pool=True)   # training keeps the full-resolution map)
            else:
                a = self._conv(name, 2, _LRELU)(a)
                a = ops.maxpool2x2(a)
        for name, _, _ in self.DEC:
            a = self._conv(name, 0, _LRELU)(a)
            a = self._conv(name, 2, _LRELU)(a)
            a = ops.upsample2x(a)
        a = self._conv('flow', 0, _LRELU)(a)
        return self._conv('flow', 2, L.ACT_NONE, L.EPI_FLOW_NCHW_F32)(a)   # 24*tanh fused

    def conv_layers(self, h, w):
        """(module, out_h, out_w) per conv, in execution order -- for FRNet.profile."""
        out = []
        for name, _, _ in self.ENC:
            out += [(getattr(self, name)[0], h, w), (getattr(self, name)[2], h, w)]
            h, w = h // 2, w // 2
        for name, _, _ in self.DEC:
            out += [(getattr(self, name)[0], h, w), (getattr(self, name)[2], h, w)]
            h, w = 2 * h, 2 * w
        out += [(self.flow[0], h, w), (self.flow[2], h, w)]
        return out


class ResidualBlock(nn.Module):
    """conv-ReLU-conv + skip (reference tecogan_nets.py:85-100); parameter holder."""

    def __init__(self, nf=64):
        super().__init__()
        self.conv = nn.Sequential(nn.Conv2d(nf, nf, 3, 1, 1, bias=True), nn.Identity(),
                                  nn.Conv2d(nf, nf, 3, 1, 1, bias=True))


class SRNet(nn.Module):
    """Reconstruction + upsampling network (reference tecogan_nets.py:103-147)."""

    def __init__(self, in_nc, out_nc, nf, nb, upsample_func, scale):
        super().__init__()
        self.in_nc, self.out_nc, self.nf, self.nb, self.scale = in_nc, out_nc, nf, nb, scale
        self.conv_in = nn.Sequential(nn.Conv2d((scale ** 2 + 1) * in_nc, nf, 3, 1, 1, bias=True),
                                     nn.Identity())
        self.resblocks = nn.Sequential(*[ResidualBlock(nf) for _ in range(nb)])
        ups = [nn.ConvTranspose2d(nf, nf, 3, 2, 1, output_padding=1, bias=True), nn.Identity()]
        if scale == 4:
            ups += [nn.ConvTranspose2d(nf, nf, 3, 2, 1, output_padding=1, bias=True), nn.Identity()]
        self.conv_up = nn.Sequential(*ups)
        self.conv_out = nn.Conv2d(nf, out_nc, 3, 1, 1, bias=True)
        self.upsample_func = upsample_func
        self._cache = _ConvCache()

    def forward(self, lr_curr, hr_prev_tran):
        """lr_curr nchw, hr_prev_tran n(s*s*c)hw (both fp32) -> hr nchw fp32"""
        g1 = lr_curr
        lr_curr = _cuda_f32(lr_curr, 'lr_curr')
        no_autograd('SRNet.forward', g1, hr_prev_tran, *(self.parameters() if self.training else ()))
        x = ops.nchw_to_nhwc(torch.cat([lr_curr, _cuda_f32(hr_prev_tran, 'hr_prev_tran')], dim=1))
        return self.run_nhwc(x, lr_curr)

    def run_nhwc(self, x, lr_curr, out=None, out_u8=None):
        """x = SRNet input NHWC fp16 [n,h,w,64] (channels [lr_curr | space_to_depth(warp) | 0])."""
        c = self._cache
        body = [c.get('in', self.conv_in[0], L.CONV_3X3, _RELU)]
        for i, blk in enumerate(self.resblocks):
            body += [c.get(('r', i, 0), blk.conv[0], L.CONV_3X3, _RELU),
                     c.get(('r', i, 2), blk.conv[2], L.CONV_3X3, L.ACT_NONE)]
        ups = [c.get(('up', u), self.conv_up[u], L.CONVT_3X3_S2, _RELU) for u in range(0, len(self.conv_up), 2)]
        # Each conv walks its tiles opposite to the launch that wrote its input, so it starts on the tiles that are
        # still in L2: conv_in last to first against warp_s2d_concat's forward walk, then alternating down the body
        # to the first transposed conv.  A residual conv also reads `a` right after the plain conv read it the
        # other way round.
        for i, pc in enumerate(body + ups):
            pc.reverse = i % 2 == 0
        a = body[0](x)
        for i in range(len(self.resblocks)):
            t = body[1 + 2 * i](a)
            a = body[2 + 2 * i](t, residual=a)
        pc_out = c.get('out', self.conv_out, L.CONV_3X3, L.ACT_NONE, L.EPI_OUT_NCHW_F32)
        tail = ops.tail_mode()
        if (tail and ops.default_conv_impl() == 'tcgen05' and ups[-1].cin == 64 and ups[-1].cout == 64
                and pc_out.cin == 64 and pc_out.cout_real <= 3):
            # last transposed conv + ReLU + conv_out + residual in ONE launch: the 64-channel HR map (88 MB per
            # frame) stays in shared memory and never reaches HBM.  mode 'acc': `out` is first filled with upsample_func(lr_curr) by the
            # (pure-write) upsample kernel and the tail accumulates onto it -- one coalesced read per pixel;
            # mode 'fused': the residual (and the uint8 frame) are evaluated inside the tail kernel.
            for up in ups[:-1]:
                a = up(a)
            mode = up_mode_of(self.upsample_func)
            if tail == 'acc':
                out = ops.upsample(lr_curr, self.scale, mode, y=out)
                out = ops.fused_tail(ups[-1], pc_out, a, None, self.scale, mode, y=out, accumulate=True)
                if out_u8 is not None:
                    ops.float_to_uint8_nhwc(out, out_u8)
                return out
            return ops.fused_tail(ups[-1], pc_out, a, lr_curr, self.scale, mode, y=out, y_u8=out_u8)
        for up in ups:
            a = up(a)
        # out = conv_out(a) (pure-store epilogue), then out += upsample_func(lr_curr).
        out = pc_out(a, y=out)
        out = ops.upsample(lr_curr, self.scale, up_mode_of(self.upsample_func), y=out, accumulate=True)
        if out_u8 is not None:
            ops.float_to_uint8_nhwc(out, out_u8)
        return out

    def conv_layers(self, h, w):
        out = [(self.conv_in[0], h, w)]
        for blk in self.resblocks:
            out += [(blk.conv[0], h, w), (blk.conv[2], h, w)]
        for u in range(0, len(self.conv_up), 2):
            out.append((self.conv_up[u], h, w))     # reference counts ConvT at INPUT resolution
            h, w = 2 * h, 2 * w
        out.append((self.conv_out, h, w))
        return out


class BaseSequenceGenerator(nn.Module):
    """Interface of codes/models/networks/base_nets.py:4-35."""

    def generate_dummy_data(self, lr_size):
        return None

    def profile(self, *args, **kwargs):
        pass

    def forward(self, *args, **kwargs):
        pass

    def forward_sequence(self, lr_data):
        pass

    def step(self, *args, **kwargs):
        pass

    def infer_sequence(self, lr_data, device):
        pass


def _conv_gflops(layers):
    """reference counter: 2*Cin*kh*kw*Cout*out_px (codes/metrics/model_summary.py:16-26,42-53)"""
    tot = 0.0
    for m, oh, ow in layers:
        o, i, kh, kw = m.weight.shape
        tot += (2 * i * kh * kw) * o * oh * ow / 1e9
    return tot


class FRNet(BaseSequenceGenerator):
    """Frame-recurrent generator (reference tecogan_nets.py:150-314) on sm_90a kernels."""

    def __init__(self, in_nc, out_nc, nf, nb, degradation, scale):
        super().__init__()
        # SRNet adds upsample_func(lr_curr) (in_nc channels) to its out_nc-channel output, and its input -- lr_curr
        # and the space_to_depth of the warped out_nc-channel HR frame -- is one NHWC map of at most 64 channels
        if in_nc != out_nc:
            raise L.TecoganB200Error(f'FRNet: in_nc={in_nc} != out_nc={out_nc}: the residual and the recurrent HR '
                                     'frame need as many output channels as input channels')
        if (scale ** 2 + 1) * in_nc > 64:
            raise L.TecoganB200Error(f'FRNet: (scale^2 + 1) * in_nc = {(scale ** 2 + 1) * in_nc} SRNet input '
                                     f'channels at scale {scale}, in_nc {in_nc}: at most 64')
        self.scale = scale
        self.degradation = degradation
        self.upsample_func = get_upsampling_func(self.scale, degradation)
        self.fnet = FNet(in_nc)
        self.srnet = SRNet(in_nc, out_nc, nf, nb, self.upsample_func, self.scale)

    # ------------------------------------------------------------------ dispatch (DDP interface)
    def forward(self, lr_data, device=None):
        if self.training:
            return self.forward_sequence(lr_data)
        return self.infer_sequence(lr_data, device)

    # ------------------------------------------------------------------ one recurrent frame
    def step(self, lr_curr, lr_prev, hr_prev):
        """lr_curr, lr_prev nchw; hr_prev nc(sh)(sw); any batch n (lock-stepped clips)."""
        return self.step_into(lr_curr, lr_prev, hr_prev, None)

    def step_into(self, lr_curr, lr_prev, hr_prev, out, out_u8=None):
        """step() writing hr_curr into `out` (nchw fp32, allocated when None) and, when given, the
        quantised frame into `out_u8` (uint8 nhwc).  Enqueues ~25 kernels on the current stream and
        nothing else, so it is CUDA-graph capturable."""
        g = (lr_curr, lr_prev, hr_prev)
        lr_curr, lr_prev = _cuda_f32(lr_curr, 'lr_curr'), _cuda_f32(lr_prev, 'lr_prev')
        hr_prev = _cuda_f32(hr_prev, 'hr_prev')
        no_autograd('FRNet.step', *g, *(self.parameters() if self.training else ()))
        with torch.no_grad():
            lr_flow = self.fnet(lr_curr, lr_prev)
            # reflect-pad + upsample_func + *scale + warp + space_to_depth + concat: one kernel
            x = ops.warp_s2d_concat_lrflow(hr_prev, lr_flow, lr_curr, self.scale,
                                           up_mode_of(self.upsample_func))
            return self.srnet.run_nhwc(x, lr_curr, out=out, out_u8=out_u8)

    # ------------------------------------------------------------------ training forward
    def forward_sequence(self, lr_data):
        """lr_data ntchw -> dict(hr_data, hr_flow, lr_prev, lr_curr, lr_flow), reference :174-225.

        Under autograd (training) the whole sequence is ONE autograd node (autograd.SequenceFunction):
        forward and backward -- dgrad / wgrad of every conv, the warp's scatter/gather, pool / upsample
        / tanh derivatives -- run on the library's kernels and the parameters receive fp32 gradients,
        so VSRModel.train / VSRGANModel.train (and DDP's gradient all-reduce) work unchanged.
        lr_data is data: no gradient is produced for it."""
        no_autograd('FRNet.forward_sequence (lr_data gradient)', lr_data)
        if needs_grad(*self.parameters()):
            from .autograd import SequenceFunction
            lr_data = _cuda_f32(lr_data, 'lr_data')
            n, t, c, lr_h, lr_w = lr_data.shape
            hr_data, hr_flow, lr_flow = SequenceFunction.apply(self, lr_data, *self.parameters())
            return {
                'hr_data': hr_data, 'hr_flow': hr_flow,
                'lr_prev': lr_data[:, :-1].reshape(n * (t - 1), c, lr_h, lr_w),
                'lr_curr': lr_data[:, 1:].reshape(n * (t - 1), c, lr_h, lr_w),
                'lr_flow': lr_flow,
            }
        lr_data = _cuda_f32(lr_data, 'lr_data')
        n, t, c, lr_h, lr_w = lr_data.shape
        s = self.scale
        lr_prev = lr_data[:, :-1].reshape(n * (t - 1), c, lr_h, lr_w)
        lr_curr = lr_data[:, 1:].reshape(n * (t - 1), c, lr_h, lr_w)
        lr_flow = self.fnet(lr_curr, lr_prev)
        hr_flow = ops.upsample(lr_flow, s, up_mode_of(self.upsample_func), mul=float(s))
        hr_flow = hr_flow.view(n, t - 1, 2, s * lr_h, s * lr_w)
        frames = lr_data.transpose(0, 1).contiguous()       # t,n,c,h,w
        flows = hr_flow.transpose(0, 1).contiguous()        # t-1,n,2,H,W
        hr_data = torch.empty((t, n, c, s * lr_h, s * lr_w), dtype=torch.float32, device=lr_data.device)
        x0 = ops.nchw_to_nhwc(frames[0])                    # hr_prev_tran = zeros (reference :194-197)
        self.srnet.run_nhwc(x0, frames[0], out=hr_data[0])
        for i in range(1, t):
            x = ops.warp_s2d_concat_hrflow(hr_data[i - 1], flows[i - 1], frames[i], s)
            self.srnet.run_nhwc(x, frames[i], out=hr_data[i])
        return {
            'hr_data': hr_data.transpose(0, 1).contiguous(),   # n,t,c,hr_h,hr_w
            'hr_flow': hr_flow,
            'lr_prev': lr_prev,
            'lr_curr': lr_curr,
            'lr_flow': lr_flow,
        }

    # ------------------------------------------------------------------ inference over a clip
    def infer_sequence(self, lr_data, device):
        """lr_data tchw fp32 (host or device) -> uint8 ndarray thwc (reference :254-281).

        Also accepts ntchw (n lock-stepped clips) and then returns nthwc."""
        from .engine import infer_clips
        device = torch.device('cuda') if device is None else torch.device(device)
        if lr_data.dim() == 4:
            return infer_clips(self, lr_data.unsqueeze(0), device)[0]
        return infer_clips(self, lr_data, device)

    def stream(self, n, h, w, device=None, input='uint8', channel_order='rgb', out_format='rgb', in_color='bt601',
               out_color='bt601', out_size=None, resize_filter='bicubic', scene_cut=None, crop=None, out_frame=None,
               out_origin=None, pad_front=0, padding_mode='reflect', in_size=None, in_filter='bicubic'):
        """A VideoStream of n lock-stepped slots of h x w LR frames: video pushed in chunks of any length, the
        recurrent state carried from one push to the next, and a slot restarted (reset=) when its video ends and
        the next one begins while the other slots keep running.

        input='uint8': frames uint8 [n,k,h,w,c] as decoders and cv2.imread produce them, converted on the device
        to float32 / 255 exactly as the reference's loader does (paired_folder_dataset.py:49); channel_order='bgr'
        takes cv2's BGR order.  input='float32': frames fp32 [n,k,c,h,w] in [0,1], the reference layout.
        push() returns uint8 [n,k,H,W,c] frames, byte-identical to infer_sequence over the concatenated pushes.

        YUV 4:2:0 video (BT.601 limited range, as ffmpeg's yuv420p / PyAV give it, NVDEC decodes and NVENC takes):
        input='nv12' or 'i420' takes uint8 [n,k,3h/2,w] frames (the Y plane, then the interleaved UV plane or the U
        and V planes) and converts them on the device exactly as cv2.cvtColor(frame, COLOR_YUV2RGB_NV12 / _I420)
        followed by the loader's / 255.  out_format='nv12' or 'i420' returns uint8 [n,k,3H/2,W] frames:
        cv2.cvtColor(rgb, COLOR_RGB2YUV_I420) of the RGB output (chroma of each 2x2 block from its top-left
        pixel), for 'nv12' with U and V interleaved.  Both need even h and w; any input works with any
        out_format.
        10-bit video: 'p010' (NV12 planes, uint16 words, sample in the high 10 bits; NVDEC / NVENC, ffmpeg p010le)
        and 'i420_10' (I420 planes, uint16 words, sample in the low 10 bits; ffmpeg / PyAV yuv420p10le), as input
        (uint16 [n,k,3h/2,w], converted to RGB / 1023) or out_format (uint16 [n,k,3H/2,W], encoded from the fp32 HR
        frame, so the two bits below the uint8 output are kept).
        4:2:2 and 4:4:4 video, as input or out_format: 'yuy2' / 'uyvy' (packed, uint8 [n,k,h,2w] per pixel pair
        Y0 U Y1 V / U Y0 V Y1, w even; V4L2 webcams, SDI capture) decode and encode exactly as cv2.cvtColor's
        COLOR_YUV2RGB_YUY2 / _UYVY and COLOR_RGB2YUV_YUY2 / _UYVY (chroma of each pair's mean); 'i444' (uint8) and
        'i444_10' (uint16, sample in the low 10 bits) are planar [n,k,3h,w] frames with a chroma sample per pixel.
        Neither needs an even h.
        10-bit 4:2:2 video (professional and broadcast), as input or out_format, w even, any h: 'p210' (uint16
        [n,k,2h,w]: the Y plane, then a full-height interleaved UV plane, samples in the high 10 bits; GPU video
        engines), 'i422_10' (uint16 [n,k,2h,w]: the Y plane, then U and V planes of h x w/2, samples in the low 10
        bits; ffmpeg yuv422p10le, what ProRes 422 and DNxHR decode into) and 'v210' (uint8 [n,k,h,S] with
        S = 128 * ceil(w / 48): 6 pixels per 16-byte group, rows padded to 128 bytes; SDI capture and playout).
        Decode is the 10-bit row with nearest chroma; the encode takes the fp32 HR frame, Y per pixel and U, V from
        each pair's sum.  A v210 crop or out_origin starts on a 6-pixel group and ends on one or at the frame's right
        edge.
        in_color / out_color pick the YUV side's colour: 'bt601' (the default, limited range; for 8-bit frames
        exactly cv2's conversion), 'bt709', 'bt601-full', 'bt709-full' (ITU-T H.273 quantisation, integer fixed
        point as oracle/yuv_color.py specifies).  Take in_color from the decoder (ffprobe's color_space /
        color_range) and tag the encoded output with out_color.  A colour other than 'bt601' on an RGB or float32
        side raises ValueError.
        out_size=(Ho, Wo) resizes every output frame from H x W to Ho x Wo on the device, from the fp32 HR frame
        and before the uint8 quantisation or the YUV encode: push() then returns uint8 [n,k,Ho,Wo,c] or YUV words
        ([n,k,3Ho/2,Wo] for 4:2:0, [n,k,Ho,2Wo] for 4:2:2, [n,k,3Ho,Wo] for 4:4:4).
        resize_filter is 'bicubic' (the default) or 'lanczos': Pillow's antialiased filters
        (Image.resize on 'F' images, as oracle/resample.py specifies), widened by the ratio on a downscale.  Each
        axis needs H/4 <= Ho <= 2H (likewise W), even Ho and Wo for 4:2:0 output, even Wo for 4:2:2.
        out_size=(H, W) gives the bytes of the stream without it.
        scene_cut=threshold (a number in (0, 100]; 10.0 is a good start, the default of ffmpeg's scdet) detects
        hard cuts on the device, inside the step: each frame is scored against the previous one of its slot (the
        mean absolute difference of the 8-bit codes and its change, as oracle/scene_cut.py specifies), and a score
        >= threshold restarts the slot at that frame exactly as reset= would have.  After each push the stream's
        last_cuts (bool [n,k]) and last_scores (float64 [n,k]) tell where, e.g. to ask the encoder for a keyframe.
        None (the default) turns detection off; any input and output format work with it.
        Letterboxed / pillarboxed video: crop=(top, left, ch, cw) runs the net, FNet's flow and scene_cut on the
        ch x cw picture at (top, left) of the h x w frames pushed (h x w stays the frame's size in the input layout's
        shape); the output picture is s*ch x s*cw (or out_size, whose ratio limits then refer to the picture).  The
        bars are never read.  A decoder surface of pitch P words and R rows (NVDEC NV12 / P010: the chroma plane at
        P * R) is the frame h, w = R, P with crop=(0, 0, rows, cols) -- no copy into a packed frame.  tecogan_b200.
        detect_bars(frames, input=...) finds the box on the device.  crop needs uint8 or YUV input and the input
        layout's chroma grid (4:2:0: even top, left, ch, cw; 4:2:2: even left and cw).
        out_frame=(Hf, Wf) returns Hf x Wf frames in out_format with the picture at out_origin=(y, x) (default: centred,
        rounded down to the output layout's chroma grid) and everything else the format's exact black (RGB 0; Y 16 /
        C 128 at 8-bit limited range, Y 0 full range, 64 / 512 and 0 / 512 at 10 bits, P010 words << 6).  The bars
        are written once, when the stream is built; each step writes only the picture.  tecogan_b200.fit_size gives
        the largest out_size of the picture's display aspect that fits the frame (pillarbox / letterbox).
        A crop or picture that does not fit, or lies off the chroma grid, raises ValueError.
        Temporal padding, as the reference's test pipeline pads (VSRModel.infer -> BaseModel.pad_sequence,
        base_model.py:230-251; test.yml's num_pad_front / padding_mode): pad_front=p (an int in [0, 32]) and
        padding_mode='reflect' or 'replicate' warm each slot's recurrent state on p pad frames at every shot start --
        frame 0, a reset= and a detected scene_cut -- so the frames of a shot of L frames are byte-identical to
        infer_sequence(pad_sequence(shot, q))[q:], with q = min(p, L - 1) for 'reflect' (the reference asserts p < L;
        a shorter shot gets the longest reflection it has) and q = p for 'replicate'.  'reflect' reads the p frames
        after a shot start before it can produce that start, so push() returns every slot's frames p frames behind
        its input: [n,k_out,...] with k_out < k only while the first p frames fill the stream.  flush() ends every
        slot's video and returns the held frames (then every slot starts anew at the next push); close() drops them.
        A reset= ends the slot's previous video with the previous push, and its held tail comes out, padded for that
        end, in the rows of this push.  last_cuts / last_scores stay those of the unpadded stream (pad frames are
        never scored) and row j describes returned frame j.  The warm-up steps run on state of their own before the
        main step of the shot's first frame, batch-n and shared by the slots starting a shot at the same frame.
        pad_front=0 (the default) is the stream without padding, launch for launch.
        Any input resolution: in_size=(hn, wn) resizes the picture (the whole frame, or the crop box) on the device to
        hn x wn, inside the frame-input launch, and the net runs at that size: the output is s*hn x s*wn (out_size,
        out_frame and out_origin refer to it).  in_filter is 'bicubic' (the default) or 'lanczos', Pillow's
        antialiased filters as for out_size.  The net's LR frame is oracle/resample.resize(decode(picture), (hn, wn),
        in_filter), kept in fp32 and not re-quantised to 8 bits, where decode is what the frame input computes
        without in_size (uint8 / 255, or the YUV conversion; 10 bit / 1023).  scene_cut scores these resized frames.
        Each axis needs picture/4 <= in_size <= 2*picture; uint8 and YUV input only.  in_size equal to the picture
        (every source already at the LR size) is the stream without it, launch for launch and byte for byte.  E.g. a
        1080p NV12 source through a x4 net: h, w = 1080, 1920, in_size=(540, 960), NV12 2160x3840 out.
        The CUDA graphs are captured by the first push; the stream holds the net."""
        from .engine import VideoStream
        return VideoStream(self, n, h, w, device, input, channel_order, out_format, in_color, out_color, out_size,
                           resize_filter, scene_cut, crop, out_frame, out_origin, pad_front, padding_mode, in_size,
                           in_filter)

    def refresh_packed_weights(self, force=False):
        self.fnet._cache.refresh_all(force)
        self.srnet._cache.refresh_all(force)

    # ------------------------------------------------------------------ profile protocol
    def generate_dummy_data(self, lr_size, device):
        c, lr_h, lr_w = lr_size
        s = self.scale
        lr_curr = torch.rand(1, c, lr_h, lr_w, dtype=torch.float32).to(device)
        lr_prev = torch.rand(1, c, lr_h, lr_w, dtype=torch.float32).to(device)
        hr_prev = torch.rand(1, c, s * lr_h, s * lr_w, dtype=torch.float32).to(device)
        return [lr_curr, lr_prev, hr_prev]

    def profile(self, lr_size, device=None):
        """(gflops_dict, params_dict) keyed 'FNet','SRNet' -- the numbers the reference's
        forward-hook counter prints (tecogan_nets.py:295-314), computed analytically because
        the parameter-holder modules are never executed."""
        _, lr_h, lr_w = lr_size
        gflops, params = OrderedDict(), OrderedDict()
        gflops['FNet'] = _conv_gflops(self.fnet.conv_layers(lr_h, lr_w))
        params['FNet'] = sum(p.numel() for p in self.fnet.parameters())
        gflops['SRNet'] = _conv_gflops(self.srnet.conv_layers(lr_h, lr_w))
        params['SRNet'] = sum(p.numel() for p in self.srnet.parameters())
        return gflops, params
