"""TEST INFRASTRUCTURE ONLY -- a torch/CPU stand-in for the kernels behind `tecogan-pytorch_b200/ops.py`
(the training path and the inference step),
with exactly the contracts of include/tecogan_b200.h (NHWC fp16 activations padded to 64 channels,
loss-scaled fp16 gradients, fp32 parameter gradients in the parameters' layouts).

Purpose: the training orchestration (autograd.py: which buffer feeds which dgrad / wgrad, masks,
residual skips, frame order of the BPTT, n-major vs t-major flow layouts) can be checked on the CPU
against the reference-generated gradient fixture BEFORE any GPU time is spent; the GPU tests then
only have to establish that each kernel honours its contract.  Never imported by the package.
"""
import math

import torch
import torch.nn.functional as F

from oracle import frnet_torchref as R

CONV_3X3, CONVT_3X3_S2, CONV_3X3_S2 = 0, 1, 2
ACT_NONE, ACT_RELU, ACT_LRELU02 = 0, 1, 2
EPI_NHWC_F16, EPI_FLOW_NCHW_F32, EPI_OUT_NCHW_F32 = 0, 1, 2
UP_BICUBIC, UP_BILINEAR = 0, 1


def pad64(c):
    return (c + 63) // 64 * 64


def to_nchw(x, c):            # NHWC fp16 -> NCHW fp32 (first c channels)
    return x[..., :c].to(COMPUTE).permute(0, 3, 1, 2).contiguous()


STORAGE = torch.float16      # torch.float32: no rounding anywhere -> the orchestration must be EXACT
COMPUTE = torch.float32      # arithmetic type (tests/kernel_contracts.py: float64 references on the kernels' inputs)


def _store(v):
    return v.to(STORAGE).to(COMPUTE)


def to_nhwc(x, cpad, out=None):   # NCHW fp32 -> NHWC (fp16 storage) padded
    n, c, h, w = x.shape
    y = torch.zeros(n, h, w, cpad, dtype=STORAGE) if out is None else out
    if out is not None:
        y.zero_()
    y[..., :c] = x.permute(0, 2, 3, 1).to(STORAGE)
    return y


def _act(v, act):
    if act == ACT_RELU:
        return torch.clamp_min(v, 0)
    if act == ACT_LRELU02:
        return torch.where(v >= 0, v, 0.2 * v)
    return v


def _dact(m, act):
    if act == ACT_NONE:
        return torch.ones_like(m)
    return torch.where(m > 0, torch.ones_like(m), torch.full_like(m, 0.0 if act == ACT_RELU else 0.2))


class PackedConv:
    def __init__(self, weight, bias, kind=CONV_3X3, act=ACT_NONE, epilogue=EPI_NHWC_F16):
        self.kind, self.act, self.epilogue = kind, act, epilogue
        if kind == CONV_3X3:
            self.cout_real, self.cin_real = weight.shape[0], weight.shape[1]
        else:
            self.cin_real, self.cout_real = weight.shape[0], weight.shape[1]
        self.cin = pad64(self.cin_real)
        self.tapn = epilogue != EPI_NHWC_F16
        self.cout = pad64(self.cout_real) if not self.tapn else 48
        self.refresh(weight, bias)

    def refresh(self, weight, bias, force=False):
        self.w = _store(weight.detach())        # fp16 storage of the packed weights
        self.b = bias.detach().to(COMPUTE)
        self.packed = self.w

    def __call__(self, x, y=None, residual=None, impl=None, a_mode=None, max_ctas=0, pool=False):
        xin = to_nchw(x, self.cin_real)
        if self.kind == CONV_3X3:
            v = F.conv2d(xin, self.w, self.b, 1, 1)
        else:
            v = F.conv_transpose2d(xin, self.w, self.b, 2, 1, output_padding=1)
        if self.epilogue == EPI_FLOW_NCHW_F32:
            v = 24 * torch.tanh(v)
        elif self.epilogue == EPI_NHWC_F16:
            v = _act(v, self.act)
            if residual is not None:
                v = v + to_nchw(residual, self.cout_real)
            if pool:                     # nn.MaxPool2d(2, 2) of the activated map (floor: odd last row / col dropped)
                v = F.max_pool2d(v, 2, 2)
        if self.epilogue == EPI_NHWC_F16:
            out = to_nhwc(v, self.cout)
        else:
            out = v
        if y is not None:
            y.copy_(out)
            return y
        return out


class PackedDgrad:
    def __init__(self, fwd, weight):
        self.fwd = fwd
        self.cin, self.cout = pad64(fwd.cout_real), fwd.cin
        self.refresh(weight)

    def refresh(self, weight, force=False):
        self.w = _store(weight.detach())

    def __call__(self, dz, y=None, residual=None, mask=None, mask_act=ACT_NONE, impl=None):
        f = self.fwd
        g = to_nchw(dz, f.cout_real)
        if f.kind == CONV_3X3:
            v = F.conv_transpose2d(g, self.w, None, 1, 1)            # = conv with flipped taps, roles swapped
        else:
            v = F.conv2d(g, self.w, None, 2, 1)                      # stride-2 conv with Wt read as OIHW
        if residual is not None:
            v = v + to_nchw(residual, f.cin_real)
        if mask is not None:
            v = v * _dact(to_nchw(mask, f.cin_real), mask_act)
        out = to_nhwc(v, self.cout)
        if y is not None:
            y.copy_(out)
            return y
        return out


class GradScale:
    TARGET = 256.0

    def __init__(self, device):
        self.ws = torch.tensor([1.0, 1.0, 0.0, 0.0])

    def _set(self, amax, target=None):
        # 2^floor(log2(target / amax)) with the exponent computed exactly: amax = ma * 2^ea, target = mt * 2^et
        # (ma, mt in [0.5, 1)) -> floor(log2(target / amax)) = et - ea - (mt < ma)
        s = 1.0
        if amax > 0 and math.isfinite(amax):
            ma, ea = math.frexp(amax)
            mt, et = math.frexp(target or self.TARGET)
            s = 2.0 ** max(-24, min(24, et - ea - (mt < ma)))
        self.ws[0], self.ws[1] = s, 1.0 / s
        return self

    def from_amax(self, a, b=None, target=None):
        amax = float(a.abs().max())
        if b is not None:
            bmax = float(b.abs().max())
            amax = bmax if math.isnan(bmax) else max(amax, bmax)
        return self._set(amax, target)

    @property
    def s(self):
        return float(self.ws[0])


def _s(scale):
    return scale.s if scale is not None else 1.0


@torch.enable_grad()
def wgrad(fwd, x, dz, dw, scale=None, impl=None, max_ctas=0, db=None):
    if db is not None:
        bias_grad(dz, db, scale)
    xin = to_nchw(x, fwd.cin_real).requires_grad_(False)
    g = to_nchw(dz, fwd.cout_real)
    w = torch.zeros_like(dw, requires_grad=True)
    if fwd.kind == CONV_3X3:
        y = F.conv2d(xin, w, None, 1, 1)
    else:
        y = F.conv_transpose2d(xin, w, None, 2, 1, output_padding=1)
    gw, = torch.autograd.grad(y, [w], g)
    dw += gw / _s(scale)
    return dw


def bias_grad(dz, db, scale=None):
    db += dz[..., :db.numel()].to(COMPUTE).sum((0, 1, 2)) / _s(scale)
    return db


def grad_pack(a, b=None, scale=None, cpad=64, y=None):
    v = a if b is None else a + b
    return to_nhwc(v * _s(scale), cpad, out=y)


def pack_pair(x1, x2, y=None, cpad=64):
    return to_nhwc(torch.cat([x1, x2], 1), cpad, out=y)


def nchw_to_nhwc(x, cpad=None, y=None):
    return to_nhwc(x, cpad or pad64(x.shape[1]), out=y)


def maxpool2x2(x, y=None):
    c = x.shape[-1]
    return to_nhwc(F.max_pool2d(to_nchw(x, c), 2, 2), c, out=y)


def upsample2x(x, y=None):
    c = x.shape[-1]
    return to_nhwc(F.interpolate(to_nchw(x, c), scale_factor=2, mode='bilinear', align_corners=False), c, out=y)


ABS_TAPS = False             # |filter taps|: the magnitude of the terms, for the error bounds of tests/kernel_contracts.py


def _up(x, scale, up_mode):
    from oracle.ops_oracle import bicubic_kernels
    k = torch.from_numpy(bicubic_kernels(scale)).to(x.dtype)
    p = {'upsample_func.kernels': k.abs() if ABS_TAPS else k}
    return R.upsample(p, x, scale, 'BD' if up_mode == UP_BICUBIC else 'BI')


def _reflect_pad(x, hw):
    """F.pad(x, 'reflect') on the bottom / right up to hw = (h, w) (tecogan_nets.py:239-241)"""
    if hw is None:
        return x
    h, w = hw
    return F.pad(x, (0, w - x.shape[3], 0, h - x.shape[2]), mode='reflect')


def upsample(x, scale, up_mode, out_hw=None, mul=1.0, y=None, accumulate=False):
    v = mul * _up(_reflect_pad(x, out_hw), scale, up_mode)
    if y is not None:
        if accumulate:
            y += v
        else:
            y.copy_(v)
        return y
    return v


@torch.enable_grad()
def upsample_bwd(gy, scale_factor, up_mode, mul=1.0, gx=None, accumulate=False):
    n, c, H, W = gy.shape
    x = torch.zeros(n, c, H // scale_factor, W // scale_factor, dtype=gy.dtype, requires_grad=True)
    g, = torch.autograd.grad(mul * _up(x, scale_factor, up_mode), [x], gy)
    if gx is None:
        return g
    if accumulate:
        gx += g
    else:
        gx.copy_(g)
    return gx


def warp_s2d_concat_hrflow(hr_prev, hr_flow, lr_curr, scale, out=None, cpad=64):
    v = torch.cat([lr_curr, R.s2d(R.warp(hr_prev, hr_flow), scale)], 1)
    return to_nhwc(v, cpad, out=out)


def warp_s2d_concat_lrflow(hr_prev, lr_flow, lr_curr, scale, up_mode, out=None, cpad=64):
    h, w = lr_curr.shape[2], lr_curr.shape[3]
    hr_flow = scale * _up(_reflect_pad(lr_flow, (h, w)), scale, up_mode)
    return warp_s2d_concat_hrflow(hr_prev, hr_flow, lr_curr, scale, out=out, cpad=cpad)


def float_to_uint8_nhwc(x, y=None):
    """uint8(clip(rint(x * 255), 0, 255)) as NHWC; the product is taken in fp32 (oracle.ops_oracle.float32_to_uint8),
    torch.round is round-half-to-even"""
    v = torch.round(x.to(torch.float32) * 255.0).clamp_(0, 255).to(torch.uint8).permute(0, 2, 3, 1)
    return _out(v.contiguous(), y)


def fused_tail(up, outc, x, lr_curr, lr_scale, up_mode, y=None, y_u8=None, max_ctas=0, accumulate=False):
    """SRNet tail: t = relu(convT(x) + b_up) at the storage precision, v = conv_out(t) + b_out;
    accumulate: y += v, else y = v + upsample_func(lr_curr) (lr_curr None: no residual) [, y_u8 = uint8(y)]"""
    v = outc(up(x))
    if accumulate:
        y += v
        return y
    if lr_curr is not None:
        v = v + _up(lr_curr, lr_scale, up_mode)
    y = _out(v, y)
    if y_u8 is not None:
        float_to_uint8_nhwc(y, y_u8)
    return y


@torch.enable_grad()
def warp_s2d_concat_bwd(gx, hr_prev, hr_flow, scale_factor, d_hr_prev=None, d_hr_flow=None, scale=None):
    c = hr_prev.shape[1]
    cin = (scale_factor ** 2 + 1) * c
    g = to_nchw(gx, cin)[:, c:] / _s(scale)
    hp = hr_prev.clone().requires_grad_(True)
    hf = hr_flow.clone().requires_grad_(True)
    v = R.s2d(R.warp(hp, hf), scale_factor)
    ghp, ghf = torch.autograd.grad(v, [hp, hf], g)
    if d_hr_prev is not None:
        d_hr_prev += ghp
    if d_hr_flow is not None:
        d_hr_flow.copy_(ghf)


@torch.enable_grad()
def maxpool2x2_bwd(x, gy, act, gx=None):
    c = x.shape[-1]
    a = to_nchw(x, c).requires_grad_(True)
    g, = torch.autograd.grad(F.max_pool2d(a, 2, 2), [a], to_nchw(gy, c))
    return to_nhwc(g * _dact(a.detach(), act), c, out=gx)


@torch.enable_grad()
def upsample2x_bwd(gy, m, act, gx=None):
    c = m.shape[-1]
    a = to_nchw(m, c).requires_grad_(True)
    g, = torch.autograd.grad(F.interpolate(a, scale_factor=2, mode='bilinear', align_corners=False), [a],
                             to_nchw(gy, c))
    return to_nhwc(g * _dact(a.detach(), act), c, out=gx)


def flow_head_bwd(gflow, flow, scale, gflow2=None, cpad=64, dz=None):
    g = gflow if gflow2 is None else gflow + gflow2
    v = g * (24.0 - flow * flow / 24.0)
    scale._set(float(v.abs().max()))
    return to_nhwc(v * scale.s, cpad, out=dz)


def _out(v, y):
    if y is None:
        return v
    y.copy_(v)
    return y


def backward_warp(x, flow, y=None):
    return _out(R.warp(x, flow), y)


@torch.enable_grad()
def backward_warp_bwd(x, flow, gy, need_x=True, need_flow=True):
    xx, ff = x.clone().requires_grad_(True), flow.clone().requires_grad_(True)
    gx, gf = torch.autograd.grad(R.warp(xx, ff), [xx, ff], gy)
    return (gx if need_x else None), (gf if need_flow else None)


def space_to_depth(x, scale, y=None):
    return _out(R.s2d(x, scale), y)


@torch.enable_grad()
def depth_to_space(gy, scale_factor):
    n, cs, oh, ow = gy.shape
    x = torch.zeros(n, cs // scale_factor ** 2, oh * scale_factor, ow * scale_factor, dtype=gy.dtype,
                    requires_grad=True)
    g, = torch.autograd.grad(R.s2d(x, scale_factor), [x], gy)
    return g


# every op of the training path, in the package's op layer, that this module stands in for
FAKED = ('PackedConv', 'PackedDgrad', 'GradScale', 'wgrad', 'bias_grad', 'grad_pack', 'pack_pair', 'nchw_to_nhwc',
         'maxpool2x2', 'upsample2x', 'upsample', 'upsample_bwd', 'warp_s2d_concat_hrflow', 'warp_s2d_concat_bwd',
         'maxpool2x2_bwd', 'upsample2x_bwd', 'flow_head_bwd', 'backward_warp', 'backward_warp_bwd',
         'space_to_depth', 'depth_to_space')
# the ops only the inference step (FRNet.step_into) adds to those
INFER_FAKED = ('fused_tail', 'warp_s2d_concat_lrflow', 'float_to_uint8_nhwc')


def install(monkeypatch, pkg_ops, networks, net_utils, autograd):
    """Route the package's op layer to this module (CPU tensors accepted)."""
    import sys
    me = sys.modules[__name__]
    for name in FAKED + INFER_FAKED:
        monkeypatch.setattr(pkg_ops, name, getattr(me, name))
    monkeypatch.setattr(networks, '_cuda_f32', lambda t, name: t.detach().float().contiguous())
    monkeypatch.setattr(net_utils, '_chk', lambda t, name: t)
    monkeypatch.setattr(net_utils, '_f32', lambda t, name: t.detach().float().contiguous())
