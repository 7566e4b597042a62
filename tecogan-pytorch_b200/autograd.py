"""Training path of the generator: forward AND backward on libtecogan_b200 kernels, exposed to
PyTorch as torch.autograd.Function objects so the reference's training loops run unchanged
(VSRModel.train / VSRGANModel.train: codes/models/vsr_model.py:61-95, vsrgan_model.py:98-286).

What autograd sees                                   reference lines
  SequenceFunction   FRNet.forward_sequence           tecogan_nets.py:174-225
  FNetFunction       net_G.fnet(x1, x2)               tecogan_nets.py:67-82, called bare by the D at :420
  WarpFunction       net_utils.backward_warp          net_utils.py:50-82  (warp loss, D input builder)
  UpsampleFunction   net_G.upsample_func              net_utils.py:85-156 (bi_data for the D)
  SpaceToDepthFunction                                net_utils.py:36-47

Design (DESIGN.md section 8): activations are kept as the forward stored them (NHWC fp16, one buffer
per layer covering all T frames), gradients travel between conv layers as loss-scaled NHWC fp16,
  dgrad  = the forward wgmma implicit GEMM with swapped roles / flipped taps (+ act' epilogue),
  wgrad  = a wgmma GEMM over pixels, ONE launch per layer over all T*n images,
  warp   = scatter-add into the fp32 state gradient + gather for the flow gradient,
parameter gradients come out fp32 in the parameters' own layouts.  Nothing here calls a PyTorch
library kernel for arithmetic; torch is used for allocation, views and transposes of the fp32
boundary tensors.
"""
import torch
from torch.autograd.function import once_differentiable

from . import lib as L
from . import ops
from .net_utils import up_mode_of

_RELU, _LRELU, _NONE = L.ACT_RELU, L.ACT_LRELU02, L.ACT_NONE
_ACT_DTYPE = torch.float16      # storage type of activations and (loss-scaled) gradients between layers


def _f32c(t):
    return t.detach().float().contiguous()


class _Grads:
    """fp32 gradient buffers keyed by parameter (zero-initialised on first touch)."""

    def __init__(self):
        self.by_id = {}

    def of(self, p):
        g = self.by_id.get(id(p))
        if g is None:
            g = self.by_id[id(p)] = torch.zeros_like(p, dtype=torch.float32)
        return g

    def result(self, params):
        return tuple(self.by_id.get(id(p)) for p in params)


def _param_grads(pc, module, x, dz, scale, grads):
    """weight + bias gradient of one conv layer (x = its input, dz = d loss / d pre-activation)"""
    n = x.shape[0] * x.shape[1] if x.dim() == 5 else None
    if n is not None:                      # [T,n,h,w,c] buffers: one launch over all T*n images
        x = x.view(-1, *x.shape[2:])
        dz = dz.view(-1, *dz.shape[2:])
    # the bias gradient comes from the wgrad call (conv layers: a reduction after its GEMM) or a separate reduction
    ops.wgrad(pc, x, dz, grads.of(module.weight), scale, db=grads.of(module.bias))


# ================================================================================ FNet
def fnet_forward_train(fnet, x1, x2):
    """FNet.forward keeping every layer's output: -> (flow NCHW fp32, tape)"""
    a = ops.pack_pair(x1, x2)
    tape = {}
    for name, _, _ in fnet.ENC:
        ya = fnet._conv(name, 0, _LRELU)(a)
        yb = fnet._conv(name, 2, _LRELU)(ya)
        tape[name] = (a, ya, yb)
        a = ops.maxpool2x2(yb)
    for name, _, _ in fnet.DEC:
        ya = fnet._conv(name, 0, _LRELU)(a)
        yb = fnet._conv(name, 2, _LRELU)(ya)
        tape[name] = (a, ya, yb)
        a = ops.upsample2x(yb)
    f0 = fnet._conv('flow', 0, _LRELU)(a)
    flow = fnet._conv('flow', 2, _NONE, L.EPI_FLOW_NCHW_F32)(f0)
    tape['flow'] = (a, f0, flow)
    return flow, tape


def fnet_backward(fnet, tape, g_flow, g_flow2, grads):
    """parameter gradients of FNet from d loss / d flow (two addends allowed); no input gradient."""
    sc = ops.GradScale(g_flow.device)
    u3, f0, flow = tape['flow']
    dg = fnet._cache.dgrad
    dz = ops.flow_head_bwd(g_flow, flow, sc, gflow2=g_flow2)                 # also picks the loss scale
    _param_grads(fnet._conv('flow', 2, _NONE, L.EPI_FLOW_NCHW_F32), fnet.flow[2], f0, dz, sc, grads)
    dz = dg(('flow', 2), fnet.flow[2])(dz, mask=f0, mask_act=_LRELU)
    _param_grads(fnet._conv('flow', 0, _LRELU), fnet.flow[0], u3, dz, sc, grads)
    g = dg(('flow', 0), fnet.flow[0])(dz)
    for name, _, _ in reversed(fnet.DEC):
        a_in, ya, yb = tape[name]
        blk = getattr(fnet, name)
        dz = ops.upsample2x_bwd(g, yb, _LRELU)
        _param_grads(fnet._conv(name, 2, _LRELU), blk[2], ya, dz, sc, grads)
        dz = dg((name, 2), blk[2])(dz, mask=ya, mask_act=_LRELU)
        _param_grads(fnet._conv(name, 0, _LRELU), blk[0], a_in, dz, sc, grads)
        g = dg((name, 0), blk[0])(dz)
    for name, _, _ in reversed(fnet.ENC):
        a_in, ya, yb = tape[name]
        blk = getattr(fnet, name)
        dz = ops.maxpool2x2_bwd(yb, g, _LRELU)
        _param_grads(fnet._conv(name, 2, _LRELU), blk[2], ya, dz, sc, grads)
        dz = dg((name, 2), blk[2])(dz, mask=ya, mask_act=_LRELU)
        _param_grads(fnet._conv(name, 0, _LRELU), blk[0], a_in, dz, sc, grads)
        if name != fnet.ENC[0][0]:
            g = dg((name, 0), blk[0])(dz)


class FNetFunction(torch.autograd.Function):
    """net_G.fnet(x1, x2) under autograd (the ST-discriminator calls it bare, tecogan_nets.py:420)."""

    @staticmethod
    def forward(ctx, fnet, x1, x2, *params):
        flow, tape = fnet_forward_train(fnet, _f32c(x1), _f32c(x2))
        ctx.fnet, ctx.tape, ctx.params = fnet, tape, params
        return flow

    @staticmethod
    @once_differentiable
    def backward(ctx, g_flow):
        grads = _Grads()
        fnet_backward(ctx.fnet, ctx.tape, _f32c(g_flow), None, grads)
        ctx.tape = None
        return (None, None, None) + grads.result(ctx.params)


# ================================================================================ SRNet / sequence
class _SeqTape:
    pass


def _srnet_layers(srnet):
    c = srnet._cache
    pc_in = c.get('in', srnet.conv_in[0], L.CONV_3X3, _RELU)
    pcs1 = [c.get(('r', i, 0), blk.conv[0], L.CONV_3X3, _RELU) for i, blk in enumerate(srnet.resblocks)]
    pcs2 = [c.get(('r', i, 2), blk.conv[2], L.CONV_3X3, _NONE) for i, blk in enumerate(srnet.resblocks)]
    ups = [c.get(('up', u), srnet.conv_up[u], L.CONVT_3X3_S2, _RELU) for u in range(0, len(srnet.conv_up), 2)]
    pc_out = c.get('out', srnet.conv_out, L.CONV_3X3, _NONE, L.EPI_OUT_NCHW_F32)
    return pc_in, pcs1, pcs2, ups, pc_out


def sequence_forward_train(net, lr_data):
    """FRNet.forward_sequence keeping what the backward needs (reference :174-225)."""
    n, t, c, h, w = lr_data.shape
    s = net.scale
    dev = lr_data.device
    srnet, fnet = net.srnet, net.fnet
    if h % 8 or w % 8:
        raise L.TecoganB200Error('forward_sequence: LR size must be a multiple of 8 (the reference upsamples the '
                                 'FNet flow without padding, tecogan_nets.py:189)')
    up_mode = up_mode_of(net.upsample_func)
    tp = _SeqTape()
    tp.shape = (n, t, c, h, w)
    lr_prev = lr_data[:, :-1].reshape(n * (t - 1), c, h, w)
    lr_curr = lr_data[:, 1:].reshape(n * (t - 1), c, h, w)
    lr_flow, tp.fnet = fnet_forward_train(fnet, lr_curr, lr_prev)
    hr_flow = ops.upsample(lr_flow, s, up_mode, mul=float(s)).view(n, t - 1, 2, s * h, s * w)
    tp.flows = hr_flow.transpose(0, 1).contiguous()                      # [t-1,n,2,H,W]
    frames = lr_data.transpose(0, 1).contiguous()                        # [t,n,c,h,w]
    tp.hr = torch.empty((t, n, c, s * h, s * w), dtype=torch.float32, device=dev)

    pc_in, pcs1, pcs2, ups, pc_out = _srnet_layers(srnet)
    nb = len(pcs1)
    f16 = dict(dtype=_ACT_DTYPE, device=dev)
    tp.x = torch.empty((t, n, h, w, 64), **f16)
    tp.a = [torch.empty((t, n, h, w, 64), **f16) for _ in range(nb + 1)]
    tp.tt = [torch.empty((t, n, h, w, 64), **f16) for _ in range(nb)]
    tp.up = [torch.empty((t, n, h << (k + 1), w << (k + 1), 64), **f16) for k in range(len(ups))]
    for i in range(t):
        if i == 0:
            ops.nchw_to_nhwc(frames[0], 64, y=tp.x[0])                   # hr_prev_tran = zeros (:194-197)
        else:
            ops.warp_s2d_concat_hrflow(tp.hr[i - 1], tp.flows[i - 1], frames[i], s, out=tp.x[i])
        pc_in(tp.x[i], y=tp.a[0][i])
        for b in range(nb):
            pcs1[b](tp.a[b][i], y=tp.tt[b][i])
            pcs2[b](tp.tt[b][i], y=tp.a[b + 1][i], residual=tp.a[b][i])
        src = tp.a[nb][i]
        for k, up in enumerate(ups):
            up(src, y=tp.up[k][i])
            src = tp.up[k][i]
        pc_out(src, y=tp.hr[i])
        ops.upsample(frames[i], s, up_mode, y=tp.hr[i], accumulate=True)
    out = {
        'hr_data': tp.hr.transpose(0, 1).contiguous(),                   # n,t,c,H,W
        'hr_flow': hr_flow,
        'lr_prev': lr_prev,
        'lr_curr': lr_curr,
        'lr_flow': lr_flow,
    }
    return out, tp


def sequence_backward(net, tp, g_hr_data, g_hr_flow, g_lr_flow, grads):
    n, t, c, h, w = tp.shape
    s = net.scale
    srnet, fnet = net.srnet, net.fnet
    up_mode = up_mode_of(net.upsample_func)
    dev = tp.hr.device
    pc_in, pcs1, pcs2, ups, pc_out = _srnet_layers(srnet)
    nb = len(pcs1)
    dg = srnet._cache.dgrad
    H, W = s * h, s * w
    d_flows = torch.zeros((t - 1, n, 2, H, W), dtype=torch.float32, device=dev)
    if g_hr_data is not None:
        # state gradient per frame: the loss's own gradient, plus what later frames scatter into it
        d_hr = g_hr_data.detach().float().transpose(0, 1).contiguous()   # [t,n,c,H,W] (a copy: accumulated into)
        if d_hr.data_ptr() == g_hr_data.data_ptr():
            d_hr = d_hr.clone()
        sc = ops.GradScale(dev).from_amax(d_hr)
        f16 = dict(dtype=_ACT_DTYPE, device=dev)
        dz_out = torch.empty((t, n, H, W, 64), **f16)
        dz_up = [torch.empty_like(u) for u in tp.up]
        dz_c1 = [torch.empty((t, n, h, w, 64), **f16) for _ in range(nb)]
        dz_c2 = [torch.empty((t, n, h, w, 64), **f16) for _ in range(nb)]
        dz_in = torch.empty((t, n, h, w, 64), **f16)
        gx = torch.empty((n, h, w, 64), **f16)
        dg_out = dg('out', srnet.conv_out, pc_out)
        dg_up = [dg(('up', 2 * k), srnet.conv_up[2 * k], ups[k]) for k in range(len(ups))]
        dg_c1 = [dg(('r', b, 0), srnet.resblocks[b].conv[0], pcs1[b]) for b in range(nb)]
        dg_c2 = [dg(('r', b, 2), srnet.resblocks[b].conv[2], pcs2[b]) for b in range(nb)]
        dg_in = dg('in', srnet.conv_in[0], pc_in)
        for i in range(t - 1, -1, -1):
            ops.grad_pack(d_hr[i], scale=sc, y=dz_out[i])
            # conv_out -> last transposed conv (ReLU') -> ... -> first transposed conv
            dg_out(dz_out[i], y=dz_up[-1][i], mask=tp.up[-1][i], mask_act=_RELU)
            for k in range(len(ups) - 1, 0, -1):
                dg_up[k](dz_up[k][i], y=dz_up[k - 1][i], mask=tp.up[k - 1][i], mask_act=_RELU)
            if nb == 0:
                dg_up[0](dz_up[0][i], y=dz_in[i], mask=tp.a[0][i], mask_act=_RELU)
            else:
                dg_up[0](dz_up[0][i], y=dz_c2[nb - 1][i])               # d a[nb] = dz of the last conv2 (no act)
                for b in range(nb - 1, -1, -1):
                    dg_c2[b](dz_c2[b][i], y=dz_c1[b][i], mask=tp.tt[b][i], mask_act=_RELU)
                    if b > 0:                                             # d a[b] = dgrad + skip
                        dg_c1[b](dz_c1[b][i], y=dz_c2[b - 1][i], residual=dz_c2[b][i])
                    else:                                                 # a[0] = relu(conv_in)
                        dg_c1[0](dz_c1[0][i], y=dz_in[i], residual=dz_c2[0][i], mask=tp.a[0][i], mask_act=_RELU)
            if i > 0:
                dg_in(dz_in[i], y=gx)
                ops.warp_s2d_concat_bwd(gx, tp.hr[i - 1], tp.flows[i - 1], s, d_hr_prev=d_hr[i - 1],
                                        d_hr_flow=d_flows[i - 1], scale=sc)
        # parameter gradients: one wgrad launch per layer over all t*n images
        _param_grads(pc_out, srnet.conv_out, tp.up[-1], dz_out, sc, grads)
        for k in range(len(ups) - 1, -1, -1):
            _param_grads(ups[k], srnet.conv_up[2 * k], tp.up[k - 1] if k > 0 else tp.a[nb], dz_up[k], sc, grads)
        for b in range(nb):
            _param_grads(pcs2[b], srnet.resblocks[b].conv[2], tp.tt[b], dz_c2[b], sc, grads)
            _param_grads(pcs1[b], srnet.resblocks[b].conv[0], tp.a[b], dz_c1[b], sc, grads)
        _param_grads(pc_in, srnet.conv_in[0], tp.x, dz_in, sc, grads)
    # ---- flow path: d hr_flow (from the warps + the caller's own) -> d lr_flow -> FNet
    d_hr_flow = d_flows.transpose(0, 1).contiguous().view(n * (t - 1), 2, H, W)
    if g_hr_flow is not None:
        d_hr_flow = d_hr_flow + g_hr_flow.detach().float().reshape(n * (t - 1), 2, H, W)
    d_lr_flow = ops.upsample_bwd(d_hr_flow, s, up_mode, mul=float(s))
    g2 = _f32c(g_lr_flow) if g_lr_flow is not None else None
    fnet_backward(fnet, tp.fnet, d_lr_flow, g2, grads)


class SequenceFunction(torch.autograd.Function):
    """FRNet.forward_sequence: outputs (hr_data, hr_flow, lr_flow); gradients flow to the parameters
    (lr_data is data: its gradient is not produced)."""

    @staticmethod
    def forward(ctx, net, lr_data, *params):
        out, tape = sequence_forward_train(net, _f32c(lr_data))
        ctx.net, ctx.tape, ctx.params = net, tape, params
        ctx.aux = (out['lr_prev'], out['lr_curr'])
        return out['hr_data'], out['hr_flow'], out['lr_flow']

    @staticmethod
    @once_differentiable
    def backward(ctx, g_hr_data, g_hr_flow, g_lr_flow):
        grads = _Grads()
        sequence_backward(ctx.net, ctx.tape, g_hr_data, g_hr_flow, g_lr_flow, grads)
        ctx.tape = None
        return (None, None) + grads.result(ctx.params)


# ================================================================================ module-boundary ops
class WarpFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, flow):
        x, flow = _f32c(x), _f32c(flow)
        ctx.save_for_backward(x, flow)
        return ops.backward_warp(x, flow)

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        x, flow = ctx.saved_tensors
        gx, gf = ops.backward_warp_bwd(x, flow, _f32c(gy), ctx.needs_input_grad[0], ctx.needs_input_grad[1])
        return gx, gf


class UpsampleFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, scale, up_mode):
        ctx.scale, ctx.up_mode = scale, up_mode
        return ops.upsample(_f32c(x), scale, up_mode)

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        return ops.upsample_bwd(_f32c(gy), ctx.scale, ctx.up_mode), None, None


class SpaceToDepthFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, scale):
        ctx.scale = scale
        return ops.space_to_depth(_f32c(x), scale)

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        return ops.depth_to_space(_f32c(gy), ctx.scale), None


class StDiscInputFunction(torch.autograd.Function):
    """The tensor plumbing in front of the spatio-temporal discriminator (tecogan_nets.py:438-463) as one
    kernel + one gradient kernel; gradient flows to `data` only (the reference detaches the flows)."""

    @staticmethod
    def forward(ctx, data, bi_data, hr_flow_merge, t, pad, csize):
        data, bi, flow = _f32c(data), _f32c(bi_data), _f32c(hr_flow_merge)
        ctx.save_for_backward(flow)
        ctx.meta = (tuple(data.shape), t, pad, csize)
        return ops.st_disc_input(data, bi, flow, t, pad, csize)

    @staticmethod
    @once_differentiable
    def backward(ctx, gout):
        flow, = ctx.saved_tensors
        shape, t, pad, csize = ctx.meta
        return ops.st_disc_input_bwd(_f32c(gout), flow, shape, t, pad, csize), None, None, None, None, None


def st_discriminator_input(data, bi_data, hr_flow_merge, spatial_size, crop_border_ratio=0.75):
    """Drop-in for lines 438-463 of SpatioTemporalDiscriminator.forward_sequence: data / bi_data [n,T,c,H,W]
    (only the first T//3*3 frames are used), hr_flow_merge [n*(T//3*3), 2, H, W] -> [n*T//3, 9c, H, W]."""
    t = data.shape[1] // 3 * 3
    csize = int(spatial_size * crop_border_ratio)
    pad = (spatial_size - csize) // 2
    return StDiscInputFunction.apply(data, bi_data[:, :data.shape[1]], hr_flow_merge.detach(), t, pad, csize)


# ================================================================================ VGG19 perceptual loss
def vgg_forward(vgg, x, keep):
    """VGGFeatureExtractor.forward on the kernels: x NCHW fp32 [N,3,H,W] -> (features NCHW fp32, tape).  keep=True
    keeps every conv's NHWC fp16 output (the ReLU' masks and max-pool routes of the backward) in the tape; keep=False
    keeps nothing, and each map is freed once the next layer has read it."""
    layers = vgg.packed_layers()
    a = ops.grad_pack_ex(x, sub=vgg.mean.view(3), div=vgg.std.view(3))     # (x - mean) / std, 64 channels
    outs, feats = [], {}
    for u, ((fwd, _), (_, _, pool)) in enumerate(zip(layers, vgg._units)):
        a = fwd(a)
        if u in vgg._taps:
            feats[u] = ops.nhwc_to_nchw(a, fwd.cout_real)
        if keep:
            outs.append(a)
        if pool and u + 1 < len(layers):
            a = ops.maxpool2x2(a)
    return [feats[u] for u in vgg._taps], outs


def vgg_backward(vgg, outs, grads):
    """input gradient of the extractor: grads[k] = d loss / d feature k (NCHW fp32) -> d loss / d x (NCHW fp32).

    Walks the units from the deepest tap to conv1_1 with dz = d loss / d (pre-ReLU output of the unit), loss-scaled
    NHWC fp16 under ONE scale chosen from the amax over all the taps' gradients.  A tap on a unit followed by a conv
    joins as the dgrad epilogue's residual, (dgrad + tap) * ReLU'; a tap on a unit followed by a max-pool joins after
    the pool's backward, (route + tap) * ReLU' (tg_grad_pack_ex_nhwc_f16)."""
    layers = vgg.packed_layers()
    tap_of = {u: k for k, u in enumerate(vgg._taps)}
    sc = ops.GradScale(outs[0].device).from_amax_of(grads)
    last = len(layers) - 1
    dz = ops.grad_pack_ex(grads[tap_of[last]], scale=sc, mask=outs[last], mask_act=_RELU, cpad=outs[last].shape[-1])
    for u in range(last, 0, -1):
        dg = layers[u][1]
        prev, pool = outs[u - 1], vgg._units[u - 1][2]
        k = tap_of.get(u - 1)
        if not pool:
            res = ops.grad_pack(grads[k], scale=sc, cpad=prev.shape[-1]) if k is not None else None
            dz = dg(dz, residual=res, mask=prev, mask_act=_RELU)
        elif k is None:
            dz = ops.maxpool2x2_bwd(prev, dg(dz), _RELU)
        else:
            route = ops.maxpool2x2_bwd(prev, dg(dz), _NONE)
            dz = ops.grad_pack_ex(grads[k], scale=sc, add=route, mask=prev, mask_act=_RELU, cpad=prev.shape[-1])
    g = layers[0][1](dz)                                                 # d loss / d normalised input, 64 channels
    return ops.grad_unpack_ex(g, 3, vgg.std.view(3), scale=sc)


class VGGFeaturesFunction(torch.autograd.Function):
    """VGGFeatureExtractor.forward under autograd: outputs the features; the gradient flows to the input only."""

    @staticmethod
    def forward(ctx, vgg, x):
        feats, outs = vgg_forward(vgg, _f32c(x), keep=True)
        ctx.vgg, ctx.outs = vgg, outs
        return tuple(feats)

    @staticmethod
    @once_differentiable
    def backward(ctx, *g):
        gx = vgg_backward(ctx.vgg, ctx.outs, [_f32c(t) for t in g])
        ctx.outs = None
        return None, gx
