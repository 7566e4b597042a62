"""TEST INFRASTRUCTURE ONLY -- CPU precision model of the CUDA path.

Same algorithm as frnet_torchref.step, but with the storage precision of the sm_90a kernels:
weights and every inter-layer activation rounded to fp16, accumulation / bias / activation /
residual add in fp32, and the flow head, warp coordinates, bicubic residual and final output in
fp32 (DESIGN.md "precision").  It separates two questions in the GPU tests:

  * is the CUDA path a correct implementation of its own design?  -> GPU vs this model (tight)
  * is the design within the north-star tolerance of the reference? -> GPU vs the fp32 fixtures

With chaotic weights (gain 2.0 fixtures) the fp16 design itself is 3e-3 away from fp32; the
GPU result is then required to stay within a small factor of THIS model's distance.
"""
import torch
import torch.nn.functional as F

from . import frnet_torchref as R


def q(x):
    return x.half().float()


def step(p, lr_curr, lr_prev, hr_prev, scale, degradation, nb=10):
    pq = {k: (q(v) if k.endswith('weight') else v) for k, v in p.items()}

    def c(x, k, act=None):
        y = F.conv2d(x, pq[k + '.weight'], p[k + '.bias'], 1, 1)
        if act == 'lrelu':
            y = F.leaky_relu(y, 0.2)
        elif act == 'relu':
            y = F.relu(y)
        return y

    o = q(torch.cat([lr_curr, lr_prev], 1))
    for e in ('encoder1', 'encoder2', 'encoder3'):
        o = q(c(o, f'fnet.{e}.0', 'lrelu'))
        o = q(c(o, f'fnet.{e}.2', 'lrelu'))
        o = F.max_pool2d(o, 2, 2)
    for d in ('decoder1', 'decoder2', 'decoder3'):
        o = q(c(o, f'fnet.{d}.0', 'lrelu'))
        o = q(c(o, f'fnet.{d}.2', 'lrelu'))
        o = q(F.interpolate(o, scale_factor=2, mode='bilinear', align_corners=False))
    o = q(c(o, 'fnet.flow.0', 'lrelu'))
    flow = torch.tanh(c(o, 'fnet.flow.2')) * 24                       # fp32 out of the epilogue
    ph = lr_curr.size(2) - lr_curr.size(2) // 8 * 8
    pw = lr_curr.size(3) - lr_curr.size(3) // 8 * 8
    hr_flow = scale * R.upsample(p, F.pad(flow, (0, pw, 0, ph), 'reflect'), scale, degradation)
    x = q(torch.cat([lr_curr, R.s2d(R.warp(hr_prev, hr_flow), scale)], 1))
    o = q(c(x, 'srnet.conv_in.0', 'relu'))
    for i in range(nb):
        t = q(c(o, f'srnet.resblocks.{i}.conv.0', 'relu'))
        o = q(c(t, f'srnet.resblocks.{i}.conv.2') + o)
    for u in range(2 if scale == 4 else 1):
        k = f'srnet.conv_up.{2 * u}'
        o = q(F.relu(F.conv_transpose2d(o, pq[k + '.weight'], p[k + '.bias'], 2, 1, output_padding=1)))
    return c(o, 'srnet.conv_out') + R.upsample(p, lr_curr, scale, degradation), flow
