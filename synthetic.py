"""Seeded synthetic weights and clips for benchmarks, smoke tests and parity tests.

Neutral module: neither product code (tecogan-pytorch_b200/) nor checker (oracle/) -- both the
bench driver and the tests draw their inputs from here so that every box regenerates identical
data from a seed (numpy PCG64 stream) instead of shipping tensors.  The reference has no
equivalent: codes/main.py:227-228 profiles with PyTorch's default init and
FRNet.generate_dummy_data draws torch.rand inputs (tecogan_nets.py:283-293).
"""
from collections import OrderedDict

import numpy as np
import torch

F32 = np.float32


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a))


def bicubic_kernels(scale, a=-0.75):
    """kernels[d] = cubic @ [1, t, t^2, t^3], t = d/scale -- the BicubicUpsampler buffer
    (codes/utils/net_utils.py:116-131); part of a BD state_dict."""
    cubic = np.array([[0, a, -2 * a, a],
                      [1, 0, -(a + 3), a + 2],
                      [0, -a, (2 * a + 3), -(a + 2)],
                      [0, 0, a, -a]], dtype=F32)
    ks = []
    for d in range(scale):
        t = F32(1.0 * d / scale)
        ks.append(cubic @ np.array([1, t, t * t, t * t * t], dtype=F32))
    return np.stack(ks).astype(F32)


def _smooth_upsample(x, scale):
    """separable 4-tap cubic interpolation with replicate borders (only used to make the
    synthetic clips smooth; vertical pass first)"""
    x = np.asarray(x, dtype=F32)
    n, c, h, w = x.shape
    s = scale
    k = bicubic_kernels(s)
    ry = np.clip(np.arange(h)[:, None] + np.arange(-1, 3)[None, :], 0, h - 1)
    rx = np.clip(np.arange(w)[:, None] + np.arange(-1, 3)[None, :], 0, w - 1)
    v = np.zeros((n, c, h, s, w), dtype=F32)
    for i in range(4):
        v += k[None, None, None, :, i, None] * x[:, :, ry[:, i], :][:, :, :, None, :]
    v = v.reshape(n, c, h * s, w)
    o = np.zeros((n, c, h * s, w, s), dtype=F32)
    for j in range(4):
        o += k[None, None, None, None, :, j] * v[:, :, :, rx[:, j]][..., None]
    return o.reshape(n, c, h * s, w * s).astype(F32)


# ---------------------------------------------------------------------------- weights
# deterministic weights with the reference's state_dict layout (SURVEY.md 8-b)
def frnet_param_shapes(in_nc=3, out_nc=3, nf=64, nb=10, scale=4, degradation='BD'):
    shapes = OrderedDict()

    def conv(name, cin, cout):
        shapes[name + '.weight'] = (cout, cin, 3, 3)
        shapes[name + '.bias'] = (cout,)

    if degradation == 'BD':
        shapes['upsample_func.kernels'] = (scale, 4)
    chans = [('encoder1', 2 * in_nc, 32, 32), ('encoder2', 32, 64, 64), ('encoder3', 64, 128, 128),
             ('decoder1', 128, 256, 256), ('decoder2', 256, 128, 128), ('decoder3', 128, 64, 64)]
    for nm, a, b, c2 in chans:
        conv(f'fnet.{nm}.0', a, b)
        conv(f'fnet.{nm}.2', b, c2)
    conv('fnet.flow.0', 64, 32)
    conv('fnet.flow.2', 32, 2)
    conv('srnet.conv_in.0', (scale * scale + 1) * in_nc, nf)
    for i in range(nb):
        conv(f'srnet.resblocks.{i}.conv.0', nf, nf)
        conv(f'srnet.resblocks.{i}.conv.2', nf, nf)
    for u in range(2 if scale == 4 else 1):
        shapes[f'srnet.conv_up.{2 * u}.weight'] = (nf, nf, 3, 3)  # ConvT: [Cin,Cout,kH,kW]
        shapes[f'srnet.conv_up.{2 * u}.bias'] = (nf,)
    conv('srnet.conv_out', nf, out_nc)
    if degradation == 'BD':
        shapes['srnet.upsample_func.kernels'] = (scale, 4)
    return shapes


def make_frnet_params(seed=0, in_nc=3, out_nc=3, nf=64, nb=10, scale=4, degradation='BD',
                      gain=1.0):
    """Seeded weights, U(-b, b) with b = gain/sqrt(fan_in) like PyTorch's default
    conv init (what codes/main.py:227-228 profiles with; no checkpoint is loaded).
    numpy PCG64 stream -> identical on every box."""
    rng = np.random.default_rng(seed)
    p = OrderedDict()
    for name, shp in frnet_param_shapes(in_nc, out_nc, nf, nb, scale, degradation).items():
        if name.endswith('kernels'):
            p[name] = _t(bicubic_kernels(scale))
            continue
        if name.endswith('.weight'):
            if 'conv_up' in name:
                fan_in = shp[1] * 9   # torch computes fan_in from dim 1 for ConvTranspose2d
            else:
                fan_in = shp[1] * 9
            last_fan_in = fan_in
        else:
            fan_in = last_fan_in
        b = gain / np.sqrt(fan_in)
        p[name] = _t(rng.uniform(-b, b, size=shp).astype(np.float32))
    return p


def make_clip(seed, t, c, h, w, shift=1):
    """Smooth translating pattern (SURVEY.md 8-d): bicubic-upsampled seeded noise
    shifted `shift` px per frame, values in [0,1]."""
    rng = np.random.default_rng(seed)
    gh, gw = h // 4 + 4, (w + shift * t) // 4 + 4
    base = rng.uniform(0.0, 1.0, size=(1, c, gh, gw)).astype(np.float32)
    big = np.clip(_smooth_upsample(base, 4), 0.0, 1.0)
    frames = [big[0, :, 2:2 + h, 2 + shift * i:2 + shift * i + w] for i in range(t)]
    return _t(np.stack(frames).astype(np.float32))


def make_lpips_params(seed=0):
    """Seeded weights of LPIPS net-lin AlexNet v0.1 (numpy float32), under torchvision's keys features.{0,3,6,8,10}.*
    and the heads lin{0..4}.model.1.weight.  Convs at the scale of PyTorch's default Conv2d init (uniform in
    +-1/sqrt(fan_in)); heads non-negative, as the published ones are."""
    rng = np.random.default_rng(seed)
    shapes = ((64, 3, 11, 11), (192, 64, 5, 5), (384, 192, 3, 3), (256, 384, 3, 3), (256, 256, 3, 3))
    p = OrderedDict()
    for idx, shape in zip((0, 3, 6, 8, 10), shapes):
        bound = 1.0 / np.sqrt(np.prod(shape[1:]))
        p[f'features.{idx}.weight'] = rng.uniform(-bound, bound, shape).astype(np.float32)
        p[f'features.{idx}.bias'] = rng.uniform(-bound, bound, shape[0]).astype(np.float32)
    for l, shape in enumerate(shapes):
        p[f'lin{l}.model.1.weight'] = rng.uniform(0, 0.5, (1, shape[0], 1, 1)).astype(np.float32)
    return p
