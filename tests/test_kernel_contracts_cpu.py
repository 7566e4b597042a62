"""The call-level contract replay (tests/kernel_contracts.py) run without a GPU: the stand-ins of
tests/fake_ops.py (fp16 storage, fp32 arithmetic) play the kernels.  Unperturbed, every call must stay inside
its bound and every faked op must be exercised; with one stand-in deliberately wrong, the replay must flag
it -- so the bounds the GPU test applies to the real kernels are tight enough to catch these mistakes."""
import importlib
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import tecogan_b200 as T                      # noqa: E402
import fake_ops as FK                         # noqa: E402
import kernel_contracts as KC                 # noqa: E402

P = 'tecogan-pytorch_b200.'


def _recorder(monkeypatch, perturb=None):
    ops = sys.modules[P + 'ops']
    FK.install(monkeypatch, ops, sys.modules[P + 'networks'], sys.modules[P + 'net_utils'],
               importlib.import_module(P + 'autograd'))
    monkeypatch.setattr(FK, 'STORAGE', torch.float16)
    for name, fn in (perturb or {}).items():
        monkeypatch.setattr(ops, name, fn)
    return KC.Recorder(ops, monkeypatch), ops


def _run(ops, nc=3):
    KC.run_sequence(T, 'cpu', 31, nb=1, n=2, t=3, h=16, w=16, nc=nc)
    KC.run_sequence(T, 'cpu', 32, nb=2, n=1, t=3, h=16, w=16, flow_losses=False, loss_mul=1e-7, nc=nc)
    KC.run_sequence(T, 'cpu', 33, nb=1, n=1, t=3, h=16, w=24, degradation='BI', scale=2, nc=nc)
    KC.run_module_ops(T, ops, 'cpu', 34)


@pytest.mark.parametrize('nc,degradation,scale,h,w', [(1, 'BD', 4, 8, 16), (2, 'BI', 2, 16, 8)],
                         ids=['nc1_bd4', 'nc2_bi2'])
def test_stand_ins_match_the_reference_sequence(monkeypatch, nc, degradation, scale, h, w):
    """FRNet(nc, nc).forward_sequence and its backward on the stand-ins with fp32 storage (no rounding) is
    oracle/frnet_torchref.forward_sequence under autograd: outputs and every parameter gradient, loss on hr_data,
    hr_flow and lr_flow"""
    import importlib
    from oracle import frnet_oracle as O
    from oracle import frnet_torchref as R
    FK.install(monkeypatch, sys.modules[P + 'ops'], sys.modules[P + 'networks'], sys.modules[P + 'net_utils'],
               importlib.import_module(P + 'autograd'))
    monkeypatch.setattr(FK, 'STORAGE', torch.float32)
    monkeypatch.setattr(importlib.import_module(P + 'autograd'), '_ACT_DTYPE', torch.float32)
    p = O.make_frnet_params(24, in_nc=nc, out_nc=nc, nb=1, scale=scale, degradation=degradation, gain=1.5)
    net = T.FRNet(nc, nc, 64, 1, degradation, scale)
    net.load_state_dict(p, strict=True)
    net.train()
    x = KC._rand(25, 2, 3, nc, h, w)
    keys = ('hr_data', 'hr_flow', 'lr_flow')
    d = net(x)
    ws = [KC._rand(26 + i, *d[k].shape, lo=-1, hi=1) for i, k in enumerate(keys)]
    sum((d[k] * g).sum() for k, g in zip(keys, ws)).backward()
    q = {k: v.clone().requires_grad_(v.is_floating_point() and not k.endswith('kernels')) for k, v in p.items()}
    dr = R.forward_sequence(q, x, scale, degradation, nb=1)
    names = [k for k in q if q[k].requires_grad]
    refs = torch.autograd.grad(sum((dr[k] * g).sum() for k, g in zip(keys, ws)), [q[k] for k in names])
    for k in keys:
        rel = float((d[k].detach() - dr[k].detach()).norm() / dr[k].detach().norm())
        assert rel <= 1e-6, (k, rel)
    named = dict(net.named_parameters())
    for k, gr in zip(names, refs):
        rel = float((named[k].grad - gr).norm() / gr.norm())
        assert rel <= 1e-5, (k, rel)


def test_replay_of_the_stand_ins_passes_and_covers_every_faked_op(monkeypatch):
    rec, ops = _recorder(monkeypatch)
    _run(ops)
    print(KC.report(rec))
    assert not rec.failures, rec.failures[:5]
    assert set(FK.FAKED) <= rec.seen, sorted(set(FK.FAKED) - rec.seen)
    assert not rec.unfaked


# ----------------------------------------------------------------------------------- perturbed stand-ins
class _DropTap(FK.PackedConv):
    """the centre tap of the output pixel in the middle of every image is left out"""

    def __call__(self, x, y=None, residual=None, **kw):
        out = super().__call__(x, y=y, residual=residual, **kw)
        if self.kind != FK.CONV_3X3 or self.epilogue != FK.EPI_NHWC_F16:
            return out
        w = self.w
        self.w = w.clone()
        self.w[:, :, 1, 1] = 0
        alt = super().__call__(x, residual=residual)
        self.w = w
        h, wd = out.shape[1] // 2, out.shape[2] // 2
        out[:, h, wd] = alt[:, h, wd]
        return out


def _wgrad_skips_last_pixel(fwd, x, dz, dw, scale=None, impl=None, max_ctas=0, db=None):
    dz = dz.clone()
    dz[-1, -1, -1] = 0
    return FK.wgrad(fwd, x, dz, dw, scale, impl, max_ctas, db)


def _upsample_bwd_overwrites(gy, scale_factor, up_mode, mul=1.0, gx=None, accumulate=False):
    return FK.upsample_bwd(gy, scale_factor, up_mode, mul, gx, False)


def _maxpool_bwd_last_max(x, gy, act, gx=None):
    c = x.shape[-1]
    a = FK.to_nchw(x, c)
    n, _, h, w = a.shape
    win = a[:, :, :h // 2 * 2, :w // 2 * 2].reshape(n, c, h // 2, 2, w // 2, 2).permute(0, 1, 2, 4, 3, 5)
    win = win.reshape(n, c, h // 2, w // 2, 4)
    last = 3 - win.flip(-1).argmax(-1)                         # the LAST maximum in row-major order
    g = torch.zeros_like(win).scatter_(-1, last.unsqueeze(-1), FK.to_nchw(gy, c).unsqueeze(-1))
    g = g.reshape(n, c, h // 2, w // 2, 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(n, c, h // 2 * 2, w // 2 * 2)
    g = F.pad(g, (0, w - w // 2 * 2, 0, h - h // 2 * 2))
    return FK.to_nhwc(g * FK._dact(a, act), c, out=gx)


def _warp_c1_swaps_s2d_channels(hr_prev, hr_flow, lr_curr, scale, out=None, cpad=64):
    """single-channel frames: the space_to_depth channels of sub-pixels (0, 0) and (0, 1) exchanged"""
    y = FK.warp_s2d_concat_hrflow(hr_prev, hr_flow, lr_curr, scale, out=out, cpad=cpad)
    if hr_prev.shape[1] == 1:
        y[..., 1], y[..., 2] = y[..., 2].clone(), y[..., 1].clone()
    return y


class _ScaleTwiceTooLarge(FK.GradScale):
    def _set(self, amax, target=None):
        super()._set(amax, target)
        self.ws[0], self.ws[1] = self.ws[0] * 2, self.ws[1] / 2
        return self


@pytest.mark.parametrize('name,fn,nc', [
    ('PackedConv', _DropTap, 3),
    ('wgrad', _wgrad_skips_last_pixel, 3),
    ('upsample_bwd', _upsample_bwd_overwrites, 3),
    ('maxpool2x2_bwd', _maxpool_bwd_last_max, 3),
    ('GradScale', _ScaleTwiceTooLarge, 3),
    ('warp_s2d_concat_hrflow', _warp_c1_swaps_s2d_channels, 1),
    ('wgrad', _wgrad_skips_last_pixel, 1),
], ids=['conv_drops_a_tap', 'wgrad_skips_last_pixel', 'upsample_bwd_ignores_accumulate',
        'maxpool_bwd_last_tied_maximum', 'loss_scale_one_power_too_large', 'warp_c1_swaps_s2d_channels',
        'wgrad_skips_last_pixel_nc1'])
def test_replay_flags_a_wrong_stand_in(monkeypatch, name, fn, nc):
    rec, ops = _recorder(monkeypatch, {name: fn})
    _run(ops, nc)
    flagged = [f for f in rec.failures if f.startswith(name + ' ')]
    print(KC.report(rec), rec.failures[:3])
    assert flagged, f'the replay did not flag the perturbed {name}'
