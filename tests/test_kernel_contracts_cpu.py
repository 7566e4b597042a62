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


def _run(ops):
    KC.run_sequence(T, 'cpu', 31, nb=1, n=2, t=3, h=16, w=16)
    KC.run_sequence(T, 'cpu', 32, nb=2, n=1, t=3, h=16, w=16, flow_losses=False, loss_mul=1e-7)
    KC.run_sequence(T, 'cpu', 33, nb=1, n=1, t=3, h=16, w=24, degradation='BI', scale=2)
    KC.run_module_ops(T, ops, 'cpu', 34)


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


class _ScaleTwiceTooLarge(FK.GradScale):
    def _set(self, amax, target=None):
        super()._set(amax, target)
        self.ws[0], self.ws[1] = self.ws[0] * 2, self.ws[1] / 2
        return self


@pytest.mark.parametrize('name,fn', [
    ('PackedConv', _DropTap),
    ('wgrad', _wgrad_skips_last_pixel),
    ('upsample_bwd', _upsample_bwd_overwrites),
    ('maxpool2x2_bwd', _maxpool_bwd_last_max),
    ('GradScale', _ScaleTwiceTooLarge),
], ids=['conv_drops_a_tap', 'wgrad_skips_last_pixel', 'upsample_bwd_ignores_accumulate',
        'maxpool_bwd_last_tied_maximum', 'loss_scale_one_power_too_large'])
def test_replay_flags_a_wrong_stand_in(monkeypatch, name, fn):
    rec, ops = _recorder(monkeypatch, {name: fn})
    _run(ops)
    flagged = [f for f in rec.failures if f.startswith(name + ' ')]
    print(KC.report(rec), rec.failures[:3])
    assert flagged, f'the replay did not flag the perturbed {name}'
