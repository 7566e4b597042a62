"""The contract replay of the inference step (tests/kernel_contracts.py) without a GPU.

First the stand-ins of tests/fake_ops.py are pinned to the reference: with fp32 storage, FRNet.step_into on them
(fused tail in both modes or the separate launches, pooled or separate max-pools, the lrflow warp with its reflect
pad, the uint8 frame) is oracle/frnet_torchref.step.  Then, with fp16 storage, the stand-ins play the kernels: the
replay of small ragged scenarios must pass and reach every op of the inference path, and with one stand-in
deliberately wrong it must flag that op -- so the bounds the GPU test applies to the real kernels catch these
mistakes."""
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
from oracle import frnet_oracle as O          # noqa: E402
from oracle import frnet_torchref as R        # noqa: E402
from oracle import ops_oracle as K            # noqa: E402

P = 'tecogan-pytorch_b200.'
NAMES = FK.FAKED + FK.INFER_FAKED


def _install(monkeypatch, storage):
    ops = sys.modules[P + 'ops']
    FK.install(monkeypatch, ops, sys.modules[P + 'networks'], sys.modules[P + 'net_utils'],
               importlib.import_module(P + 'autograd'))
    monkeypatch.setattr(FK, 'STORAGE', storage)
    return ops


def _dispatch(monkeypatch, ops, tail, pool):
    monkeypatch.setattr(ops, 'tail_mode', lambda: tail)
    monkeypatch.setattr(ops, 'pool_fused', lambda: pool)


# ----------------------------------------------------------------------------------- the stand-ins are the reference
@pytest.mark.parametrize('pool', [True, False], ids=['pool_fused', 'pool_separate'])
@pytest.mark.parametrize('tail', ['acc', 'fused', None], ids=['tail_acc', 'tail_fused', 'tail_separate'])
@pytest.mark.parametrize('degradation,scale,h,w', [('BD', 4, 17, 23), ('BI', 2, 20, 24)], ids=['bd4_17x23', 'bi2_20x24'])
def test_stand_ins_match_the_reference_step(monkeypatch, degradation, scale, h, w, tail, pool):
    ops = _install(monkeypatch, torch.float32)
    _dispatch(monkeypatch, ops, tail, pool)
    p = O.make_frnet_params(41, nb=2, scale=scale, degradation=degradation, gain=1.5)
    net = T.FRNet(3, 3, 64, 2, degradation, scale)
    net.load_state_dict(p, strict=True)
    net.eval()
    n = 2
    lr_curr, lr_prev = KC._rand(42, n, 3, h, w), KC._rand(43, n, 3, h, w)
    hr_prev = KC._rand(44, n, 3, scale * h, scale * w)
    hr = torch.empty(n, 3, scale * h, scale * w)
    u8 = torch.empty(n, scale * h, scale * w, 3, dtype=torch.uint8)
    net.step_into(lr_curr, lr_prev, hr_prev, hr, out_u8=u8)
    with torch.no_grad():
        ref = R.step(p, lr_curr, lr_prev, hr_prev, scale, degradation, nb=2)
    rel = float((hr - ref).abs().max() / ref.abs().max())
    assert rel <= 1e-5, rel
    assert torch.equal(u8, torch.from_numpy(K.float32_to_uint8(hr.numpy()).transpose(0, 2, 3, 1))), \
        'uint8 frame != float32_to_uint8 of the fp32 frame'


# ----------------------------------------------------------------------------------- the replay
# (tail, pool, n, h, w, degradation, scale): 17 rows pool to 8 (an odd map), the fused tail spans two tile rows
# (68 HR rows > 30), 9x8 gives h < 16 and a 1-row map at the bottom of FNet, 20x24 the scale-2 tail
SCENARIOS = [('acc', True, 2, 17, 23, 'BD', 4), ('fused', False, 1, 17, 23, 'BD', 4), (None, True, 1, 9, 8, 'BD', 4),
             ('fused', True, 1, 20, 24, 'BI', 2)]


def _replay(monkeypatch, perturb=None):
    ops = _install(monkeypatch, torch.float16)
    for name, fn in (perturb or {}).items():
        monkeypatch.setattr(ops, name, fn)
    rec = KC.Recorder(ops, monkeypatch, NAMES)
    reached = set()
    for i, (tail, pool, n, h, w, degradation, scale) in enumerate(SCENARIOS):
        _dispatch(monkeypatch, ops, tail, pool)
        KC.run_inference(T, ops, 'cpu', 50 + i, 2, n, 2, h, w, degradation, scale)
        reached |= KC.inference_ops(tail, pool)
    KC.run_inference_module_ops(T, ops, 'cpu', 60)
    return rec, reached


def test_replay_of_the_stand_ins_passes_and_covers_the_inference_ops(monkeypatch):
    rec, reached = _replay(monkeypatch)
    print(KC.report(rec))
    assert not rec.failures, rec.failures[:5]
    assert set(FK.INFER_FAKED) <= reached <= rec.seen, sorted(reached - rec.seen)
    assert 'maxpool2x2' in reached and 'upsample' in reached
    assert not rec.unfaked


# ----------------------------------------------------------------------------------- perturbed stand-ins
class _PoolDropsLastWindowElement(FK.PackedConv):
    """pooled epilogue on a map of odd height: the bottom-right element of every window in the last full window row
    (rows h-3, h-2; row h-1 is dropped by the floor) is left out of the maximum"""

    def __call__(self, x, y=None, residual=None, impl=None, a_mode=None, max_ctas=0, pool=False):
        if not pool or x.shape[1] % 2 == 0:
            return super().__call__(x, y, residual, impl, a_mode, max_ctas, pool)
        v = FK.to_nchw(super().__call__(x, residual=residual), self.cout)
        v[:, :, v.shape[2] - 2, 1::2] = float('-inf')
        return FK._out(FK.to_nhwc(F.max_pool2d(v, 2, 2), self.cout), y)


def _tail_drops_a_seam_tap(up, outc, x, lr_curr, lr_scale, up_mode, y=None, y_u8=None, max_ctas=0, accumulate=False):
    """HR row 29 opens the second row of tail tiles (a tile covers 30 HR rows, the first one rows -1..28): there the
    conv_out tap (0, 1), which reads row 28 of the tile above, is lost"""
    y0 = y.clone() if accumulate else None
    y = FK.fused_tail(up, outc, x, lr_curr, lr_scale, up_mode, y, y_u8, max_ctas, accumulate)
    if y.shape[2] > 29:
        w = outc.w
        outc.w = w.clone()
        outc.w[:, :, 0, 1] = 0
        alt = FK.fused_tail(up, outc, x, lr_curr, lr_scale, up_mode, y0, None, max_ctas, accumulate)
        outc.w = w
        y[:, :, 29] = alt[:, :, 29]
        if y_u8 is not None:
            FK.float_to_uint8_nhwc(y, y_u8)
    return y


def _tail_overwrites(up, outc, x, lr_curr, lr_scale, up_mode, y=None, y_u8=None, max_ctas=0, accumulate=False):
    return FK.fused_tail(up, outc, x, lr_curr, lr_scale, up_mode, y, y_u8, max_ctas, False)


def _lrflow_replicate_pad(hr_prev, lr_flow, lr_curr, scale, up_mode, out=None, cpad=64):
    h, w = lr_curr.shape[2], lr_curr.shape[3]
    f = F.pad(lr_flow, (0, w - lr_flow.shape[3], 0, h - lr_flow.shape[2]), mode='replicate')
    return FK.warp_s2d_concat_hrflow(hr_prev, scale * FK._up(f, scale, up_mode), lr_curr, scale, out=out, cpad=cpad)


def _uint8_truncates(x, y=None):
    v = torch.floor(x.to(torch.float32) * 255.0).clamp_(0, 255).to(torch.uint8).permute(0, 2, 3, 1)
    return FK._out(v.contiguous(), y)


@pytest.mark.parametrize('name,fn', [
    ('PackedConv', _PoolDropsLastWindowElement),
    ('fused_tail', _tail_drops_a_seam_tap),
    ('fused_tail', _tail_overwrites),
    ('warp_s2d_concat_lrflow', _lrflow_replicate_pad),
    ('float_to_uint8_nhwc', _uint8_truncates),
], ids=['pool_drops_last_window_element', 'tail_drops_a_seam_tap', 'tail_accumulate_overwrites',
        'lrflow_replicate_pads_the_flow', 'uint8_truncates'])
def test_replay_flags_a_wrong_inference_stand_in(monkeypatch, name, fn):
    rec, _ = _replay(monkeypatch, {name: fn})
    flagged = [f for f in rec.failures if f.startswith(name + ' ')]
    print(KC.report(rec), rec.failures[:3])
    assert flagged, f'the replay did not flag the perturbed {name}'
