"""pytest -m gpu: every op call of real training steps replayed against its CPU contract
(tests/kernel_contracts.py): the kernels at the arguments the training path passes -- the real layer widths
(6->32, the 2-channel flow head, 51->64, the 128 / 256-channel split-K layers), n*t batched wgrad, mul = s in
upsample_bwd, gflow2 in flow_head_bwd, d_hr_prev accumulated across frames, the loss scale -- each judged per
element on its own inputs against a float64 reference."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu


def test_training_step_kernel_calls_honour_their_contracts(monkeypatch):
    import torch
    assert torch.cuda.is_available(), 'pytest -m gpu needs a GPU'
    import kernel_contracts as KC
    import fake_ops as FK
    import tecogan_b200 as T
    ops = sys.modules['tecogan-pytorch_b200.ops']
    rec = KC.Recorder(ops, monkeypatch)
    KC.scenarios(T, ops, 'cuda:0')
    torch.cuda.synchronize()
    print('per-op (checked calls, worst |err| / bound):', KC.report(rec))
    print('exercised:', sorted(rec.seen))
    assert set(FK.FAKED) <= rec.seen, f'ops never exercised: {sorted(set(FK.FAKED) - rec.seen)}'
    assert not rec.unfaked, f'kernels launched without a CPU contract: {sorted(set(rec.unfaked))}'
    assert not rec.failures, '\n'.join(rec.failures[:20])


def test_single_and_two_channel_training_step_kernel_calls_honour_their_contracts(monkeypatch):
    """FRNet(1, 1) at 4x BD and FRNet(2, 2) at 2x BI: pack_pair and FNet's first conv at 2 / 4 real channels, the
    warp and its backward at C = 1 / 2 (the CTA-lock-step kernel, not the RGB one), conv_in at 17 / 10 real
    channels (one real channel in the last 16-channel k-step at 17) and conv_out, its dgrad and its wgrad at
    1 / 2 output channels"""
    import torch
    assert torch.cuda.is_available(), 'pytest -m gpu needs a GPU'
    import kernel_contracts as KC
    import fake_ops as FK
    import tecogan_b200 as T
    ops = sys.modules['tecogan-pytorch_b200.ops']
    rec = KC.Recorder(ops, monkeypatch)
    KC.run_sequence(T, 'cuda:0', 35, nb=2, n=2, t=4, h=32, w=32, nc=1)
    KC.run_sequence(T, 'cuda:0', 36, nb=1, n=1, t=3, h=16, w=24, degradation='BI', scale=2, nc=2)
    torch.cuda.synchronize()
    print('per-op (checked calls, worst |err| / bound):', KC.report(rec))
    # the ops only run_module_ops reaches: the bare backward_warp, space_to_depth and bias_grad
    expect = set(FK.FAKED) - {'backward_warp', 'backward_warp_bwd', 'space_to_depth', 'depth_to_space', 'bias_grad'}
    assert expect <= rec.seen, f'ops never exercised: {sorted(expect - rec.seen)}'
    assert not rec.unfaked, f'kernels launched without a CPU contract: {sorted(set(rec.unfaked))}'
    assert not rec.failures, '\n'.join(rec.failures[:20])
