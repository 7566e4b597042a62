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
