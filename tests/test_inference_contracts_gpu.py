"""pytest -m gpu: every kernel call of the inference step (ClipEngine.run_frame -> FRNet.step_into) replayed against
its CPU contract (tests/kernel_contracts.py), each judged per element on its own inputs against a float64 reference:
the benchmark's workload itself, the other tail mode at full size, small ragged shapes under every dispatch (tail
fused / accumulating / separate launches, max-pool in the conv epilogue or separate), SRNet's convs forced to
either A-operand path, the 2x BI tail, and warp_s2d_concat_lrflow at its edges.  Each scenario prints its wall
time and the per-op (checked calls, worst |err| / bound)."""
import os
import sys
import time

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
P = 'tecogan-pytorch_b200.'


def _replay(monkeypatch, tag, run, tail='acc', pool=True, a_mode=None, expect=None):
    """run(T, ops) under the dispatch (tail, pool; a_mode forced on SRNet's convs when given) with every op recorded;
    the replay must pass, launch nothing without a stand-in and reach every op of the dispatch (or `expect`)"""
    import torch
    assert torch.cuda.is_available(), 'pytest -m gpu needs a GPU'
    import fake_ops as FK
    import kernel_contracts as KC
    import tecogan_b200 as T
    ops, networks, L = sys.modules[P + 'ops'], sys.modules[P + 'networks'], sys.modules[P + 'lib']
    monkeypatch.setattr(ops, 'tail_mode', lambda: tail)
    monkeypatch.setattr(ops, 'pool_fused', lambda: pool)
    if a_mode is not None:
        # SRNet's convs are 64 -> 64 (conv_in, residual blocks, transposed convs); FNet's 128 / 256-channel layers
        # keep their automatic choice (their weights do not fit the halo kernel's shared memory)
        forced = {'on': False}
        mode = {'halo': L.AMODE_HALO, 'tap': L.AMODE_TAP}[a_mode]
        monkeypatch.setattr(ops, 'default_a_mode', lambda: mode if forced['on'] else L.AMODE_AUTO)
        run_nhwc = networks.SRNet.run_nhwc

        def srnet_forced(self, *a, **k):
            forced['on'] = True
            try:
                return run_nhwc(self, *a, **k)
            finally:
                forced['on'] = False
        monkeypatch.setattr(networks.SRNet, 'run_nhwc', srnet_forced)
    rec = KC.Recorder(ops, monkeypatch, FK.FAKED + FK.INFER_FAKED)
    t0 = time.perf_counter()
    run(T, ops)
    torch.cuda.synchronize()
    print(f'{tag}: {time.perf_counter() - t0:.1f} s; per-op (checked calls, worst |err| / bound): {KC.report(rec)}')
    expect = KC.inference_ops(tail, pool) if expect is None else expect
    assert expect <= rec.seen, f'ops never exercised: {sorted(expect - rec.seen)}'
    assert not rec.unfaked, f'kernels launched without a CPU contract: {sorted(set(rec.unfaked))}'
    assert not rec.failures, '\n'.join(rec.failures[:20])


def test_bench_workload_kernel_calls_honour_their_contracts(monkeypatch):
    """exactly the step bench.py times: its weights and clips, 4 x BD, 4 clips of 134x320, nb = 10, default dispatch
    (tail 'acc', pooled epilogue, a_mode auto).  FNet pools 134 -> 67 -> 33 rows, runs its 128 / 256-channel
    split-K layers and reflect-pads the flow from 128 to 134 rows; frame 1 warps a real HR frame."""
    import kernel_contracts as KC
    import bench

    def run(T, ops):
        KC.run_inference(T, ops, DEV, 0, 10, 4, 2, 134, 320, 'BD', 4, params=bench.make_params(),
                         clips=bench.synthetic_clips(4, 2, seed=100))
    _replay(monkeypatch, 'bench 4xBD n=4 134x320', run)


def test_fused_tail_mode_full_size(monkeypatch):
    import kernel_contracts as KC
    _replay(monkeypatch, 'tail fused 1x134x320',
            lambda T, ops: KC.run_inference(T, ops, DEV, 70, 10, 1, 2, 134, 320, 'BD', 4), tail='fused')


@pytest.mark.parametrize('pool', [True, False], ids=['pool_fused', 'pool_separate'])
@pytest.mark.parametrize('tail', ['acc', 'fused', None], ids=['tail_acc', 'tail_fused', 'tail_separate'])
def test_small_ragged_shapes(monkeypatch, tail, pool):
    """h < 16, odd pooled sizes, single tiles and ragged last tiles"""
    import kernel_contracts as KC

    def run(T, ops):
        for i, (n, h, w) in enumerate(((1, 9, 8), (2, 17, 23), (3, 37, 45))):
            KC.run_inference(T, ops, DEV, 80 + i, 2, n, 2, h, w, 'BD', 4)
    _replay(monkeypatch, f'small tail={tail} pool={pool}', run, tail=tail, pool=pool)


@pytest.mark.parametrize('a_mode', ['halo', 'tap'])
def test_forced_a_operand_path(monkeypatch, a_mode):
    import kernel_contracts as KC
    _replay(monkeypatch, f'a_mode={a_mode} 2x17x23',
            lambda T, ops: KC.run_inference(T, ops, DEV, 90, 2, 2, 2, 17, 23, 'BD', 4), a_mode=a_mode)


@pytest.mark.parametrize('n,h,w', [(1, 20, 24), (1, 268, 640)], ids=['20x24', '268x640'])
def test_bi2_tail(monkeypatch, n, h, w):
    """scale 2: the tail is the only transposed conv, the residual is bilinear"""
    import kernel_contracts as KC
    _replay(monkeypatch, f'2xBI {n}x{h}x{w}',
            lambda T, ops: KC.run_inference(T, ops, DEV, 100, 10 if h > 100 else 2, n, 2, h, w, 'BI', 2))


def test_inference_module_ops(monkeypatch):
    import kernel_contracts as KC
    _replay(monkeypatch, 'module ops', lambda T, ops: KC.run_inference_module_ops(T, ops, DEV, 110),
            expect={'warp_s2d_concat_lrflow', 'float_to_uint8_nhwc'})
