"""CPU: pin the oracle (oracle/) against outputs of the UNMODIFIED reference.

The fixtures in tests/golden were written by oracle/gen_golden.py, which imports
the reference and runs it on seeded inputs; at the BASELINE size 3x134x320 a
seeded sample of the reference's output is stored.
"""
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import ops_oracle as K
from oracle import frnet_oracle as O

G = os.path.join(os.path.dirname(__file__), 'golden')


def rand(seed, *shape, lo=0.0, hi=1.0):
    return torch.from_numpy(np.random.default_rng(seed).uniform(lo, hi, size=shape).astype(np.float32))


def relerr(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-12)


# ------------------------------------------------------------------ functional ops
def test_ops_against_reference_outputs():
    g = np.load(os.path.join(G, 'ops.npz'))
    x = rand(20, 2, 3, 20, 24).numpy()
    flow = rand(21, 2, 2, 20, 24, lo=-4.0, hi=4.0).numpy()
    flow[0, :, 0, 0] = [-30.0, 40.0]
    w = K.backward_warp(x, flow)
    assert np.abs(w - g['warped']).max() <= 2e-6          # fp32 sampling
    w2 = K.backward_warp(x, flow, exact_reference_grid=False)
    assert np.abs(w2 - g['warped']).max() <= 2e-5         # closed form x+u: ~1e-4 px of fp32 rounding
    # pure index permutations: bit exact
    assert np.array_equal(K.space_to_depth(rand(22, 2, 3, 16, 24).numpy(), 4), g['s2d4'])
    assert np.array_equal(K.space_to_depth(rand(22, 2, 3, 16, 24).numpy(), 2), g['s2d2'])
    xs = rand(23, 1, 3, 9, 11).numpy()
    assert np.abs(K.bicubic_upsample(xs, 4) - g['bic4']).max() <= 1e-6
    assert np.abs(K.bicubic_upsample(xs, 2) - g['bic2']).max() <= 1e-6
    assert np.abs(K.bilinear_upsample(xs, 4) - g['bil4']).max() <= 1e-6
    assert np.abs(K.bilinear_upsample(xs, 2) - g['bil2']).max() <= 1e-6
    # uint8 quantisation incl. x.5 ties (round-half-even): bit exact
    assert np.array_equal(K.float32_to_uint8(g['q_in']), g['q'])
    # ConvTranspose2d(3,2,1,op=1) == 4 parity sub-convs interleaved (pixel-shuffle)
    wt = rand(25, 8, 8, 3, 3, lo=-1, hi=1).numpy()
    bt = rand(26, 8, lo=-1, hi=1).numpy()
    ct = K.conv_transpose3x3s2_parity(rand(27, 1, 8, 5, 7).numpy(), wt, bt)
    assert np.abs(ct - g['convt']).max() <= 5e-6


def test_downsample_bd_against_reference_outputs():
    """BD degradation (data_utils.py:11-53): oracle and the package's create_kernel vs the
    reference-generated fixture."""
    import tecogan_b200 as T
    g = np.load(os.path.join(G, 'downsample_bd.npz'))
    k2 = K.create_kernel(1.5)
    assert k2.shape == (9, 9)
    assert np.array_equal(g['kernel'][0, 0], k2) and np.array_equal(g['kernel'][2, 2], k2)
    assert np.array_equal(T.create_kernel(1.5).numpy(), g['kernel'])
    rng = lambda seed, *shape: np.random.default_rng(seed).uniform(0, 1, size=shape).astype(np.float32)  # noqa: E731
    for name, seed, shape, s, pad in (('s4_pad', 30, (2, 3, 36, 44), 4, True), ('s4_valid', 31, (1, 3, 41, 45), 4, False),
                                      ('s2_pad', 32, (1, 3, 27, 30), 2, True)):
        out = K.downsample_bd(rng(seed, *shape), k2, s, pad)
        assert out.shape == g[name].shape
        assert np.abs(out - g[name]).max() <= 1e-6, name


def test_bicubic_kernel_values():
    k = K.bicubic_kernels(4)
    assert np.array_equal(k[0], np.array([0, 1, 0, 0], np.float32))
    assert np.array_equal(k[1], np.array([-0.10546875, 0.87890625, 0.26171875, -0.03515625], np.float32))
    assert np.array_equal(k[2], np.array([-0.09375, 0.59375, 0.59375, -0.09375], np.float32))
    assert np.array_equal(K.bicubic_kernels(2), k[[0, 2]])


# ------------------------------------------------------------------ FRNet.step
@pytest.mark.parametrize('tag,gain', [('g1', 1.0), ('g15', 1.5), ('g2', 2.0)])
def test_step_bd4(tag, gain):
    g = np.load(os.path.join(G, f'step_bd4_18x28_{tag}.npz'))
    p = O.make_frnet_params(11, scale=4, degradation='BD', gain=gain)
    lr_curr, lr_prev, hr_prev = rand(1, 1, 3, 18, 28), rand(2, 1, 3, 18, 28), rand(3, 1, 3, 72, 112)
    taps = {}
    hr = O.frnet_step(p, lr_curr, lr_prev, hr_prev, 4, 'BD', taps=taps)
    assert taps['lr_flow'].shape == (1, 2, 16, 24)         # 8*floor(h/8)
    assert relerr(taps['lr_flow'].numpy(), g['lr_flow']) <= 2e-5
    assert relerr(hr.numpy(), g['hr_curr']) <= 2e-5


def test_step_bi2():
    g = np.load(os.path.join(G, 'step_bi2_20x24_g15.npz'))
    p = O.make_frnet_params(12, scale=2, degradation='BI', gain=1.5)
    assert 'upsample_func.kernels' not in p and 'srnet.conv_up.2.weight' not in p
    assert p['srnet.conv_in.0.weight'].shape == (64, 15, 3, 3)
    hr = O.frnet_step(p, rand(4, 1, 3, 20, 24), rand(5, 1, 3, 20, 24), rand(6, 1, 3, 40, 48), 2, 'BI')
    assert relerr(hr.numpy(), g['hr_curr']) <= 2e-5


def test_infer_sequence_uint8():
    g = np.load(os.path.join(G, 'infer_seq_bd4_16x24_g15.npz'))
    p = O.make_frnet_params(13, scale=4, degradation='BD', gain=1.5)
    seq = O.frnet_infer_sequence(p, O.make_clip(7, 4, 3, 16, 24), 4, 'BD')
    assert seq.shape == g['hr_seq'].shape and seq.dtype == np.uint8
    d = np.abs(seq.astype(np.int32) - g['hr_seq'].astype(np.int32))
    assert d.max() <= 1 and (d != 0).mean() < 1e-3       # fp32 reassociation can flip a .5 tie


def test_forward_sequence():
    g = np.load(os.path.join(G, 'fwd_seq_bd4_16x16_g15.npz'))
    p = O.make_frnet_params(14, scale=4, degradation='BD', gain=1.5)
    d = O.frnet_forward_sequence(p, rand(8, 1, 3, 3, 16, 16), 4, 'BD')
    for k in ('hr_data', 'hr_flow', 'lr_prev', 'lr_curr', 'lr_flow'):
        assert tuple(d[k].shape) == g[k].shape, k
        assert relerr(d[k].numpy(), g[k]) <= 3e-5, k


def test_sequence_gradients_against_reference():
    """Oracle of the generator BACKWARD (SURVEY 8-f1, next round): autograd through the torch port
    of forward_sequence vs gradients the reference itself produced (loss.backward() through
    FRNet.forward_sequence, oracle/gen_golden.py): loss, d/d lr_data, eight whole parameter
    gradients and the norm of all 44."""
    from oracle import frnet_torchref as R
    g = np.load(os.path.join(G, 'fwd_seq_grads_bd4_16x16_nb2_g15.npz'))
    p = O.make_frnet_params(15, nb=2, scale=4, degradation='BD', gain=1.5)
    loss, grads, gx = R.sequence_loss_and_grads(p, rand(9, 1, 3, 3, 16, 16), 4, 'BD', 16, nb=2)
    assert abs(float(loss) - float(g['loss'])) <= 1e-4 * abs(float(g['loss']))
    assert relerr(gx.numpy(), g['d_lr_data']) <= 1e-5
    names = [str(k) for k in g['names']]
    assert sorted(names) == sorted(grads)
    for k, nrm in zip(names, g['norms']):
        assert abs(float(grads[k].norm()) - nrm) <= 1e-4 * max(nrm, 1e-9), k
    for k in g.files:
        if k.startswith('g:'):
            assert relerr(grads[k[2:]].numpy(), g[k]) <= 1e-5, k


def test_state_dict_layout_matches_reference_counts():
    # SURVEY.md section 9: BD 4x = 78 entries (76 params + 2 kernels buffers); BI 4x = 76
    assert len(O.frnet_param_shapes(scale=4, degradation='BD')) == 78
    assert len(O.frnet_param_shapes(scale=4, degradation='BI')) == 76
    n = sum(int(np.prod(s)) for k, s in O.frnet_param_shapes(scale=4, degradation='BI').items())
    assert n == 2589093


# ------------------------------------------------------------------ reference at full size
def test_oracle_vs_live_reference_full_size():
    """The unmodified reference FRNet.step at the bench size (1 clip, 3x134x320 -> 536x1280, 2x weights),
    stored as a fixed, seeded sample of 65536 output values (the full frame exceeds the fixture budget)."""
    g = np.load(os.path.join(G, 'step_bd4_134x320_g2_sample.npz'))
    p = O.make_frnet_params(5, gain=2.0)
    lr_curr, lr_prev, hr_prev = rand(1, 1, 3, 134, 320), rand(2, 1, 3, 134, 320), rand(3, 1, 3, 536, 1280)
    hr = O.frnet_step(p, lr_curr, lr_prev, hr_prev, 4, 'BD').numpy().reshape(-1)
    assert relerr(hr[g['index']], g['hr_curr']) <= 5e-5


# ------------------------------------------------------------------ library-op restatement (bench CPU baseline)
def test_torchref_matches_oracle_and_golden():
    from oracle import frnet_torchref as R
    g = np.load(os.path.join(G, 'step_bd4_18x28_g2.npz'))
    p = O.make_frnet_params(11, scale=4, degradation='BD', gain=2.0)
    a, b, c = rand(1, 1, 3, 18, 28), rand(2, 1, 3, 18, 28), rand(3, 1, 3, 72, 112)
    with torch.no_grad():
        hr = R.step(p, a, b, c, 4, 'BD')
    assert relerr(hr.numpy(), g['hr_curr']) <= 2e-5
    assert relerr(hr.numpy(), O.frnet_step(p, a, b, c, 4, 'BD').numpy()) <= 2e-5
    g2 = np.load(os.path.join(G, 'step_bi2_20x24_g15.npz'))
    p2 = O.make_frnet_params(12, scale=2, degradation='BI', gain=1.5)
    with torch.no_grad():
        hr2 = R.step(p2, rand(4, 1, 3, 20, 24), rand(5, 1, 3, 20, 24), rand(6, 1, 3, 40, 48), 2, 'BI')
    assert relerr(hr2.numpy(), g2['hr_curr']) <= 2e-5


def test_fp16_precision_model_distance_to_fp32():
    """The precision model of the CUDA path (fp16 storage, fp32 accumulate) against the fp32
    reference fixtures: within the 1e-3 north-star bar for PyTorch-default (g1) and 1.5x (g15)
    weights; the chaotic 2x weights (g2) are outside it by design and are used as a stress case."""
    from oracle import frnet_fp16emu as E
    a, b, c = rand(1, 1, 3, 18, 28), rand(2, 1, 3, 18, 28), rand(3, 1, 3, 72, 112)
    dist = {}
    for tag, gain in (('g1', 1.0), ('g15', 1.5), ('g2', 2.0)):
        g = np.load(os.path.join(G, f'step_bd4_18x28_{tag}.npz'))
        p = O.make_frnet_params(11, scale=4, degradation='BD', gain=gain)
        with torch.no_grad():
            hr, _ = E.step(p, a, b, c, 4, 'BD')
        dist[tag] = float(np.linalg.norm(hr.numpy() - g['hr_curr']) / np.linalg.norm(g['hr_curr']))
    assert dist['g1'] <= 1e-4 and dist['g15'] <= 1e-3, dist
    assert 1e-3 < dist['g2'] < 1e-2, dist
