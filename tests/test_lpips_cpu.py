"""CPU tests (no GPU): oracle/lpips.py against TecoGAN's two LPIPS copies (tests/golden/lpips.npz, made by
oracle/gen_lpips_golden.py from the unmodified reference code with seeded AlexNet weights), the device's remapped
conv1 / conv2 layouts and pools against the direct AlexNet in float64, and the argument checks of LPIPS and of the
metric functions that take it."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                            # noqa: E402
import synthetic                                    # noqa: E402
from oracle import lpips as O                       # noqa: E402
from oracle import gen_lpips_golden as G            # noqa: E402

M = T.metrics


@pytest.fixture(scope='module')
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, 'lpips.npz'))


@pytest.fixture(scope='module')
def seqs(golden_dir):
    g = np.load(os.path.join(golden_dir, 'official_metrics.npz'))
    return [(g['true_0'], g['pred_0']), (g['true_1'], g['pred_1'])]


@pytest.mark.parametrize('h,w', [(31, 31), (64, 96), (67, 101), (130, 77), (512, 1248)])
def test_remapped_layouts_equal_direct_alexnet(h, w):
    p = synthetic.make_lpips_params(3)
    rng = np.random.default_rng(h * w)
    n = 1 if h * w > 100000 else 2
    x = O.scaled_input(rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8))
    f, r = O.features(p, x), O.features_remapped(p, x)
    pairs = [(r['grid1'][:, :, 1:-1, 1:-1], f[0]), (r['pool1'], torch.nn.functional.max_pool2d(f[0], 3, 2)),
             (r['grid2'][:, :, 1:-1, 1:-1], f[1]), (r['pool2'], torch.nn.functional.max_pool2d(f[1], 3, 2)),
             (r['f3'], f[2]), (r['f4'], f[3]), (r['f5'], f[4])]
    for got, want in pairs:
        assert got.shape == want.shape
        assert float((got - want).abs().max()) <= 1e-12 * max(1.0, float(want.abs().max()))
    sz = M.lpips_sizes(h, w)
    assert tuple(r['grid1'].shape[2:]) == sz[0][0] and tuple(r['grid2'].shape[2:]) == sz[1][0]
    assert tuple(f[2].shape[2:]) == sz[2][0]


def test_sizes_of_the_benchmark_crop():
    # crop_8x8 of 536 x 1280 is 512 x 1248
    sz = M.lpips_sizes(512, 1248)
    assert sz[0] == ((129, 313), (1, 1, 127, 311))
    assert sz[1] == ((65, 157), (1, 1, 63, 155))
    assert sz[2][0] == (31, 77)


def test_oracle_reproduces_the_reference(gold, seqs):
    p = synthetic.make_lpips_params(int(gold['seed']))
    per = []
    for k, (t, pr) in enumerate(seqs):
        got = O.official_lpips(p, t, pr)
        np.testing.assert_allclose(got['LPIPS'], gold[f'lpips_{k}'], rtol=1e-5, atol=0)
        np.testing.assert_allclose(got['tLP100'], gold[f'tlp100_{k}'], rtol=1e-4, atol=1e-6)
        h, w = min(t.shape[1], pr.shape[1]), min(t.shape[2], pr.shape[2])
        np.testing.assert_allclose(O.lpips(p, t[:, :h, :w], pr[:, :h, :w], 'calc'), gold[f'calc_lpips_{k}'],
                                   rtol=1e-5, atol=0)
        per.append({'LPIPS': gold[f'lpips_{k}'], 'tLP100': gold[f'tlp100_{k}']})
    # the script's totals follow from its per-frame lists exactly as official_averages forms them
    tot = M.official_averages(per)
    for key in ('LPIPS', 'tLP100'):
        assert tot['FrameAvg_' + key] == gold['FrameAvg_' + key]
        assert tot['FolderAvg_' + key] == gold['FolderAvg_' + key]
        np.testing.assert_array_equal(tot['Avg_' + key], gold['Avg_' + key])


@pytest.mark.skipif(not os.path.isdir(os.environ.get('TECOGAN_REFERENCE', '/root/reference') + '/codes'),
                    reason='no reference checkout')
def test_oracle_equals_both_pnetlin_copies_live():
    """the unmodified PNetLin of both copies, in fp32, against the oracle: 1e-5 relative"""
    ref = os.environ.get('TECOGAN_REFERENCE', '/root/reference')
    p = synthetic.make_lpips_params(G.SEED)
    rng = np.random.default_rng(5)
    t = rng.integers(0, 256, (3, 40, 52, 3), dtype=np.uint8)
    q = np.clip(t.astype(int) + rng.integers(-30, 31, t.shape), 0, 255).astype(np.uint8)
    np.testing.assert_allclose(G.calc_lpips(ref, t, q), O.lpips(p, t, q, 'calc'), rtol=1e-5)
    np.testing.assert_allclose(G.official_pnetlin_lpips(ref, t, q), O.lpips(p, t, q, 'official'), rtol=1e-5)


def _lp_stub():
    lp = M.LPIPS.__new__(M.LPIPS)
    lp.device = torch.device('cuda', 0)
    return lp


def test_state_dict_checks():
    sd = synthetic.make_lpips_params(0)
    convs, heads = M._lpips_weights(sd)
    assert [tuple(c[0].shape) for c in convs] == [s for s in M._ALEX_SHAPES]
    assert [h.shape[0] for h in heads] == [64, 192, 384, 256, 256]
    # the LPIPS package's keys give the same tensors; other keys are ignored
    alt = {}
    for l, fi in enumerate(M._ALEX_CONVS):
        for s in ('weight', 'bias'):
            alt[f'net.slice{l + 1}.{fi}.{s}'] = sd[f'features.{fi}.{s}']
        alt[f'lin{l}.model.1.weight'] = sd[f'lin{l}.model.1.weight']
    alt['scaling_layer.shift'] = np.zeros(3)
    convs2, heads2 = M._lpips_weights(alt)
    for a, b in zip(convs + heads, convs2 + heads2):
        assert all(torch.equal(x, y) for x, y in zip(a, b)) if isinstance(a, tuple) else torch.equal(a, b)
    bad = dict(sd)
    del bad['features.6.bias']
    with pytest.raises(ValueError, match='features.6.bias'):
        M.LPIPS(bad)
    bad = dict(sd)
    bad['lin2.model.1.weight'] = np.zeros((1, 383, 1, 1), np.float32)
    with pytest.raises(ValueError, match='shape'):
        M.LPIPS(bad)
    bad = dict(sd)
    bad['features.3.weight'] = np.zeros((192, 64, 3, 3), np.float32)
    with pytest.raises(ValueError, match='shape'):
        M.LPIPS(bad)


def test_metric_argument_checks():
    x = np.zeros((6, 64, 64, 3), np.uint8)
    for keys in (('PSNR', 'LPIPS'), ('tLP100',), ('LPIPS',)):
        with pytest.raises(ValueError, match='lpips='):
            M.official_sequence_metrics(x, x, keys=keys)
    with pytest.raises(ValueError, match='must be a tecogan_b200.metrics.LPIPS'):
        M.sequence_metrics(x, x, lpips=object())
    with pytest.raises(ValueError, match='must be a tecogan_b200.metrics.LPIPS'):
        M.official_sequence_metrics(x, x, keys=('LPIPS',), lpips='alex')
    small = np.zeros((2, 30, 64, 3), np.uint8)
    with pytest.raises(ValueError, match='31x31'):
        M.sequence_metrics(small, small, lpips=_lp_stub())
    with pytest.raises(ValueError, match='31x31'):
        _lp_stub()(small, small)
    assert M.OFFICIAL_KEYS == ('PSNR', 'SSIM', 'tOF')
