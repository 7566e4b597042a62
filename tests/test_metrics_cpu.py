"""CPU tests (no GPU): the metric specification -- oracle/farneback.py against cv2's Farneback flows, the gray and Y
rules of oracle/metrics_oracle.py against cv2 and the reference's rgb_to_ycbcr (from the fixture, and live where
cv2 / the reference are importable), the oracle's PSNR and tOF against the reference's MetricCalculator -- and the
argument checks of tecogan_b200.metrics and the new C entry points."""
import ctypes
import os
import sys
from collections import OrderedDict

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402
import refimport                               # noqa: E402
from oracle import farneback as F              # noqa: E402
from oracle import metrics_oracle as MO        # noqa: E402

L = sys.modules['tecogan-pytorch_b200.lib']
P = ctypes.c_void_p(256)                       # a non-null, aligned pointer that is never dereferenced
INVALID, UNSUPPORTED = -1, -2
FLOW_CASES = ('small', 'odd', 'tiny', 'large', 'flat', 'deep')


@pytest.fixture(scope='module')
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, 'metrics_cv2.npz'))


def test_level_rules():
    assert F.level_count(134, 160, 0.5, 3) == 2          # 160 / 8 < 32
    assert F.level_count(259, 270, 0.5, 3) == 3
    assert F.level_count(40, 31, 0.5, 3) == 0
    assert F.level_params(67, 101, 0.5, 1)[2:] == (34, 50)   # 33.5 -> 34, 50.5 -> 50: half to even
    assert F.level_params(259, 270, 0.5, 3) == (3.5, 19, 32, 34)
    assert F.level_params(259, 270, 0.5, 1)[1] == 3          # rint(2.5) = 2, | 1 = 3
    assert list(F.gaussian_taps(3, 0.0)) == [0.25, 0.5, 0.25]


@pytest.mark.parametrize('name', FLOW_CASES)
def test_farneback_oracle_matches_cv2(gold, name):
    got = F.farneback(gold[f'{name}_prev'], gold[f'{name}_next'])[::int(gold[f'{name}_rows'])]
    d = np.abs(got - gold[f'{name}_flow'])
    assert np.median(d) <= 1e-6, np.median(d)
    assert d.max() <= 1e-2, d.max()


def test_large_flow_leaves_the_frame(gold):
    f = gold['large_flow']
    xs = np.arange(f.shape[1])[None, :] + f[..., 0]
    assert (xs < 0).any()                                    # the "outside" branch of update_matrices is exercised


def test_tof_oracle_matches_cv2(gold):
    t, p = gold['tof_true'], gold['tof_pred']
    v = MO.tof(t[0], t[1], p[0], p[1])
    assert abs(v - float(gold['tof_value'])) <= 1e-6 * float(gold['tof_value'])


def test_gray_rule(gold):
    assert np.array_equal(MO.rgb_to_gray(gold['gray_rgb']), gold['gray_cv2'])


def test_y_rule_at_the_ties(gold):
    assert len(gold['tie_rgb']) == 194
    assert np.array_equal(MO.rgb_to_y(gold['tie_rgb']), gold['tie_y'])
    for c in MO.Y_EXCEPTIONS:                                # the exceptions are among the fixture's colours
        assert any((gold['tie_rgb'] == np.uint8(c)).all(1))


def _all_colours():
    c = np.arange(1 << 24, dtype=np.int64)
    return np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)


def test_gray_rule_all_colours_live():
    cv2 = pytest.importorskip('cv2')
    rgb = _all_colours()
    assert np.array_equal(MO.rgb_to_gray(rgb), cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY))


def _reference_or_skip():
    pytest.importorskip('cv2')
    if not refimport.available():
        pytest.skip('reference not installed in oracle/_ref')
    _, _, du = refimport.import_generator()
    return du


def test_y_rule_all_colours_live():
    du = _reference_or_skip()
    rgb = _all_colours()
    assert np.array_equal(MO.rgb_to_y(rgb), du.rgb_to_ycbcr(rgb)[..., 0])


def _reference_calculator(colorspace):
    _reference_or_skip()
    import importlib
    import types
    # LPIPS (skimage, IPython, AlexNet weights) is not used by a PSNR / tOF calculator: stand in for its module
    for name in ('metrics.LPIPS', 'metrics.LPIPS.models', 'metrics.LPIPS.models.dist_model'):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules['metrics.LPIPS.models.dist_model'].__dict__.setdefault('DistModel', None)
    mc = importlib.import_module('metrics.metric_calculator')
    calc = mc.MetricCalculator.__new__(mc.MetricCalculator)   # no LPIPS: skip __init__'s DistModel
    calc.metric_opt = OrderedDict([('PSNR', {'colorspace': colorspace}), ('tOF', {'colorspace': 'rgb'})])
    calc.psnr_colorspace = colorspace
    calc.dm = None
    calc.reset()
    return calc


def seeded_sequence(T=3, h=70, w=90, hp=None, wp=None, seed=0):
    import scipy.ndimage as nd
    rng = np.random.default_rng(seed)
    base = nd.gaussian_filter(rng.uniform(0, 255, (h + 20, w + 20, 3)), (2.5, 2.5, 0))
    base = (base - base.min()) / (base.max() - base.min()) * 255
    true = np.stack([nd.shift(base, (0.8 * i, -1.3 * i, 0), order=1, mode='nearest')[10:10 + h, 10:10 + w]
                     for i in range(T)])
    true = np.clip(true, 0, 255).round().astype(np.uint8)
    hp, wp = hp or h, wp or w
    pred = np.zeros((T, hp, wp, 3), np.uint8)
    hh, ww = min(h, hp), min(w, wp)
    pred[:, :hh, :ww] = np.clip(true[:, :hh, :ww].astype(np.int64) + rng.integers(-9, 10, (T, hh, ww, 3)), 0, 255)
    return true, pred


@pytest.mark.parametrize('colorspace', ['y', 'rgb'])
def test_oracle_matches_metric_calculator(colorspace):
    calc = _reference_calculator(colorspace)
    true, pred = seeded_sequence(T=3, hp=66, wp=95)
    calc.compute_sequence_metrics('seq', true, pred)
    ref = calc.metric_dict['seq']
    got = MO.sequence_metrics(true, pred, colorspace)
    assert list(got['PSNR']) == list(ref['PSNR'])                # exact
    assert np.allclose(got['tOF'], ref['tOF'], rtol=1e-6, atol=0)


def test_python_argument_checks():
    M = T.metrics
    x = np.zeros((2, 8, 8, 3), np.uint8)
    with pytest.raises(ValueError):
        M.sequence_metrics(x, x, psnr='lab')
    with pytest.raises(ValueError):
        M.sequence_metrics(x.astype(np.float32), x)
    with pytest.raises(ValueError):
        M.sequence_metrics(x[..., :2], x)
    with pytest.raises(ValueError):
        M.sequence_metrics(x, x[:1])
    with pytest.raises(ValueError):
        M.sequence_metrics(x, x, tof=1)
    with pytest.raises(ValueError):
        M.rgb_to_gray(torch.zeros(4, 4, 3, dtype=torch.uint8))       # not on a CUDA device
    g = torch.zeros(1, 8, 8, dtype=torch.uint8)
    with pytest.raises(ValueError):
        M.farneback(g, g)                                             # not on a CUDA device
    for kw in ({'pyr_scale': 1.0}, {'pyr_scale': 0}, {'levels': -1}, {'winsize': 0}, {'winsize': 2.5},
               {'iterations': 0}, {'poly_n': 6}, {'poly_sigma': 0.0}, {'poly_sigma': float('nan')}, {'flags': 4},
               {'flags': 256}):
        with pytest.raises(ValueError):
            M._check_farneback_args(**{**dict(pyr_scale=0.5, levels=3, winsize=15, iterations=3, poly_n=5,
                                              poly_sigma=1.2, flags=0), **kw})
    for kw in ({'pyr_scale': 1.0}, {'poly_n': 6}, {'flags': 4}):
        with pytest.raises(ValueError):
            F.check_args(**{**dict(pyr_scale=0.5, levels=3, winsize=15, iterations=3, poly_n=5, poly_sigma=1.2,
                                   flags=0), **kw})


def test_c_argument_checks():
    lib = L.load()
    good = T.ops.farneback_params(0.5, 3, 15, 3, 5, 1.2, 0)
    big = 1 << 40
    assert lib.tg_farneback_workspace_bytes(2, 1, 8, 8) == 0
    assert lib.tg_farneback_workspace_bytes(2, 4, 64, 64) > 0
    assert lib.tg_farneback(None, 1, 2, 64, 64, ctypes.byref(good), P, P, big, None) == INVALID
    assert lib.tg_farneback(P, 1, 1, 64, 64, ctypes.byref(good), P, P, big, None) == INVALID
    assert lib.tg_farneback(P, 1, 2, 64, 64, ctypes.byref(good), P, P, 16, None) == INVALID   # short workspace
    assert lib.tg_farneback(P, 1, 2, 64, 64, None, P, P, big, None) == INVALID
    for field, value in (('pyr_scale', 1.0), ('poly_n', 6), ('flags', 4), ('winsize', 64), ('iterations', 0)):
        p = T.ops.farneback_params(0.5, 3, 15, 3, 5, 1.2, 0)
        setattr(p, field, value)
        assert lib.tg_farneback(P, 1, 2, 64, 64, ctypes.byref(p), P, P, big, None) == INVALID, field
    assert lib.tg_farneback(P, 1, 2, 1, 64, ctypes.byref(good), P, P, big, None) == UNSUPPORTED
    assert lib.tg_farneback(P, 1, 2, 64, 64, ctypes.byref(good), ctypes.c_void_p(260), P, big, None) == INVALID
    assert lib.tg_metrics_frames_in(None, 8, 8, P, 8, 8, 1, L.PSNR_Y, P, P, None) == INVALID
    assert lib.tg_metrics_frames_in(P, 8, 8, P, 8, 8, 1, 3, P, P, None) == INVALID
    assert lib.tg_metrics_frames_in(P, 8, 8, None, 0, 0, 1, L.PSNR_RGB, P, P, None) == INVALID
    assert lib.tg_metrics_frames_in(P, 8, 8, P, 8, 8, 1, L.PSNR_NONE, P, P, None) == INVALID   # sse without PSNR
    assert lib.tg_metrics_frames_in(P, 8, 8, P, 8, 8, 1, L.PSNR_NONE, None, None, None) == INVALID
    assert lib.tg_metrics_frames_in(P, 8, 8, P, 8, 8, 70000, L.PSNR_Y, P, P, None) == UNSUPPORTED
    assert lib.tg_flow_epe_sum(None, P, 1, 8, 8, P, None) == INVALID
    assert lib.tg_flow_epe_sum(P, P, 0, 8, 8, P, None) == INVALID
    assert lib.tg_flow_epe_sum(P, P, 70000, 8, 8, P, None) == UNSUPPORTED
