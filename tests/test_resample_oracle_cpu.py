"""CPU tests (no GPU): oracle/resample.py, the specification of the streamed output's resize, against Pillow (live
and the tests/golden/resample_pil.npz fixture) and torch's antialiased bicubic; the library's host-side tables
(tg_resample_table) against the oracle's float32 table, bit for bit."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402,F401  (registers the package modules)
from oracle import resample as R              # noqa: E402

ops = sys.modules['tecogan-pytorch_b200.ops']
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'resample_pil.npz')
PIL_TOL = 2.5e-7            # Pillow rounds the intermediate and the result to float32
SIZES = [((67, 160), (90, 213)), ((67, 160), (50, 120)), ((67, 160), (17, 40)), ((67, 160), (134, 320)),
         ((48, 90), (54, 120)), ((48, 90), (36, 45)), ((20, 9), (5, 18))]


def _x(H, W, seed=0):
    return np.random.default_rng(seed + H * W).uniform(-0.1, 1.1, size=(H, W)).astype(np.float32)


@pytest.mark.parametrize('filt', R.FILTERS)
@pytest.mark.parametrize('src,dst', SIZES)
def test_oracle_matches_pil(filt, src, dst):
    Image = pytest.importorskip('PIL.Image')
    x = _x(*src)
    pil = {'bicubic': Image.BICUBIC, 'lanczos': Image.LANCZOS}[filt]
    want = np.asarray(Image.fromarray(x, 'F').resize(dst[::-1], pil, reducing_gap=None), dtype=np.float64)
    got = R.resize(x, dst, filt)
    assert np.abs(got - want).max() <= PIL_TOL


def test_oracle_matches_pil_golden():
    g = np.load(GOLDEN)
    cases = 0
    for key in g.files:
        parts = key.split('_')
        if parts[0] not in R.FILTERS:
            continue
        (H, W), (Ho, Wo) = (tuple(int(v) for v in p.split('x')) for p in parts[1:])
        got = R.resize(g[f'x_{H}x{W}'], (Ho, Wo), parts[0])
        assert got.shape == g[key].shape
        assert np.abs(got - g[key]).max() <= PIL_TOL, key
        cases += 1
    assert cases == 12


@pytest.mark.parametrize('src,dst', SIZES[:6])
def test_bicubic_is_close_to_torch_antialias(src, dst):
    x = _x(*src, seed=5)
    want = torch.nn.functional.interpolate(torch.from_numpy(x).double()[None, None], size=dst, mode='bicubic',
                                           antialias=True, align_corners=False)[0, 0].numpy()
    assert np.abs(R.resize(x, dst, 'bicubic') - want).max() <= 2e-5


@pytest.mark.parametrize('filt', R.FILTERS)
@pytest.mark.parametrize('n_in,n_out', [(536, 134), (536, 402), (536, 536), (402, 536), (536, 1072), (1280, 1707),
                                        (7, 2), (3, 6), (1, 2), (13, 4)])
def test_table_rows_sum_to_one(filt, n_in, n_out):
    first, w = R.table(n_in, n_out, filt)
    assert np.abs(w.sum(axis=1) - 1.0).max() <= 1e-12
    k = R.taps(n_in, n_out, filt)
    assert w.shape == (n_out, k) and k <= R.MAX_TAPS
    assert (first >= 0).all() and (first + k <= max(n_in, k)).all()    # the window ends inside the axis where it fits


@pytest.mark.parametrize('filt', R.FILTERS)
def test_scale_one_is_the_identity(filt):
    x = _x(37, 53, seed=9).astype(np.float64)
    assert np.abs(R.resize(x, (37, 53), filt) - x).max() <= 1e-15
    first, w = R.table(53, 53, filt)
    centre = np.arange(53) - first
    assert np.array_equal(w[np.arange(53), centre], np.ones(53))
    w[np.arange(53), centre] = 0
    assert np.abs(w).max() <= 1e-16


@pytest.mark.parametrize('filt', R.FILTERS)
@pytest.mark.parametrize('n_in,n_out', [(536, 134), (536, 402), (536, 536), (402, 536), (536, 1072),     # 1/4 .. 2
                                        (1280, 320), (1280, 960), (1280, 1707), (1280, 2560), (720, 810),
                                        (8, 2), (5, 2), (3, 6), (1, 2), (2, 1), (13, 4)])             # < taps
def test_library_table_is_the_oracle(filt, n_in, n_out):
    first, w = ops.resample_table(n_in, n_out, filt)
    rf, rw = R.table_f32(n_in, n_out, filt)
    assert first.dtype == torch.int32 and w.dtype == torch.float32
    assert np.array_equal(first.numpy(), rf)
    assert np.array_equal(w.numpy().view(np.uint32), rw.view(np.uint32))


def test_ratio_bounds_and_tap_counts():
    assert R.taps(536, 134, 'bicubic') == 17 and R.taps(536, 134, 'lanczos') == 25
    assert R.taps(536, 1072, 'bicubic') == 5 and R.taps(536, 1072, 'lanczos') == 7
    for n_in, n_out, ok in ((536, 134, True), (536, 133, False), (536, 1072, True), (536, 1073, False)):
        assert R.check_ratio(n_in, n_out) == ok == ops.resample_ratio_ok(n_in, n_out)
    with pytest.raises(ValueError):
        R.resize(np.zeros((8, 8)), (1, 8))
