"""CPU tests (no GPU): oracle/official_metrics.py against TecoGAN's official metric script (live through the
fixture generator's stand-ins where a reference checkout exists, else against tests/golden/official_metrics.npz),
its SSIM against a direct 7x7 window sum, and the argument checks of official_sequence_metrics / official_averages
and of the new C entry points."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                            # noqa: E402
from oracle import official_metrics as OM           # noqa: E402
from oracle import gen_official_metrics_golden as G  # noqa: E402

L = sys.modules['tecogan-pytorch_b200.lib']
P = ctypes.c_void_p(256)
INVALID, UNSUPPORTED = -1, -2
KEYS = ('PSNR', 'SSIM', 'tOF')


@pytest.fixture(scope='module')
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, 'official_metrics.npz'))


def _folders(gold):
    return [(gold[f'true_{k}'], gold[f'pred_{k}']) for k in range(len(G.FOLDERS))]


def _check_against(gold, expect):
    per = []
    for k, (t, p) in enumerate(_folders(gold)):
        got = OM.sequence_metrics(t, p)
        per.append(got)
        np.testing.assert_allclose(got['PSNR'], expect[f'psnr_{k}'], rtol=1e-12, atol=0)
        np.testing.assert_allclose(got['SSIM'], expect[f'ssim_{k}'], rtol=1e-12, atol=0)
        np.testing.assert_allclose(got['tOF'], expect[f'tof_{k}'], rtol=1e-6, atol=0)
    tot = OM.averages(per)
    for key in KEYS:
        for name in ('FrameAvg_', 'FolderAvg_', 'Avg_'):
            got, want = tot[name + key], expect[name + key]
            assert np.asarray(got).dtype == np.float32 and np.array_equal(got, want), (name, key, got, want)


def test_oracle_matches_fixture(gold):
    _check_against(gold, gold)
    assert len(gold['psnr_0']) == G.FOLDERS[0][0] - 4 and len(gold['tof_0']) == G.FOLDERS[0][0] - 5


def test_oracle_matches_live_script(gold, tmp_path):
    from oracle import vendor_reference
    script = G.script_path(vendor_reference.SRC)
    if not os.path.isfile(script):
        pytest.skip('no reference checkout: the fixture test covers the script')
    pytest.importorskip('pandas')
    pytest.importorskip('absl')
    live = {}
    outs, tars = [], []
    for k in range(len(G.FOLDERS)):
        _, _, (tar_dir, out_dir) = G.write_folders(str(tmp_path), k)
        res = G.run_script(script, str(tmp_path), [out_dir], [tar_dir], f'folder{k}')
        for key in KEYS:
            live[f'{key.lower()}_{k}'] = np.asarray(res['list'][key], np.float64)
        outs.append(out_dir)
        tars.append(tar_dir)
    live.update(G.run_script(script, str(tmp_path), outs, tars, 'all')['totals'])
    _check_against(gold, live)
    for k in range(len(G.FOLDERS)):
        np.testing.assert_array_equal(gold[f'true_{k}'], G.folder_frames(k)[0])


def test_crop_8x8_matches_script(gold):
    for n, ln, off in zip(gold['crop_n'], gold['crop_len'], gold['crop_off']):
        o, s = OM.crop_8x8(int(n))
        assert len(np.arange(int(n))[o:o + s]) == ln and o == off, n
        if n >= 48:
            assert T.metrics.crop_8x8(int(n)) == (o, s)
    assert OM.crop_8x8(536) == (12, 512) and OM.crop_8x8(1280) == (16, 1248)
    assert OM.crop_8x8(1080) == (12, 1056) and OM.crop_8x8(1920) == (16, 1888)
    assert OM.crop_8x8(47)[1] <= 0 and OM.crop_8x8(48) == (8, 32)


def test_to_uint8_is_identity_on_uint8():
    x = np.arange(256, dtype=np.uint8)
    assert np.array_equal(OM.to_uint8(x, 0, 255), x.astype(np.float32))


def test_y_matches_rgb2ycbcr_row():
    rng = np.random.default_rng(0)
    rgb = rng.integers(0, 256, (64, 64, 3)).astype(np.uint8)
    Tm = np.array([0.256788235294118, 0.504129411764706, 0.097905882352941])
    ref = np.dot(rgb.reshape(-1, 3).astype(np.float32), Tm[:, None])[:, 0] + 16
    np.testing.assert_allclose(OM.rgb_to_y(rgb).ravel(), ref, rtol=1e-15, atol=0)


@pytest.mark.parametrize('shape', [(40, 52), (7, 7), (33, 80)])
def test_ssim_equals_direct_window_sum(shape):
    rng = np.random.default_rng(shape[0])
    x = rng.uniform(16, 235, shape)
    y = np.clip(x + rng.normal(0, 8, shape), 16, 235)
    r = y.max() - y.min()
    assert abs(OM.ssim(x, y, r) - OM.ssim_direct(x, y, r)) <= 1e-12


def test_ssim_of_equal_frames_is_one():
    x = OM.rgb_to_y(np.random.default_rng(1).integers(0, 256, (50, 60, 3)).astype(np.uint8))
    assert OM.ssim(x, x, x.max() - x.min()) == 1.0


def test_ssim_of_flat_prediction_is_nan():
    flat = np.zeros((50, 60, 3), np.uint8)
    true = flat.copy()
    true[30:, 30:] = np.random.default_rng(2).integers(0, 256, (20, 30, 3))
    assert np.isnan(OM.ssim_y(true, flat))
    assert np.isnan(OM.ssim_y(flat, flat))


def test_python_argument_checks():
    M = T.metrics
    x = np.zeros((5, 64, 64, 3), np.uint8)
    with pytest.raises(ValueError):
        M.official_sequence_metrics(x, x, keys=('PSNR', 'LPIPS'))
    with pytest.raises(ValueError):
        M.official_sequence_metrics(x, x, keys='PSNR')
    with pytest.raises(ValueError):
        M.official_sequence_metrics(x, x, cutfr=-1)
    with pytest.raises(ValueError):
        M.official_sequence_metrics(x, x, cutfr=1.5)
    with pytest.raises(ValueError):
        M.official_sequence_metrics(x[:, :47], x)                 # common height 47: an empty crop
    with pytest.raises(ValueError):
        M.official_sequence_metrics(x, x[:, :, :40])
    with pytest.raises(ValueError):
        M.official_sequence_metrics(x, x[:4])
    with pytest.raises(ValueError):
        M.official_sequence_metrics(x.astype(np.float32), x)
    with pytest.raises(ValueError):
        M.official_averages([])
    with pytest.raises(ValueError):
        M.official_averages([{'PSNR': np.ones(2)}, {'SSIM': np.ones(2)}])


def test_too_few_frames_give_empty_arrays():
    x = np.zeros((4, 64, 64, 3), np.uint8)
    out = T.metrics.official_sequence_metrics(x, x)               # no device work: T - 2 cutfr == 0
    assert list(out) == list(KEYS) and all(v.shape == (0,) for v in out.values())


def test_official_averages_match_oracle(gold):
    per = [{'PSNR': gold[f'psnr_{k}'], 'SSIM': gold[f'ssim_{k}'], 'tOF': gold[f'tof_{k}']} for k in range(2)]
    got, want = T.metrics.official_averages(per), OM.averages(per)
    assert list(got) == list(want)
    for k in want:
        assert np.array_equal(got[k], want[k]) and np.asarray(got[k]).dtype == np.float32, k
        assert np.array_equal(got[k], gold[k]), k


def test_c_argument_checks():
    lib = L.load()
    big = 1 << 40
    a8 = ctypes.c_void_p(260)                                     # 4 mod 8: misaligned
    st, ss = lib.tg_official_frames_stats, lib.tg_ssim_y
    assert lib.tg_official_frames_stats_workspace_bytes(0, 32, 32) == 0
    assert lib.tg_official_frames_stats_workspace_bytes(2, 32, 32) > 0
    assert lib.tg_ssim_y_workspace_bytes(2, 6, 32) == 0
    assert lib.tg_ssim_y_workspace_bytes(2, 32, 32) > 0
    ok = (P, 64, 64, P, 64, 64, 2, 8, 8, 32, 32)
    assert st(None, *ok[1:], P, P, big, None) == INVALID
    assert st(*ok[:3], None, *ok[4:], P, P, big, None) == INVALID
    assert st(*ok, None, P, big, None) == INVALID
    assert st(*ok, P, None, big, None) == INVALID
    assert st(*ok, a8, P, big, None) == INVALID
    assert st(*ok, P, a8, big, None) == INVALID
    assert st(*ok, P, P, 8, None) == INVALID                      # short workspace
    assert st(P, 64, 64, P, 64, 40, 2, 8, 8, 32, 33, P, P, big, None) == INVALID   # past the common width
    assert st(P, 64, 64, P, 64, 64, 2, -1, 8, 32, 32, P, P, big, None) == INVALID
    assert st(P, 64, 64, P, 64, 64, 2, 8, 8, 0, 32, P, P, big, None) == INVALID
    assert st(P, 64, 64, P, 64, 64, 0, 8, 8, 32, 32, P, P, big, None) == INVALID
    assert st(P, 64, 64, P, 64, 64, 70000, 8, 8, 32, 32, P, P, big, None) == UNSUPPORTED
    assert ss(None, *ok[1:], P, P, P, big, None) == INVALID
    assert ss(*ok, None, P, P, big, None) == INVALID
    assert ss(*ok, P, None, P, big, None) == INVALID
    assert ss(*ok, P, P, None, big, None) == INVALID
    assert ss(*ok, a8, P, P, big, None) == INVALID
    assert ss(*ok, P, P, a8, big, None) == INVALID
    assert ss(*ok, P, P, P, 8, None) == INVALID
    assert ss(P, 64, 64, P, 64, 64, 2, 8, 8, 6, 32, P, P, P, big, None) == INVALID  # below the 7x7 window
    assert ss(P, 64, 64, P, 40, 64, 2, 8, 8, 33, 32, P, P, P, big, None) == INVALID
    assert ss(P, 64, 64, P, 64, 64, 70000, 8, 8, 32, 32, P, P, P, big, None) == UNSUPPORTED
    ew = lib.tg_flow_epe_sum_window
    assert ew(None, P, 1, 8, 8, 0, 0, 8, 8, P, P, 1 << 40, None) == INVALID
    assert ew(P, P, 0, 8, 8, 0, 0, 8, 8, P, P, 1 << 40, None) == INVALID
    assert ew(P, P, 1, 8, 8, 1, 0, 8, 8, P, P, 1 << 40, None) == INVALID
    assert ew(P, P, 1, 8, 8, 0, 0, 8, 0, P, P, 1 << 40, None) == INVALID
    assert ew(P, P, 1, 8, 8, 0, 0, 8, 8, a8, P, 1 << 40, None) == INVALID
    assert ew(P, P, 70000, 8, 8, 0, 0, 8, 8, P, P, 1 << 40, None) == UNSUPPORTED
    assert ew(P, P, 1, 8, 8, 0, 0, 8, 8, P, None, 1 << 40, None) == INVALID          # no workspace
    assert ew(P, P, 1, 8, 8, 0, 0, 8, 8, P, P, 8, None) == INVALID                   # short workspace
    assert ew(P, P, 1, 8, 8, 0, 0, 8, 8, P, a8, 1 << 40, None) == INVALID
    assert lib.tg_flow_epe_sum_window_workspace_bytes(3, 600) == 3 * 512 * 8
