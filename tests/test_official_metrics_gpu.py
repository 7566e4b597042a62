"""GPU tests of tecogan_b200.metrics.official_sequence_metrics / official_averages and their kernels
(tg_official_frames_stats, tg_ssim_y, tg_flow_epe_sum_window) against the official metric script's fixture
(tests/golden/official_metrics.npz) and its restatement, oracle/official_metrics.py."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402
import synthetic                               # noqa: E402
from oracle import official_metrics as OM      # noqa: E402

pytestmark = pytest.mark.gpu
L = sys.modules['tecogan-pytorch_b200.lib']
M, ops = T.metrics, T.ops
DEV = torch.device('cuda:0')
TOF_REL, TOF_ABS = 1e-4, 2e-5      # the Farneback bounds of tests/test_metrics_gpu.py
SSIM_ABS = 1e-10
KEYS = ('PSNR', 'SSIM', 'tOF')


@pytest.fixture(scope='module')
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, 'official_metrics.npz'))


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _vp(t, offset=0):
    return ctypes.c_void_p(t.data_ptr() + offset)


def _check(got, ref):
    assert list(got) == list(ref)
    np.testing.assert_allclose(got['PSNR'], ref['PSNR'], rtol=1e-12, atol=0)
    assert np.abs(got['SSIM'] - ref['SSIM']).max(initial=0) <= SSIM_ABS, (got['SSIM'], ref['SSIM'])
    d = np.abs(got['tOF'] - ref['tOF'])
    assert (d <= np.maximum(TOF_REL * np.abs(ref['tOF']), TOF_ABS)).all(), (got['tOF'], ref['tOF'])


def _seq(T_, ht, wt, hp=None, wp=None, seed=0, noise=8):
    import scipy.ndimage as nd
    rng = np.random.default_rng(seed)
    hp, wp = hp or ht, wp or wt
    h, w = max(ht, hp), max(wt, wp)
    base = nd.gaussian_filter(rng.uniform(0, 255, (h + 20, w + 20, 3)), (2.0, 2.0, 0))
    base = (base - base.min()) / (base.max() - base.min()) * 255
    full = np.clip(np.stack([nd.shift(base, (0.7 * i, -1.1 * i, 0), order=1, mode='nearest')[10:10 + h, 10:10 + w]
                             for i in range(T_)]), 0, 255).round()
    true = full[:, :ht, :wt].astype(np.uint8)
    pred = np.clip(full[:, :hp, :wp] + rng.integers(-noise, noise + 1, (T_, hp, wp, 3)), 0, 255).astype(np.uint8)
    return true, pred


def test_fixture_matches_script(gold):
    per = []
    for k in range(2):
        got = M.official_sequence_metrics(gold[f'true_{k}'], gold[f'pred_{k}'])
        _check(got, {'PSNR': gold[f'psnr_{k}'], 'SSIM': gold[f'ssim_{k}'], 'tOF': gold[f'tof_{k}']})
        per.append(got)
    tot = M.official_averages(per)
    for key in KEYS:
        for name in ('FrameAvg_', 'FolderAvg_', 'Avg_'):
            want = gold[name + key]
            if key == 'tOF':
                np.testing.assert_allclose(tot[name + key], want, rtol=TOF_REL)
            else:
                assert np.array_equal(tot[name + key], want), (name, key, tot[name + key], want)


def test_cuda_input_and_keys(gold):
    t, p = torch.from_numpy(gold['true_0']).to(DEV), torch.from_numpy(gold['pred_0']).to(DEV)
    ref = M.official_sequence_metrics(gold['true_0'], gold['pred_0'])
    got = M.official_sequence_metrics(t, p)
    for k in KEYS:
        assert np.array_equal(got[k], ref[k]), k
    only = M.official_sequence_metrics(t, p, keys=('tOF', 'SSIM'))
    assert list(only) == ['SSIM', 'tOF']
    assert np.array_equal(only['SSIM'], ref['SSIM']) and np.array_equal(only['tOF'], ref['tOF'])
    c0 = M.official_sequence_metrics(t, p, cutfr=0)
    assert c0['PSNR'].shape == (8,) and c0['tOF'].shape == (7,)
    assert np.array_equal(c0['PSNR'][2:-2], ref['PSNR'])
    short = M.official_sequence_metrics(t[:5], p[:5])
    assert short['PSNR'].shape == (1,) and short['tOF'].shape == (0,)


def test_equal_and_flat_frames():
    true, _ = _seq(5, 64, 80)
    got = M.official_sequence_metrics(true, true)
    assert np.isinf(got['PSNR']).all() and (got['SSIM'] == 1.0).all() and (got['tOF'] == 0).all()
    flat = np.zeros_like(true)
    part = flat.copy()
    part[:, 30:, 40:] = true[:, 30:, 40:]
    for t in (flat, part):                    # a black prediction: R = 0, and flat 7x7 windows in both frames
        got = M.official_sequence_metrics(t, flat, keys=('SSIM',))
        ref = OM.sequence_metrics(t, flat, keys=('SSIM',))
        assert np.isnan(ref['SSIM']).all() and np.isnan(got['SSIM']).all()


@pytest.mark.parametrize('sizes', [(49, 48, 49, 48), (67, 101, 70, 99), (131, 97, 128, 100), (100, 200, 100, 200)])
def test_sizes_against_oracle(sizes):
    ht, wt, hp, wp = sizes
    true, pred = _seq(6, ht, wt, hp, wp, seed=ht)
    _check(M.official_sequence_metrics(true, pred), OM.sequence_metrics(true, pred))


def _window_reference(true, pred, win):
    y0, x0, hc, wc = win
    h, w = min(true.shape[1], pred.shape[1]), min(true.shape[2], pred.shape[2])
    yt = OM.rgb_to_y(true[:, :h, :w][:, y0:y0 + hc, x0:x0 + wc])
    yp = OM.rgb_to_y(pred[:, :h, :w][:, y0:y0 + hc, x0:x0 + wc])
    sse = ((yt - yp) ** 2).sum(axis=(1, 2))
    mn, mx = yp.min(axis=(1, 2)), yp.max(axis=(1, 2))
    ssim = np.array([OM.ssim(a, b, b.max() - b.min()) for a, b in zip(yt, yp)])
    return sse, mn, mx, ssim


@pytest.mark.parametrize('win', [(0, 0, 7, 7), (0, 0, 60, 75), (1, 3, 40, 33), (12, 8, 32, 64), (22, 11, 38, 64),
                                 (53, 68, 7, 7), (5, 0, 55, 75)])
def test_windows_against_oracle(win):
    true, pred = _seq(3, 60, 80, 64, 75, seed=7)
    t, p = torch.from_numpy(true).to(DEV), torch.from_numpy(pred).to(DEV)
    stats = ops.official_frames_stats(t, p, win)
    ssim = ops.ssim_y(t, p, win, stats).cpu().numpy()
    stats = stats.cpu().numpy()
    sse, mn, mx, ref = _window_reference(true, pred, win)
    np.testing.assert_allclose(stats[:, 0], sse, rtol=1e-12)
    assert np.array_equal(stats[:, 1], mn) and np.array_equal(stats[:, 2], mx)
    assert np.abs(ssim - ref).max() <= SSIM_ABS
    fa, fb = torch.randn(3, 60, 75, 2, device=DEV), torch.randn(3, 60, 75, 2, device=DEV)
    y0, x0, hc, wc = win
    if y0 + hc <= 60 and x0 + wc <= 75:
        e = ops.flow_epe_sum(fa, fb, win)
        ref_e = (fa - fb)[:, y0:y0 + hc, x0:x0 + wc].double().norm(dim=-1).sum(dim=(1, 2))
        assert torch.allclose(e, ref_e, rtol=1e-6)


def test_chunks_and_reruns_are_bit_identical():
    true, pred = _seq(9, 70, 90, 66, 95, seed=3)
    full = M.official_sequence_metrics(true, pred)
    again = M.official_sequence_metrics(true, pred)
    h, w = 66, 90
    hc, wc = M.crop_8x8(h)[1], M.crop_8x8(w)[1]

    def bound(n, tof):     # the device bytes of a chunk of n frames, as official_sequence_metrics counts them
        b = n * 3 * (70 * 90 + 66 * 95) + n * 24 + ops.official_frames_stats_workspace_bytes(n, hc, wc) + n * 8
        b += ops.ssim_y_workspace_bytes(n, hc, wc)
        if tof:
            b += ops.farneback_workspace_bytes(2, n, h, w) + 2 * n * h * w + 2 * (n - 1) * h * w * 8
            b += (n - 1) * 8 + L.load().tg_flow_epe_sum_window_workspace_bytes(n - 1, hc)
        return b
    for n in (2, 3, 4):
        ch = M.official_sequence_metrics(true, pred, max_workspace_bytes=bound(n, True))
        for k in KEYS:
            assert np.array_equal(ch[k], full[k]), (n, k)
    # without tOF the chunks do not overlap: every scored frame is kept exactly once
    for n in (1, 2, 4):
        for keys in (('PSNR', 'SSIM'), ('SSIM',), ('PSNR',)):
            ch = M.official_sequence_metrics(true, pred, keys=keys, max_workspace_bytes=bound(n, False))
            for k in keys:
                assert ch[k].shape == (5,) and np.array_equal(ch[k], full[k]), (n, keys, k)
    for k in KEYS:
        assert np.array_equal(again[k], full[k]), k
    with pytest.raises(ValueError):
        M.official_sequence_metrics(true, pred, max_workspace_bytes=1000)


def test_guard_bands():
    lib = L.load()
    true, pred = _seq(3, 61, 83, 64, 80, seed=11)
    t, p = torch.from_numpy(true).to(DEV), torch.from_numpy(pred).to(DEV)
    win = (6, 8, 48, 64)
    g = 4096

    def guarded(nbytes):
        return torch.full((nbytes + 2 * g,), 0xAB, dtype=torch.uint8, device=DEV)

    def intact(buf):
        return bool((buf[:g] == 0xAB).all()) and bool((buf[-g:] == 0xAB).all())
    sw = ops.official_frames_stats_workspace_bytes(3, 48, 64)
    cw = ops.ssim_y_workspace_bytes(3, 48, 64)
    sb, swb, cb, cwb = guarded(3 * 24), guarded(sw), guarded(3 * 8), guarded(cw)
    args = (_vp(t), 61, 83, _vp(p), 64, 80, 3) + win
    L.check(lib.tg_official_frames_stats(*args, _vp(sb, g), _vp(swb, g), sw, _stream()), 'stats')
    L.check(lib.tg_ssim_y(*args, _vp(sb, g), _vp(cb, g), _vp(cwb, g), cw, _stream()), 'ssim')
    fa, fb = torch.randn(2, 61, 80, 2, device=DEV), torch.randn(2, 61, 80, 2, device=DEV)
    eb = guarded(2 * 8)
    ew = lib.tg_flow_epe_sum_window_workspace_bytes(2, 48)
    ewb = guarded(ew)
    L.check(lib.tg_flow_epe_sum_window(_vp(fa), _vp(fb), 2, 61, 80, *win, _vp(eb, g), _vp(ewb, g), ew, _stream()),
            'epe')
    torch.cuda.synchronize()
    for buf in (sb, swb, cb, cwb, eb, ewb):
        assert intact(buf)
    stats = ops.official_frames_stats(t, p, win)
    assert torch.equal(sb[g:-g].view(torch.float64).view(3, 3), stats)
    assert torch.equal(cb[g:-g].view(torch.float64), ops.ssim_y(t, p, win, stats))
    assert torch.equal(eb[g:-g].view(torch.float64), ops.flow_epe_sum(fa, fb, win))


def test_abi_refusals():
    lib = L.load()
    t = torch.zeros(2, 64, 64, 3, dtype=torch.uint8, device=DEV)
    st = torch.zeros(2, 3, dtype=torch.float64, device=DEV)
    big = 1 << 30
    w = torch.zeros(big // 8 // 1024, dtype=torch.float64, device=DEV)
    ok = (_vp(t), 64, 64, _vp(t), 64, 64, 2)
    for win, code in (((8, 8, 48, 48), 0), ((17, 8, 48, 48), -1), ((8, 8, 48, 57), -1), ((-1, 0, 8, 8), -1)):
        assert lib.tg_official_frames_stats(*ok, *win, _vp(st), _vp(w), w.numel() * 8, _stream()) == code, win
        out = torch.zeros(2, dtype=torch.float64, device=DEV)
        assert lib.tg_ssim_y(*ok, *win, _vp(st), _vp(out), _vp(w), w.numel() * 8, _stream()) == code, win
    out = torch.zeros(2, dtype=torch.float64, device=DEV)
    assert lib.tg_ssim_y(*ok, 0, 0, 6, 64, _vp(st), _vp(out), _vp(w), w.numel() * 8, _stream()) == -1
    assert lib.tg_official_frames_stats(*ok, 8, 8, 48, 48, _vp(st), _vp(w), 8, _stream()) == -1
    assert lib.tg_ssim_y(*ok, 8, 8, 48, 48, _vp(st), _vp(out), _vp(w), 8, _stream()) == -1
    assert lib.tg_official_frames_stats(*ok, 8, 8, 48, 48, _vp(st, 4), _vp(w), big, _stream()) == -1
    torch.cuda.synchronize()
    with pytest.raises(L.TecoganB200Error):
        ops.official_frames_stats(t, t, (8, 8, 60, 48))
    with pytest.raises(L.TecoganB200Error):
        ops.ssim_y(t, t[:1], (8, 8, 48, 48), st)
    with pytest.raises(L.TecoganB200Error):
        ops.flow_epe_sum(torch.zeros(1, 8, 8, 2, device=DEV), torch.zeros(1, 8, 8, 2, device=DEV), (0, 0, 9, 8))


def test_bd4_hr_sequence():
    """536x1280, T = 32: every scored frame of PSNR and SSIM against the oracle, tOF at three pairs (cv2 is slow)"""
    clip = synthetic.make_clip(3, 32, 3, 536, 1280, shift=2)
    true = (clip.permute(0, 2, 3, 1) * 255).round().to(torch.uint8).numpy()
    rng = np.random.default_rng(4)
    pred = np.clip(true.astype(np.int16) + rng.integers(-6, 7, true.shape), 0, 255).astype(np.uint8)
    got = M.official_sequence_metrics(torch.from_numpy(true).to(DEV), torch.from_numpy(pred).to(DEV))
    assert got['PSNR'].shape == (28,) and got['SSIM'].shape == (28,) and got['tOF'].shape == (27,)
    ref = OM.sequence_metrics(true, pred, keys=('PSNR', 'SSIM'))
    np.testing.assert_allclose(got['PSNR'], ref['PSNR'], rtol=1e-12, atol=0)
    assert np.abs(got['SSIM'] - ref['SSIM']).max() <= SSIM_ABS
    for i in (3, 16, 29):                     # tOF entry i - 3 is the pair (i - 1, i)
        r = OM.sequence_metrics(true[i - 1:i + 1], pred[i - 1:i + 1], cutfr=0, keys=('tOF',))['tOF'][0]
        assert abs(got['tOF'][i - 3] - r) <= max(TOF_REL * r, TOF_ABS), (i, got['tOF'][i - 3], r)
