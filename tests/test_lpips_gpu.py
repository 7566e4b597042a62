"""GPU tests of LPIPS on the device: the 192 / 384-channel convs (wgmma against the CUDA-core kernel per element, and
that against float64), each AlexNet layer's features against oracle/lpips.py, LPIPS and tLP100 against
tests/golden/lpips.npz (the reference's two copies) and the oracle, determinism across reruns and chunkings, guard
bands around the new kernels' outputs, and the key order of both metric functions."""
import os
import re
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                            # noqa: E402
import synthetic                                    # noqa: E402
from oracle import lpips as O                       # noqa: E402

M, ops = T.metrics, T.ops
L = sys.modules['tecogan-pytorch_b200.lib']
pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
# Bounds against the float64 reference, from the largest errors measured on an H100 on these sequences (DESIGN.md
# 3.7) with a margin of about 2x:
#   per-frame LPIPS within REL * d + ABS: measured 2.7e-4 relative (MetricCalculator's input), 2.0e-4 (the script's)
#   tLP100 within 100 * REL_TLP * (d_true + d_pred) + TLP_F32: measured 7.2e-5 of 100 (d_true + d_pred), where
#   d_true = d(true[i-1], true[i]) and d_pred = d(pred[i-1], pred[i]); TLP_F32 covers the script's float32 rounding
REL, ABS = 6e-4, 1e-7
REL_TLP, TLP_F32 = 2e-4, 2e-6


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.fixture(scope='module')
def params():
    return synthetic.make_lpips_params(7)


@pytest.fixture(scope='module')
def lp(params):
    return M.LPIPS(params, DEV)


@pytest.fixture(scope='module')
def seqs(golden_dir):
    g = np.load(os.path.join(golden_dir, 'official_metrics.npz'))
    return [(g['true_0'], g['pred_0']), (g['true_1'], g['pred_1'])]


@pytest.fixture(scope='module')
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, 'lpips.npz'))


@pytest.mark.parametrize('cin,cout', [(192, 384), (384, 256), (256, 192)])
@pytest.mark.parametrize('n,h,w', [(1, 16, 8), (1, 17, 9), (2, 31, 77), (1, 5, 3)])
def test_new_channel_counts_match_simt_and_float64(cin, cout, n, h, w):
    g = torch.Generator().manual_seed(cin * 1000 + cout + h)
    wt = torch.randn(cout, cin, 3, 3, generator=g) / (3 * cin ** 0.5)
    b = torch.randn(cout, generator=g) * 0.1
    x = torch.randn(n, h, w, cin, generator=g).half()
    conv = ops.PackedConv(wt.to(DEV), b.to(DEV), L.CONV_3X3, L.ACT_RELU, L.EPI_NHWC_F16)
    xd = x.to(DEV)
    y_tc = conv(xd, impl='tcgen05')
    y_simt = conv(xd, impl='simt')
    torch.cuda.synchronize()
    ref = F.relu(F.conv2d(x.double().permute(0, 3, 1, 2), wt.half().double(), b.double(), padding=1)).permute(0, 2, 3, 1)
    d = (y_tc.float() - y_simt.float()).abs()
    tol = 2e-3 * (1 + y_simt.float().abs())          # the two round their fp32 sums to fp16 independently
    assert bool((d <= tol).all()), float(d.max())
    assert _rel(y_simt, ref) <= 1e-3


def _features(lp, params, u8, norm='calc'):
    x = torch.from_numpy(u8).to(DEV)
    n, h, w, _ = u8.shape
    feats = lp.features(x, (0, 0, h, w), L.LPIPS_NORM_CALC if norm == 'calc' else L.LPIPS_NORM_OFFICIAL)
    sz = M.lpips_sizes(h, w)
    got = []
    for f, (_, (y0, x0, hh, ww)) in zip(feats, sz):
        got.append(f[:, y0:y0 + hh, x0:x0 + ww].permute(0, 3, 1, 2))
    return got, O.features(params, O.scaled_input(u8, norm))


@pytest.mark.parametrize('h,w', [(536, 1280), (512, 1248), (67, 101), (31, 31), (33, 64)])
def test_layer_features_against_float64(lp, params, h, w):
    rng = np.random.default_rng(h + w)
    u8 = rng.integers(0, 256, (1 if h > 200 else 2, h, w, 3), dtype=np.uint8)
    got, want = _features(lp, params, u8)
    for l, (a, b) in enumerate(zip(got, want)):
        assert tuple(a.shape) == tuple(b.shape), l
        assert _rel(a, b) <= 1e-3, (l, _rel(a, b))


def test_lpips_and_tlp_against_reference_and_oracle(lp, params, seqs, gold):
    for k, (t, p) in enumerate(seqs):
        r = M.official_sequence_metrics(t, p, keys=('LPIPS', 'tLP100'), lpips=lp)
        want = O.official_lpips(params, t, p)
        for ref in (want['LPIPS'], gold[f'lpips_{k}']):
            assert np.all(np.abs(r['LPIPS'] - ref) <= REL * ref + ABS), np.abs(r['LPIPS'] - ref).max()
        # |d_true - d_pred| * 100: each of the two distances carries its own error
        bound = 100 * REL_TLP * (want['d_true'] + want['d_pred']) + TLP_F32
        for ref in (want['tLP100'], gold[f'tlp100_{k}']):
            assert np.all(np.abs(r['tLP100'] - ref) <= bound), np.abs(r['tLP100'] - ref).max()
        h, w = min(t.shape[1], p.shape[1]), min(t.shape[2], p.shape[2])
        c = lp(t, p)
        ref = gold[f'calc_lpips_{k}']
        assert np.all(np.abs(c - ref) <= REL * ref + ABS), np.abs(c - ref).max()
        np.testing.assert_allclose(c, O.lpips(params, t[:, :h, :w], p[:, :h, :w]), rtol=REL, atol=ABS)
        s = M.sequence_metrics(t, p, psnr='y', tof=False, lpips=lp)
        assert list(s) == ['PSNR', 'LPIPS']
        np.testing.assert_array_equal(s['LPIPS'], c)


def test_identical_frames_score_zero(lp):
    x = np.random.default_rng(1).integers(0, 256, (2, 40, 50, 3), dtype=np.uint8)
    assert np.all(lp(x, x) == 0)


def _smallest_workspace(fn):
    """the smallest max_workspace_bytes fn accepts: the bytes of its smallest chunk, from the refusal of 1 byte"""
    with pytest.raises(ValueError, match='below the') as e:
        fn(1)
    return int(re.search(r'below the (\d+) bytes', str(e.value)).group(1))


def _chunked(lp, monkeypatch, fn, limit):
    """fn(limit), and the number of LPIPS passes (one per chunk) it ran"""
    calls, orig = [], lp.distances
    monkeypatch.setattr(lp, 'distances', lambda *a, **k: (calls.append(1), orig(*a, **k))[1])
    out = fn(limit)
    monkeypatch.undo()
    return out, len(calls)


def test_reruns_and_chunks_give_the_same_bits(lp, seqs, monkeypatch):
    t, p = seqs[0]                                       # T = 8: 4 scored frames
    for keys in (('PSNR', 'SSIM', 'LPIPS', 'tOF', 'tLP100'), ('LPIPS', 'tLP100'), ('LPIPS',)):
        def run(limit):
            return M.official_sequence_metrics(t, p, keys=keys, lpips=lp, max_workspace_bytes=limit)
        a, b = run(M.DEFAULT_MAX_WORKSPACE_BYTES), run(M.DEFAULT_MAX_WORKSPACE_BYTES)
        small, passes = _chunked(lp, monkeypatch, run, _smallest_workspace(run))
        # two frames per chunk with a temporal metric (chunks overlap by one), else one
        assert passes == (3 if 'tLP100' in keys else 4)
        assert list(a) == list(small) == list(keys)
        for k in keys:
            np.testing.assert_array_equal(a[k], b[k])
            np.testing.assert_array_equal(a[k], small[k])
    for tof in (True, False):
        def run(limit):
            return M.sequence_metrics(t, p, tof=tof, lpips=lp, max_workspace_bytes=limit)
        s1 = run(M.DEFAULT_MAX_WORKSPACE_BYTES)
        s2, passes = _chunked(lp, monkeypatch, run, _smallest_workspace(run))
        assert passes == (7 if tof else 8)
        assert list(s1) == list(s2) == (['PSNR', 'LPIPS', 'tOF'] if tof else ['PSNR', 'LPIPS'])
        for k in s1:
            np.testing.assert_array_equal(s1[k], s2[k])

    def call(limit):
        return lp(t, p, max_workspace_bytes=limit)
    c, passes = _chunked(lp, monkeypatch, call, _smallest_workspace(call))
    assert passes == 8
    np.testing.assert_array_equal(c, lp(t, p))


def test_host_and_cuda_input_give_the_same_keys_and_values(lp, seqs):
    t, p = seqs[0]
    keys = ('tLP100', 'LPIPS', 'PSNR')
    host = M.official_sequence_metrics(t, p, keys=keys, lpips=lp)
    dev = M.official_sequence_metrics(torch.from_numpy(t).to(DEV), torch.from_numpy(p).to(DEV), keys=keys, lpips=lp)
    assert list(host) == list(dev) == ['PSNR', 'LPIPS', 'tLP100']
    for k in host:
        np.testing.assert_array_equal(host[k], dev[k])
    s = M.sequence_metrics(torch.from_numpy(t).to(DEV), torch.from_numpy(p).to(DEV), lpips=lp)
    assert list(s) == ['PSNR', 'LPIPS', 'tOF']


def _guarded(shape, dtype):
    """a tensor of `shape` inside a 0xAB-filled buffer with 4 KB of guard on each side"""
    item = torch.empty(0, dtype=dtype).element_size()
    n = int(np.prod(shape))
    g = 4096 // item
    buf = torch.full(((n + 2 * g) * item,), 0xAB, dtype=torch.uint8, device=DEV)
    return buf, buf[g * item:(g + n) * item].view(dtype).view(*shape), g * item, (g + n) * item


def _intact(buf, lo, hi):
    torch.cuda.synchronize()
    return bool((buf[:lo] == 0xAB).all()) and bool((buf[hi:] == 0xAB).all())


def test_guard_bands(lp):
    rng = np.random.default_rng(3)
    u8 = torch.from_numpy(rng.integers(0, 256, (2, 45, 70, 3), dtype=np.uint8)).to(DEV)
    sz = M.lpips_sizes(37, 61)
    buf, x, lo, hi = _guarded((2, *sz[0][0], 64), torch.float16)
    ops.lpips_frames_in(u8, (3, 5, 37, 61), L.LPIPS_NORM_OFFICIAL, x)
    assert _intact(buf, lo, hi)
    f1 = lp.convs[0](x)
    ph, pw = (sz[0][1][2] - 3) // 2 + 1, (sz[0][1][3] - 3) // 2 + 1
    for shifts, shape in ((True, (2, ph + 2, pw + 2, 256)), (False, (2, ph, pw, 64))):
        buf, y, lo, hi = _guarded(shape, torch.float16)
        ops.maxpool3x3s2(f1, sz[0][1], shifts, y)
        assert _intact(buf, lo, hi)
    pairs = torch.tensor([[0, 1], [1, 0], [1, 1]], dtype=torch.int32, device=DEV)
    buf, out, lo, hi = _guarded((3,), torch.float64)
    ops.lpips_head(f1, sz[0][1], pairs, lp.heads[0], out, accumulate=False)
    assert _intact(buf, lo, hi)
    assert out[0].item() == out[1].item() and out[2].item() == 0
