"""GPU tests of tecogan_b200.metrics against the specification (oracle/metrics_oracle.py, oracle/farneback.py) and
cv2's flows (tests/golden/metrics_cv2.npz): gray bit for bit, PSNR exactly, flows and tOF within fp32 tolerances,
chunked sequences, guard bands around every output, and the argument checks."""
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
import synthetic                               # noqa: E402
from oracle import farneback as F              # noqa: E402
from oracle import metrics_oracle as MO        # noqa: E402
from test_metrics_cpu import FLOW_CASES, seeded_sequence, _reference_calculator   # noqa: E402

pytestmark = pytest.mark.gpu
L = sys.modules['tecogan-pytorch_b200.lib']
M = T.metrics
DEV = torch.device('cuda:0')
FLOW_P999 = 5e-3          # px, 99.9th percentile of |device - reference|
TOF_REL = 1e-4            # per-frame relative difference of tOF
# On the bd4 sequence the predicted frames differ by +-6 codes of noise only, so tOF is ~0.017 px and the relative
# bound meets the fp32 rounding of the flows themselves: frame 1 measured 4.5e-6 px (2.7e-4 relative) on an H100.
# There tOF is held to TOF_REL or TOF_ABS, whichever is larger.
TOF_ABS = 2e-5            # px


@pytest.fixture(scope='module')
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, 'metrics_cv2.npz'))


def _p999(a, b):
    return float(np.quantile(np.abs(np.asarray(a, np.float64) - b), 0.999))


def test_gray_is_bit_exact(gold):
    rng = np.random.default_rng(0)
    x = rng.integers(0, 256, (3, 37, 53, 3)).astype(np.uint8)
    x.reshape(-1, 3)[:len(gold['gray_rgb'])] = gold['gray_rgb']
    got = M.rgb_to_gray(torch.from_numpy(x).to(DEV)).cpu().numpy()
    assert np.array_equal(got, MO.rgb_to_gray(x))
    assert np.array_equal(M.rgb_to_gray(torch.from_numpy(x[0]).to(DEV)).cpu().numpy(), MO.rgb_to_gray(x[0]))


def _tie_frames(gold, T_=3, h=40, w=48, hp=None, wp=None, seed=1):
    """seeded frames whose true and predicted pixels contain every near-tie colour"""
    rng = np.random.default_rng(seed)
    t = rng.integers(0, 256, (T_, h, w, 3)).astype(np.uint8)
    p = rng.integers(0, 256, (T_, hp or h, wp or w, 3)).astype(np.uint8)
    ties = gold['tie_rgb']
    for k in range(T_):
        t[k].reshape(-1, 3)[:len(ties)] = ties
        p[k].reshape(-1, 3)[:len(ties)] = ties[::-1]
    return t, p


@pytest.mark.parametrize('colorspace', ['y', 'rgb'])
@pytest.mark.parametrize('sizes', [(40, 48, 40, 48), (40, 48, 44, 45), (41, 50, 37, 52)])
def test_psnr_equals_oracle(gold, colorspace, sizes):
    h, w, hp, wp = sizes
    t, p = _tie_frames(gold, 3, h, w)
    rng = np.random.default_rng(2)
    p = rng.integers(0, 256, (3, hp, wp, 3)).astype(np.uint8)
    hh, ww = min(h, hp), min(w, wp)
    p[:, :hh, :ww] = np.where(rng.random((3, hh, ww, 1)) < 0.7, t[:, :hh, :ww], p[:, :hh, :ww])
    p[2, :hh, :ww] = t[2, :hh, :ww]                          # equal frames: inf
    ref = MO.sequence_metrics(t, p, colorspace, with_tof=False)['PSNR']
    for a, b in ((t, p), (torch.from_numpy(t).to(DEV), torch.from_numpy(p).to(DEV))):
        got = M.sequence_metrics(a, b, psnr=colorspace, tof=False)
        assert list(got) == ['PSNR']
        assert got['PSNR'].dtype == np.float64
        assert list(got['PSNR']) == list(ref)                # exact, inf included
    assert np.isinf(ref[2])


@pytest.mark.parametrize('name', FLOW_CASES)
def test_flow_matches_cv2_and_oracle(gold, name):
    a, b, step = gold[f'{name}_prev'], gold[f'{name}_next'], int(gold[f'{name}_rows'])
    got = M.farneback(torch.from_numpy(a).to(DEV), torch.from_numpy(b).to(DEV))
    assert got.dtype == torch.float32 and tuple(got.shape) == a.shape + (2,)
    got = got.cpu().numpy()
    assert _p999(got[::step], gold[f'{name}_flow']) <= FLOW_P999
    assert _p999(got, F.farneback(a, b)) <= FLOW_P999


def test_flow_batch_and_parameters(gold):
    names = ('small', 'small', 'small')
    a = np.stack([gold[f'{n}_prev'] for n in names])
    b = np.stack([gold[f'{n}_next'] for n in names])
    b[1] = gold['small_prev']                                # identical pair: zero flow
    b[2] = np.roll(b[2], 3, axis=1)
    got = M.farneback(torch.from_numpy(a).to(DEV), torch.from_numpy(b).to(DEV)).cpu().numpy()
    for i in (0, 2):
        assert _p999(got[i], F.farneback(a[i], b[i])) <= FLOW_P999
    # Identical frames: the flow is small but ill-conditioned near the corners (the right / bottom edge pixels take
    # the "outside" branch and the system there is nearly singular), so fp32 rounding is amplified.  cv2 (fp32)
    # itself is 1.3e-2 px from the float64 oracle at the 99.9th percentile and 4.1e-2 px at most on this pair.
    assert np.abs(got[1]).max() < 0.25
    assert _p999(got[1], F.farneback(a[1], b[1])) <= 3e-2
    kw = dict(pyr_scale=0.6, levels=2, winsize=10, iterations=2, poly_n=7, poly_sigma=1.5)
    got = M.farneback(torch.from_numpy(a[0]).to(DEV), torch.from_numpy(b[0]).to(DEV), **kw).cpu().numpy()
    assert _p999(got, F.farneback(a[0], b[0], **kw)) <= FLOW_P999


def test_sequence_tof_matches_oracle_and_chunks():
    true, pred = seeded_sequence(T=5, h=70, w=90, hp=66, wp=95)
    ref = MO.sequence_metrics(true, pred, 'y')
    got = M.sequence_metrics(true, pred, psnr='y', tof=True)
    assert list(got) == ['PSNR', 'tOF']
    assert list(got['PSNR']) == list(ref['PSNR'])
    assert got['tOF'].shape == (4,)
    rel = np.abs(got['tOF'] - ref['tOF']) / ref['tOF']
    assert rel.max() <= TOF_REL, rel
    # a workspace bound that forces chunks of 2 and 3 frames gives the same numbers
    for n in (2, 3):
        hw = 66 * 90
        bound = (T.ops.farneback_workspace_bytes(2, n, 66, 90) + 2 * n * hw + 2 * (n - 1) * hw * 8
                 + 2 * n * hw * 6)
        ch = M.sequence_metrics(true, pred, psnr='y', tof=True, max_workspace_bytes=bound)
        assert list(ch['PSNR']) == list(got['PSNR'])
        assert np.array_equal(ch['tOF'], got['tOF'])
    assert list(M.sequence_metrics(true, pred, psnr=None, tof=True)) == ['tOF']
    one = M.sequence_metrics(true[:1], pred[:1], psnr='rgb', tof=True)
    assert one['tOF'].shape == (0,) and one['PSNR'].shape == (1,)


def test_bd4_hr_sequence():
    """536x1280, T = 32: PSNR of every frame exactly, tOF of three pairs (the oracle is slow) within TOF_REL"""
    clip = synthetic.make_clip(3, 32, 3, 536, 1280, shift=2)
    true = (clip.permute(0, 2, 3, 1) * 255).round().to(torch.uint8).numpy()
    rng = np.random.default_rng(4)
    pred = np.clip(true.astype(np.int16) + rng.integers(-6, 7, true.shape), 0, 255).astype(np.uint8)
    got = M.sequence_metrics(torch.from_numpy(true).to(DEV), torch.from_numpy(pred).to(DEV), psnr='y')
    assert got['PSNR'].shape == (32,) and got['tOF'].shape == (31,)
    ref = MO.sequence_metrics(true, pred, 'y', frames={1, 16, 31})
    assert list(got['PSNR']) == list(ref['PSNR'])
    d = {i: abs(got['tOF'][i - 1] - ref['tOF'][i - 1]) for i in (1, 16, 31)}
    assert all(d[i] <= max(TOF_REL * ref['tOF'][i - 1], TOF_ABS) for i in d), (d, ref['tOF'][[0, 15, 30]])


def test_guard_bands():
    lib = L.load()
    rng = np.random.default_rng(5)
    n, t, h, w, g = 2, 3, 45, 70, 4096
    gray = torch.from_numpy(rng.integers(0, 256, (n * t, h, w)).astype(np.uint8)).to(DEV)
    params = T.ops.farneback_params(0.5, 3, 15, 3, 5, 1.2, 0)
    need = T.ops.farneback_workspace_bytes(n, t, h, w)
    nflow = n * (t - 1) * h * w * 2
    fbuf = torch.full((nflow + 2 * g,), float('nan'), device=DEV)
    wbuf = torch.full((need + 2 * g * 4,), 0xA5, dtype=torch.uint8, device=DEV)
    L.check(lib.tg_farneback(ctypes.c_void_p(gray.data_ptr()), n, t, h, w, ctypes.byref(params),
                             ctypes.c_void_p(fbuf.data_ptr() + 4 * g), ctypes.c_void_p(wbuf.data_ptr() + 4 * g), need,
                             ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), 'tg_farneback')
    torch.cuda.synchronize()
    assert torch.isnan(fbuf[:g]).all() and torch.isnan(fbuf[-g:]).all()
    assert not torch.isnan(fbuf[g:-g]).any()
    assert (wbuf[:4 * g] == 0xA5).all() and (wbuf[-4 * g:] == 0xA5).all()
    ref = T.ops.farneback(gray, n, params)
    assert torch.equal(fbuf[g:-g].view_as(ref), ref)         # same bits as a call with its own buffers
    # frame input: gray and sse inside guard bands
    tr = torch.from_numpy(rng.integers(0, 256, (t, h, w, 3)).astype(np.uint8)).to(DEV)
    pr = torch.from_numpy(rng.integers(0, 256, (t, h, w, 3)).astype(np.uint8)).to(DEV)
    gb = torch.full((2 * t * h * w + 2 * g,), 0x5A, dtype=torch.uint8, device=DEV)
    sb = torch.full((t + 2 * 8,), -7, dtype=torch.int64, device=DEV)
    L.check(lib.tg_metrics_frames_in(ctypes.c_void_p(tr.data_ptr()), h, w, ctypes.c_void_p(pr.data_ptr()), h, w, t,
                                     L.PSNR_RGB, ctypes.c_void_p(gb.data_ptr() + g),
                                     ctypes.c_void_p(sb.data_ptr() + 64),
                                     ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), 'frames_in')
    torch.cuda.synchronize()
    assert (gb[:g] == 0x5A).all() and (gb[-g:] == 0x5A).all()
    assert (sb[:8] == -7).all() and (sb[-8:] == -7).all()
    a, b = tr.cpu().numpy().astype(np.int64), pr.cpu().numpy().astype(np.int64)
    assert list(sb[8:-8].cpu().numpy()) == [int(((a[k] - b[k]) ** 2).sum()) for k in range(t)]
    gray_ref = np.concatenate([MO.rgb_to_gray(a.astype(np.uint8)), MO.rgb_to_gray(b.astype(np.uint8))]).ravel()
    assert np.array_equal(gb[g:-g].cpu().numpy(), gray_ref)
    # epe sums
    fa = torch.randn(3, h, w, 2, device=DEV)
    fb = torch.randn(3, h, w, 2, device=DEV)
    sums = torch.full((3 + 16,), float('nan'), dtype=torch.float64, device=DEV)
    L.check(lib.tg_flow_epe_sum(ctypes.c_void_p(fa.data_ptr()), ctypes.c_void_p(fb.data_ptr()), 3, h, w,
                                ctypes.c_void_p(sums.data_ptr() + 64),
                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), 'epe')
    torch.cuda.synchronize()
    assert torch.isnan(sums[:8]).all() and torch.isnan(sums[-8:]).all()
    ref = (fa - fb).double().norm(dim=-1).sum(dim=(1, 2))
    assert torch.allclose(sums[8:-8], ref, rtol=1e-6)


def test_bad_arguments_raise():
    x = torch.zeros(2, 16, 16, dtype=torch.uint8, device=DEV)
    with pytest.raises(ValueError):
        M.farneback(x, x[:1])
    with pytest.raises(ValueError):
        M.farneback(x.float(), x)
    with pytest.raises(ValueError):
        M.farneback(x, x, flags=256)
    with pytest.raises(ValueError):
        M.farneback(x, x, pyr_scale=1.5)
    with pytest.raises(ValueError):
        M.rgb_to_gray(x)
    f = torch.zeros(2, 16, 16, 3, dtype=torch.uint8, device=DEV)
    with pytest.raises(ValueError):
        M.sequence_metrics(f, f[:1])
    with pytest.raises(ValueError):
        M.sequence_metrics(f, f, max_workspace_bytes=1000)
    with pytest.raises(T.TecoganB200Error):
        T.ops.farneback(x[:, :1], 2, T.ops.farneback_params(0.5, 3, 15, 3, 5, 1.2, 0))   # 1-row frames


class GpuMetricCalculator:
    """the subclass of INTEGRATION.md, built on the reference's MetricCalculator at test time"""

    @staticmethod
    def make(base):
        class Calc(base):
            def compute_sequence_metrics(self, seq_idx, true_seq, pred_seq):
                opt = self.metric_opt
                dev = M.sequence_metrics(true_seq, pred_seq,
                                         psnr=self.psnr_colorspace if 'PSNR' in opt else None,
                                         tof='tOF' in opt)
                lpips = OrderedDict((k, v) for k, v in opt.items() if k == 'LPIPS')
                saved, self.metric_opt = self.metric_opt, lpips
                try:
                    super().compute_sequence_metrics(seq_idx, true_seq, pred_seq)
                finally:
                    self.metric_opt = saved
                self.metric_dict[seq_idx] = OrderedDict(
                    (k, list(dev[k]) if k in dev else self.metric_dict[seq_idx][k]) for k in opt)
        return Calc


@pytest.mark.parametrize('colorspace', ['y', 'rgb'])
def test_integration_subclass_matches_reference(colorspace):
    ref_calc = _reference_calculator(colorspace)
    true, pred = seeded_sequence(T=4, h=64, w=80, hp=64, wp=78, seed=9)
    ref_calc.compute_sequence_metrics('s', true, pred)
    calc = _reference_calculator(colorspace)
    calc.__class__ = GpuMetricCalculator.make(type(calc))
    calc.compute_sequence_metrics('s', true, pred)
    ref, got = ref_calc.metric_dict['s'], calc.metric_dict['s']
    assert list(got) == list(ref)
    assert got['PSNR'] == ref['PSNR']
    assert np.allclose(got['tOF'], ref['tOF'], rtol=TOF_REL, atol=0)
