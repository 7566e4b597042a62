"""pytest -m gpu: the resize kernel tg_resample_nchw_f32 against oracle/resample.py (float64), at the ratios 1/4 to 2
per axis, ragged and anamorphic sizes, 1 to 4 channels, both outputs.  The input sits inside a NaN guard band (an
out-of-image read would show up as NaN in the output) and every output inside a 0xAB / NaN guard band."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402,F401
from oracle import resample as R              # noqa: E402

pytestmark = pytest.mark.gpu

ops = sys.modules['tecogan-pytorch_b200.ops']
DEV = torch.device('cuda', 0)
GUARD = 0xAB
F32_TOL = 4e-6

CASES = [  # (n, c, H, W) -> (Ho, Wo)
    ((2, 3, 76, 150), (19, 38)),        # 1/4
    ((2, 3, 74, 150), (37, 75)),        # 1/2
    ((3, 3, 68, 136), (51, 102)),       # 3/4
    ((2, 3, 37, 141), (37, 141)),       # 1
    ((2, 3, 64, 136), (72, 153)),       # 9/8
    ((2, 3, 45, 99), (60, 132)),        # 4/3
    ((2, 3, 35, 70), (70, 140)),        # 2
    ((2, 3, 60, 136), (45, 153)),       # anamorphic: 3/4 x 9/8
    ((2, 4, 40, 200), (30, 50)),        # 4 channels, 3/4 x 1/4
    ((3, 1, 9, 7), (3, 14)),            # 1 channel, axes shorter than the tap count
    ((2, 3, 536, 1280), (402, 960)),    # bench.py's bd4 HR frame to 402x960
]
IDS = [f'{H}x{W}-{Ho}x{Wo}-c{c}' for (n, c, H, W), (Ho, Wo) in CASES]


def _input(n, c, H, W, seed):
    """fp32 [n,c,H,W] in [-0.1, 1.1] placed 5 floats into a NaN buffer with a NaN tail: (tensor, numpy copy)."""
    x = np.random.default_rng(seed).uniform(-0.1, 1.1, size=(n, c, H, W)).astype(np.float32)
    buf = torch.full((x.size + 5 + 37,), float('nan'), device=DEV)
    region = buf[5:5 + x.size]
    region.copy_(torch.from_numpy(x.reshape(-1)))
    return region.view(x.shape), x


def _tables(H, W, Ho, Wo, filt):
    return [tuple(t.to(DEV) for t in ops.resample_table(a, b, filt)) for a, b in ((H, Ho), (W, Wo))]


def _run_u8(x, tabs, shape, offset):
    nbytes = int(np.prod(shape))
    buf = torch.full((offset + nbytes + 64,), GUARD, dtype=torch.uint8, device=DEV)
    out = buf[offset:offset + nbytes].view(shape)
    ops.resample(x, *tabs, out_u8=out)
    torch.cuda.synchronize()
    b = buf.cpu().numpy()
    guard = bool((b[:offset] == GUARD).all() and (b[offset + nbytes:] == GUARD).all())
    return b[offset:offset + nbytes].reshape(shape), guard


def _run_f32(x, tabs, shape, offset):
    count = int(np.prod(shape))
    buf = torch.full((offset + count + 16,), float('nan'), device=DEV)
    before = buf.view(torch.int32).clone()
    out = buf[offset:offset + count].view(shape)
    ops.resample(x, *tabs, out_f32=out)
    torch.cuda.synchronize()
    bits = buf.view(torch.int32)
    guard = bool(torch.equal(bits[:offset], before[:offset]) and torch.equal(bits[offset + count:],
                                                                               before[offset + count:]))
    return buf[offset:offset + count].cpu().numpy().reshape(shape), guard


@pytest.mark.parametrize('filt', R.FILTERS)
@pytest.mark.parametrize('case', CASES, ids=IDS)
def test_kernel_matches_oracle(case, filt):
    (n, c, H, W), (Ho, Wo) = case
    x, xn = _input(n, c, H, W, seed=H * 1000 + W + Ho)
    tabs = _tables(H, W, Ho, Wo, filt)
    ref = R.resize(xn, (Ho, Wo), filt)                                            # float64 [n,c,Ho,Wo]

    y32, guard = _run_f32(x, tabs, (n, c, Ho, Wo), offset=3)
    assert guard
    err = np.abs(y32.astype(np.float64) - ref)
    assert err.max() <= F32_TOL, float(err.max())                                # NaN (an outside read) fails too
    y32b, _ = _run_f32(x, tabs, (n, c, Ho, Wo), offset=3)
    assert np.array_equal(y32.view(np.uint32), y32b.view(np.uint32))            # two launches: the same bits

    for offset in (0, 7):
        y8, guard = _run_u8(x, tabs, (n, Ho, Wo, c), offset)
        assert guard, offset
        want = R.to_uint8(ref).transpose(0, 2, 3, 1)
        diff = np.abs(y8.astype(np.int32) - want.astype(np.int32))
        near = R.near_boundary(ref).transpose(0, 2, 3, 1)
        assert diff.max() <= 1 and not (diff[~near] > 0).any(), (int((diff > 0).sum()), int(near.sum()))
        # the uint8 output is the quantisation of the fp32 output, bit for bit
        assert np.array_equal(y8, R.to_uint8(y32).transpose(0, 2, 3, 1))


def test_scale_one_is_the_identity():
    x, xn = _input(2, 3, 57, 130, seed=1)
    for filt in R.FILTERS:
        y32, guard = _run_f32(x, _tables(57, 130, 57, 130, filt), (2, 3, 57, 130), offset=0)
        assert guard and np.array_equal(y32.view(np.uint32), xn.view(np.uint32)), filt
