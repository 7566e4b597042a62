"""pytest -m gpu: the forward halo conv 64->64 (plain, with a residual, pooled) with three consumer warpgroups on one
shared ring of halo stages, and half-height MMAs for a bottom tile row with at most 8 rows inside the image.

- Grid independence, bit for bit: the CTA's tiles go to consumer i mod 3, so the grids below leave a CTA from 1 to
  72 tiles (counts = 0, 1 and 2 mod 3, and CTAs whose second or third consumer has no tile), with cout = 64 and with
  cout = 128 split over two CTAs.
- Half-height row, bit for bit: conv(x) equals the first h rows of conv(x'), where x' is x zero-extended to a
  multiple of 16 rows and so runs the full-height MMAs; likewise the pooled rows.
- Against a float64 conv of the fp16-rounded operands."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

GRIDS = (0, 1, 2, 3, 4, 5, 7)   # max_ctas; 0 = one CTA per SM
TOL = 3e-3                      # rel max error, as gpu_checks.check_conv


def _layer(seed, n, h, w, cout, variant, cin_real=64):
    import numpy as np
    import gpu_checks as G
    x = G.rand(seed, n, cin_real, h, w, lo=-1, hi=1)
    bound = 1.5 / np.sqrt(9 * cin_real)
    wt = G.rand(seed + 1, cout, cin_real, 3, 3, lo=-bound, hi=bound)
    b = G.rand(seed + 2, cout, lo=-0.5, hi=0.5)
    res = G.rand(seed + 3, n, cout, h, w, lo=-1, hi=1) if variant == 'residual' else None
    pc = G.ops.PackedConv(wt.to(G.DEV), b.to(G.DEV), G.L.CONV_3X3, G.L.ACT_RELU)
    return x, wt, b, res, pc


def _ref64(x, wt, b, res, pool):
    """float64 conv + ReLU (+ residual) (+ 2x2 max-pool) of the fp16-rounded operands, NCHW."""
    import torch
    import torch.nn.functional as F
    y = F.conv2d(x.half().double(), wt.half().double(), b.double(), padding=1).clamp_min(0)
    if res is not None:
        y = y + res.half().double()
    return F.max_pool2d(y, 2) if pool else y


# (n, h, w): 1 tile; 2 tiles (one CTA at max_ctas = 1: the third consumer has none); 6 tiles; 15 tiles; 2 images of
# 3x6 tiles with ragged edges (h = 37: the bottom tile row has 5 rows, the half-height MMAs)
@pytest.mark.parametrize('n,h,w', [(1, 16, 8), (1, 16, 16), (1, 20, 24), (1, 48, 40), (2, 37, 45)])
@pytest.mark.parametrize('cout', [64, 128])
@pytest.mark.parametrize('variant', ['plain', 'residual', 'pool'])
def test_three_consumers_grid_independent(variant, cout, n, h, w):
    import torch
    assert torch.cuda.is_available(), 'pytest -m gpu needs a GPU'
    import gpu_checks as G
    x, wt, b, res, pc = _layer(900 + h, n, h, w, cout, variant)
    assert pc.cout == cout
    xg = G.nhwc(x)
    rg = G.nhwc(res, cout) if res is not None else None
    pool = variant == 'pool'
    outs = [pc(xg, residual=rg, a_mode=G.L.AMODE_HALO, max_ctas=m, pool=pool) for m in GRIDS]
    torch.cuda.synchronize()
    for m, y in zip(GRIDS[1:], outs[1:]):
        assert torch.equal(y, outs[0]), f'{variant} cout={cout} n={n} h={h} w={w}: max_ctas={m} differs from the full grid'
    ref = _ref64(x, wt, b, res, pool)
    e = G.relmax(G.from_nhwc(outs[0], cout).numpy(), ref.numpy())
    assert e <= TOL, f'{variant} cout={cout} n={n} h={h} w={w}: rel max err {e} against float64'


# every h mod 16 in 1..15, below and above one tile row; h mod 16 <= 8 takes the half-height MMAs in the bottom row
@pytest.mark.parametrize('h', [r for r in range(1, 16)] + [16 + r for r in range(1, 16)])
@pytest.mark.parametrize('variant', ['plain', 'residual', 'pool'])
def test_half_height_bottom_row(variant, h):
    import torch
    assert torch.cuda.is_available(), 'pytest -m gpu needs a GPU'
    import gpu_checks as G
    if variant == 'pool' and h < 2:
        pytest.skip('the pooled epilogue needs h >= 2')
    n, w, cout = 2, 21, 64
    x, wt, b, res, pc = _layer(950 + h, n, h, w, cout, variant)
    hp = (h + 15) // 16 * 16
    xp = torch.zeros(n, 64, hp, w)
    xp[:, :, :h] = x
    resp = None
    if res is not None:
        resp = torch.zeros(n, cout, hp, w)
        resp[:, :, :h] = res
    pool = variant == 'pool'
    y = pc(G.nhwc(x), residual=G.nhwc(res) if res is not None else None, a_mode=G.L.AMODE_HALO, pool=pool)
    yp = pc(G.nhwc(xp), residual=G.nhwc(resp) if resp is not None else None, a_mode=G.L.AMODE_HALO, pool=pool)
    torch.cuda.synchronize()
    rows = h // 2 if pool else h
    assert y.shape[1] == rows
    assert torch.equal(y, yp[:, :rows]), f'{variant} h={h}: differs from the zero-extended {hp}-row input'
    ref = _ref64(x, wt, b, res, pool)
    e = G.relmax(G.from_nhwc(y, cout).numpy(), ref.numpy())
    assert e <= TOL, f'{variant} h={h}: rel max err {e} against float64'


# thin input (FNet's first layer: 6 real channels, one k-step per tap) through the half-height row
@pytest.mark.parametrize('h', [5, 24, 25])
def test_half_height_thin_input(h):
    import torch
    assert torch.cuda.is_available(), 'pytest -m gpu needs a GPU'
    import gpu_checks as G
    n, w, cout = 2, 30, 64
    x, wt, b, _, pc = _layer(990 + h, n, h, w, cout, 'plain', cin_real=6)
    hp = (h + 15) // 16 * 16
    xp = torch.zeros(n, 6, hp, w)
    xp[:, :, :h] = x
    y = pc(G.nhwc(x), a_mode=G.L.AMODE_HALO)
    yp = pc(G.nhwc(xp), a_mode=G.L.AMODE_HALO)
    torch.cuda.synchronize()
    assert torch.equal(y, yp[:, :h]), f'thin h={h}: differs from the zero-extended {hp}-row input'
    e = G.relmax(G.from_nhwc(y, cout).numpy(), _ref64(x, wt, b, None, False).numpy())
    assert e <= TOL, f'thin h={h}: rel max err {e} against float64'
