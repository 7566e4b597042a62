"""pytest -m gpu: the forward halo conv 64->64 (plain, with a residual, pooled) gives the same bits whatever the
grid.  The two consumer warpgroups of a CTA take turns issuing their MMAs tile by tile; the sizes include an image
so small that some CTAs' second consumer has no tile, and grids that leave a CTA an odd number of tiles."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

GRIDS = (0, 1, 2, 3, 7)   # max_ctas; 0 = one CTA per SM


# (n, h, w): 2x3 tiles (fewer tiles than CTAs: one tile per CTA); 3x5 tiles (15: odd per CTA at 1, 3 and 7 CTAs);
# 3x6 tiles x 2 images with ragged edges
@pytest.mark.parametrize('n,h,w', [(1, 20, 24), (1, 48, 40), (2, 37, 45)])
@pytest.mark.parametrize('variant', ['plain', 'residual', 'pool'])
def test_halo_conv_grid_independent(variant, n, h, w):
    import torch
    assert torch.cuda.is_available(), 'pytest -m gpu needs a GPU'
    import numpy as np
    import gpu_checks as G
    L, ops = G.L, G.ops
    seed = 700
    x = G.rand(seed, n, 64, h, w, lo=-1, hi=1)
    bound = 1.5 / np.sqrt(9 * 64)
    wt = G.rand(seed + 1, 64, 64, 3, 3, lo=-bound, hi=bound)
    b = G.rand(seed + 2, 64, lo=-0.5, hi=0.5)
    res = G.rand(seed + 3, n, 64, h, w, lo=-1, hi=1) if variant == 'residual' else None
    pc = ops.PackedConv(wt.to(G.DEV), b.to(G.DEV), L.CONV_3X3, L.ACT_RELU)
    xg = G.nhwc(x)
    rg = G.nhwc(res) if res is not None else None
    pool = variant == 'pool'
    outs = [pc(xg, residual=rg, a_mode=L.AMODE_HALO, max_ctas=m, pool=pool) for m in GRIDS]
    torch.cuda.synchronize()
    for m, y in zip(GRIDS[1:], outs[1:]):
        assert torch.equal(y, outs[0]), f'{variant} n={n} h={h} w={w}: max_ctas={m} differs from the full grid'
    if pool:
        # the pooled epilogue is maxpool2x2 of the unpooled conv, bit for bit
        ref = ops.maxpool2x2(pc(xg, a_mode=L.AMODE_HALO))
        torch.cuda.synchronize()
        assert torch.equal(outs[0], ref)
    else:
        ref = G._conv_ref(x, wt, b, L.CONV_3X3, L.ACT_RELU, res)
        e = G.relmax(G.from_nhwc(outs[0], 64).numpy(), ref.numpy())
        assert e <= 3e-3, f'{variant} n={n} h={h} w={w}: rel max err {e}'
