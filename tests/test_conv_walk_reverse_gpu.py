"""pytest -m gpu: the conv kernel's reversed tile walk (TG_AMODE_REVERSE, PackedConv.reverse) gives the same bits as
the forward walk on every path of the kernel: the three-consumer halo conv (plain, residual, pooled; cout 64 and 128
split over two CTAs), split-K over a cluster (pooled or not), the pixels-on-N transposed conv, the tap kernel and the
thin NCHW head.  Shapes are ragged (half-height bottom tile rows, partial tiles at the right edge, several images),
and the grids leave a CTA with many tiles, with one tile (max_ctas at least the tile count), or with none on some
consumers.  Every output buffer is filled with NaN first, so each check also shows that every output pixel was
written."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

GRIDS = (0, 1, 3, 1 << 20)   # max_ctas; 0 = one CTA per SM, 1 << 20 = one tile per CTA


def _mods():
    import torch
    assert torch.cuda.is_available(), 'pytest -m gpu needs a GPU'
    import gpu_checks
    return torch, gpu_checks


def _layer(G, kind, cin, cout, n, h, w, seed, act=None, epilogue=None):
    L, ops = G.L, G.ops
    x = G.rand(seed, n, cin, h, w, lo=-1, hi=1)
    bound = 1.5 / np.sqrt(9 * cin)
    shape = (cout, cin, 3, 3) if kind == L.CONV_3X3 else (cin, cout, 3, 3)
    wt = G.rand(seed + 1, *shape, lo=-bound, hi=bound)
    b = G.rand(seed + 2, cout, lo=-0.3, hi=0.3)
    pc = ops.PackedConv(wt.to(G.DEV), b.to(G.DEV), kind, L.ACT_RELU if act is None else act,
                        L.EPI_NHWC_F16 if epilogue is None else epilogue)
    return pc, G.nhwc(x, pc.cin)


def _both_walks(torch, pc, xg, out_shape, dtype=None, **kw):
    """{(reverse, max_ctas): output} over both walks and GRIDS."""
    outs = {}
    for rev in (False, True):
        pc.reverse = rev
        for m in GRIDS:
            y = torch.full(out_shape, float('nan'), dtype=dtype or torch.float16, device=xg.device)
            pc(xg, y=y, max_ctas=m, **kw)
            torch.cuda.synchronize()
            assert not torch.isnan(y).any(), f'reverse={rev} max_ctas={m}: output pixels left unwritten'
            outs[(rev, m)] = y
    pc.reverse = False
    return outs


def _assert_same(torch, outs, what):
    ref = outs[(False, 0)]
    for key, y in outs.items():
        assert torch.equal(y, ref), f'{what}: reverse={key[0]} max_ctas={key[1]} differs from the forward full grid'


@pytest.mark.parametrize('n,h,w', [(1, 16, 8), (1, 20, 24), (2, 37, 45), (3, 9, 13)])
@pytest.mark.parametrize('cout', [64, 128])
@pytest.mark.parametrize('variant', ['plain', 'residual', 'pool'])
def test_halo_reverse_bit_exact(variant, cout, n, h, w):
    torch, G = _mods()
    L = G.L
    pc, xg = _layer(G, L.CONV_3X3, 64, cout, n, h, w, seed=1300 + h + cout)
    pool = variant == 'pool'
    res = G.nhwc(G.rand(1310 + h, n, cout, h, w, lo=-1, hi=1), cout) if variant == 'residual' else None
    shape = (n, h // 2, w // 2, cout) if pool else (n, h, w, cout)
    outs = _both_walks(torch, pc, xg, shape, residual=res, a_mode=L.AMODE_HALO, pool=pool)
    _assert_same(torch, outs, f'halo {variant} cout={cout} n={n} h={h} w={w}')


@pytest.mark.parametrize('cin,cout,n,h,w', [(128, 128, 2, 37, 45), (256, 256, 1, 16, 40), (256, 128, 3, 21, 13),
                                            (128, 64, 1, 5, 3)])
@pytest.mark.parametrize('pool', [False, True])
def test_splitk_reverse_bit_exact(cin, cout, n, h, w, pool):
    torch, G = _mods()
    L = G.L
    pc, xg = _layer(G, L.CONV_3X3, cin, cout, n, h, w, seed=1400 + cin + h, act=L.ACT_LRELU02)
    if pool and (h < 2 or w < 2):
        pytest.skip('the pooled epilogue needs h, w >= 2')
    shape = (n, h // 2, w // 2, cout) if pool else (n, h, w, cout)
    outs = _both_walks(torch, pc, xg, shape, a_mode=L.AMODE_AUTO, pool=pool)
    _assert_same(torch, outs, f'split-K pool={pool} cin={cin} cout={cout} n={n} h={h} w={w}')


@pytest.mark.parametrize('n,h,w', [(1, 16, 8), (2, 17, 23), (1, 33, 40)])
@pytest.mark.parametrize('a_mode', ['halo', 'tap'])
def test_convT_reverse_bit_exact(a_mode, n, h, w):
    torch, G = _mods()
    L = G.L
    pc, xg = _layer(G, L.CONVT_3X3_S2, 64, 64, n, h, w, seed=1500 + h)
    mode = {'halo': L.AMODE_HALO, 'tap': L.AMODE_TAP}[a_mode]
    outs = _both_walks(torch, pc, xg, (n, 2 * h, 2 * w, 64), a_mode=mode)
    _assert_same(torch, outs, f'convT {a_mode} n={n} h={h} w={w}')


@pytest.mark.parametrize('n,h,w', [(1, 20, 24), (2, 37, 45)])
def test_tap_mode_reverse_bit_exact(n, h, w):
    torch, G = _mods()
    L = G.L
    pc, xg = _layer(G, L.CONV_3X3, 64, 64, n, h, w, seed=1600 + h)
    res = G.nhwc(G.rand(1610 + h, n, 64, h, w, lo=-1, hi=1), 64)
    outs = _both_walks(torch, pc, xg, (n, h, w, 64), residual=res, a_mode=L.AMODE_TAP)
    _assert_same(torch, outs, f'tap n={n} h={h} w={w}')


@pytest.mark.parametrize('n,h,w', [(1, 16, 8), (2, 37, 45)])
def test_thin_head_reverse_bit_exact(n, h, w):
    torch, G = _mods()
    L = G.L
    pc, xg = _layer(G, L.CONV_3X3, 32, 2, n, h, w, seed=1700 + h, act=L.ACT_NONE, epilogue=L.EPI_FLOW_NCHW_F32)
    outs = _both_walks(torch, pc, xg, (n, 2, h, w), dtype=torch.float32)
    _assert_same(torch, outs, f'flow head n={n} h={h} w={w}')
