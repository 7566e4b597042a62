"""pytest -m gpu: the forward stride-2 transposed conv and the conv with MaxPool2d(2, 2) folded into its epilogue,
both on the pixels-on-N halo path (register epilogue, TMA tensor stores).  Every output buffer is filled with NaN
first, so each check also shows that every output pixel was written."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu


def _mods():
    import torch
    assert torch.cuda.is_available(), 'pytest -m gpu needs a GPU'
    import gpu_checks
    return torch, gpu_checks


def _run(torch, pc, xg, shape, **kw):
    y = torch.full(shape, float('nan'), dtype=torch.float16, device=xg.device)
    pc(xg, y=y, **kw)
    torch.cuda.synchronize()
    assert not torch.isnan(y).any(), 'output pixels left unwritten'
    return y


def _convT(G, n, h, w, seed):
    L, ops = G.L, G.ops
    x = G.rand(seed, n, 64, h, w, lo=-1, hi=1)
    bound = 1.5 / np.sqrt(9 * 64)
    wt = G.rand(seed + 1, 64, 64, 3, 3, lo=-bound, hi=bound)
    b = G.rand(seed + 2, 64, lo=-0.5, hi=0.5)
    pc = ops.PackedConv(wt.to(G.DEV), b.to(G.DEV), L.CONVT_3X3_S2, L.ACT_RELU)
    return pc, G.nhwc(x), x, wt, b


@pytest.mark.parametrize('n,h,w', [(4, 134, 320), (3, 21, 13), (2, 17, 9), (1, 5, 3)])
def test_convT_halo_vs_tap_and_torch(n, h, w):
    """The pixels-on-N transposed conv against the tap-mode kernel on the same packed weights (fp32 sums in
    another order, so 1 fp16 ulp here and there) and against torch fp32 conv_transpose2d + ReLU."""
    torch, G = _mods()
    import torch.nn.functional as F
    L = G.L
    pc, xg, x, wt, b = _convT(G, n, h, w, seed=700 + h)
    shape = (n, 2 * h, 2 * w, 64)
    got = _run(torch, pc, xg, shape, a_mode=L.AMODE_HALO)
    tap = _run(torch, pc, xg, shape, a_mode=L.AMODE_TAP)
    e_tap = float((got.float() - tap.float()).abs().max() / tap.float().abs().max())
    assert e_tap <= 2e-3, f'halo vs tap: rel max {e_tap}'
    ref = F.relu(F.conv_transpose2d(G.f16(x), G.f16(wt), b, 2, 1, output_padding=1))
    e_ref = G.relmax(G.from_nhwc(got, 64).numpy(), ref.numpy())
    assert e_ref <= 3e-3, f'halo vs torch: rel max {e_ref}'
    print({'rel_max_vs_tap': e_tap, 'rel_max_vs_torch': e_ref})


def test_convT_halo_grid_invariant():
    torch, G = _mods()
    L = G.L
    n, h, w = 2, 37, 45
    pc, xg, _, _, _ = _convT(G, n, h, w, seed=760)
    shape = (n, 2 * h, 2 * w, 64)
    outs = [_run(torch, pc, xg, shape, a_mode=L.AMODE_HALO, max_ctas=m) for m in (0, 1, 3, 7, 0)]
    for m, y in zip((1, 3, 7, 0), outs[1:]):
        assert torch.equal(outs[0], y), f'max_ctas={m} changed the transposed conv output'


def _pool_layer(G, cin, cout, n, h, w, seed):
    L, ops = G.L, G.ops
    x = G.rand(seed, n, cin, h, w, lo=-1, hi=1)
    wt = G.rand(seed + 1, cout, cin, 3, 3, lo=-0.1, hi=0.1)
    b = G.rand(seed + 2, cout, lo=-0.2, hi=0.2)
    pc = ops.PackedConv(wt.to(G.DEV), b.to(G.DEV), L.CONV_3X3, L.ACT_LRELU02)
    return pc, G.nhwc(x, ops.pad64(cin))


@pytest.mark.parametrize('cin,cout,n,h,w', [(32, 32, 4, 134, 320), (64, 64, 4, 67, 160), (32, 32, 3, 21, 13),
                                            (64, 128, 2, 33, 29)])
def test_pool_halo_bit_exact_and_grid_invariant(cin, cout, n, h, w):
    """The pooled epilogue equals maxpool2x2 of the plain conv bit for bit (odd sizes: floor pooling; cout 128:
    output channels split over two CTAs), for every grid size."""
    torch, G = _mods()
    L, ops = G.L, G.ops
    pc, xg = _pool_layer(G, cin, cout, n, h, w, seed=800 + h)
    ref = ops.maxpool2x2(pc(xg, a_mode=L.AMODE_HALO))
    shape = (n, h // 2, w // 2, pc.cout)
    for m in (0, 1, 3, 7, 0):
        got = _run(torch, pc, xg, shape, a_mode=L.AMODE_HALO, pool=True, max_ctas=m)
        assert torch.equal(got, ref), (m, float((got.float() - ref.float()).abs().max()))
