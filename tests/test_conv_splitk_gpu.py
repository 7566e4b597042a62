"""pytest -m gpu: forward 3x3 convs with 128 / 256 input channels on the split-K path (the K chunks split over a
thread-block cluster, partials reduced through distributed shared memory), pooled or not.  Every output buffer is
filled with NaN first, so each check also shows that every output pixel was written."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

# the six FNet layers of the 4x BD step (4 frames) and ragged sizes: h < 16, h = 33, w not a multiple of 8, n = 1-3
SHAPES = [
    (128, 128, 4, 33, 80),     # encoder3[2] (pooled in the network)
    (128, 256, 4, 16, 40),     # decoder1[0]
    (256, 256, 4, 16, 40),     # decoder1[2]
    (256, 128, 4, 32, 80),     # decoder2[0]
    (128, 128, 4, 32, 80),     # decoder2[2]
    (128, 64, 4, 64, 160),     # decoder3[0]
    (128, 128, 3, 7, 13),
    (256, 128, 1, 33, 21),
    (256, 256, 2, 9, 30),
    (128, 64, 2, 33, 45),
    (256, 64, 1, 5, 3),
]


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


def _layer(G, cin, cout, n, h, w, seed):
    L, ops = G.L, G.ops
    x = G.rand(seed, n, cin, h, w, lo=-1, hi=1)
    bound = 1.5 / np.sqrt(9 * cin)
    wt = G.rand(seed + 1, cout, cin, 3, 3, lo=-bound, hi=bound)
    b = G.rand(seed + 2, cout, lo=-0.2, hi=0.2)
    pc = ops.PackedConv(wt.to(G.DEV), b.to(G.DEV), L.CONV_3X3, L.ACT_LRELU02)
    return pc, G.nhwc(x, cin), x, wt, b


@pytest.mark.parametrize('cin,cout,n,h,w', SHAPES)
def test_splitk_vs_tap_and_torch(cin, cout, n, h, w):
    """Split-K against the tap-mode kernel on the same packed weights (the chunk partials are added last, so
    the fp32 sums differ in order) and against torch fp32 conv2d + LeakyReLU(0.2) on the fp16-rounded operands."""
    torch, G = _mods()
    L = G.L
    pc, xg, x, wt, b = _layer(G, cin, cout, n, h, w, seed=900 + cin + cout + h)
    shape = (n, h, w, cout)
    got = _run(torch, pc, xg, shape, a_mode=L.AMODE_AUTO)
    tap = _run(torch, pc, xg, shape, a_mode=L.AMODE_TAP)
    e_tap = float((got.float() - tap.float()).abs().max() / tap.float().abs().max())
    assert e_tap <= 2e-3, f'split-K vs tap: rel max {e_tap}'
    ref = G._conv_ref(x, wt, b, L.CONV_3X3, L.ACT_LRELU02)
    e_ref = G.relmax(G.from_nhwc(got, cout).numpy(), ref.numpy())
    assert e_ref <= 3e-3, f'split-K vs torch: rel max {e_ref}'
    print({'rel_max_vs_tap': e_tap, 'rel_max_vs_torch': e_ref})


@pytest.mark.parametrize('cin,cout,n,h,w', [(128, 128, 2, 37, 45), (256, 256, 1, 16, 40), (256, 128, 3, 21, 27)])
def test_splitk_grid_invariant(cin, cout, n, h, w):
    """The partials are summed in rank order whichever CTA owns an output channel: the output is the same bits
    for every grid size (max_ctas 1 / 3 / 7 round up to one cluster per N slice) and on repeated runs."""
    torch, G = _mods()
    L = G.L
    pc, xg, _, _, _ = _layer(G, cin, cout, n, h, w, seed=950 + cin)
    shape = (n, h, w, cout)
    outs = [_run(torch, pc, xg, shape, a_mode=L.AMODE_AUTO, max_ctas=m) for m in (0, 1, 3, 7, 0)]
    for m, y in zip((1, 3, 7, 0), outs[1:]):
        assert torch.equal(outs[0], y), f'max_ctas={m} changed the split-K output'


@pytest.mark.parametrize('cin,cout,n,h,w', [(128, 128, 4, 33, 80), (256, 128, 3, 21, 13), (128, 256, 2, 9, 17),
                                            (256, 64, 1, 4, 4)])
def test_splitk_pool_bit_exact_and_grid_invariant(cin, cout, n, h, w):
    """The pooled split-K epilogue equals maxpool2x2 of the unpooled split-K output bit for bit (odd sizes:
    floor pooling), for every grid size."""
    torch, G = _mods()
    L, ops = G.L, G.ops
    pc, xg, _, _, _ = _layer(G, cin, cout, n, h, w, seed=980 + h)
    ref = ops.maxpool2x2(_run(torch, pc, xg, (n, h, w, cout), a_mode=L.AMODE_AUTO))
    shape = (n, h // 2, w // 2, cout)
    for m in (0, 1, 3, 7, 0):
        got = _run(torch, pc, xg, shape, a_mode=L.AMODE_AUTO, pool=True, max_ctas=m)
        assert torch.equal(got, ref), (m, float((got.float() - ref.float()).abs().max()))
