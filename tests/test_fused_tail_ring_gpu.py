"""pytest -m gpu: the fused SRNet tail at small frames whose tile counts hit the edges of its pipelines: one tile,
two tiles (in one image and across two), and tile counts that are not a multiple of the three-stage halo ring or of
the grid.  The transposed-conv warpgroup writes parity a of a tile while a conv_out warpgroup still reads parity
a - 1, carries a tile's last parity into the next tile, and hands alternate tiles to two conv_out warpgroups, so
the first and last tiles of a CTA, CTAs with one tile (one conv_out warpgroup idle) and odd tile counts are the
cases where a ring index or mbarrier phase would go wrong."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

# (n, h, w) of the transposed conv's input; tiles = n * ceil((2h + 1) / 30) * ceil((2w + 1) / 14).  2h and 2w are
# multiples of 4, as the lr mode's bicubic x4 upsample needs.
SHAPES = {
    '1tile': (1, 8, 6),
    '2tiles': (1, 8, 12),
    '2images': (2, 8, 6),
    '7tiles': (7, 8, 6),
    '8tiles': (1, 20, 26),
    '16tiles': (1, 50, 26),
}


@pytest.mark.parametrize('accumulate', [True, False], ids=['accumulate', 'lr_uint8'])
@pytest.mark.parametrize('shape', list(SHAPES.values()), ids=list(SHAPES))
def test_fused_tail_small_frames(shape, accumulate):
    """Against the same stages run as separate kernels and against torch on the CPU."""
    import torch
    assert torch.cuda.is_available(), 'pytest -m gpu needs a GPU'
    import gpu_checks
    n, h, w = shape
    print(gpu_checks.check_fused_tail(scale=4, n=n, h=h, w=w, with_lr=True, accumulate=accumulate, seed=760 + h + w))


@pytest.mark.parametrize('accumulate', [True, False], ids=['accumulate', 'lr_uint8'])
@pytest.mark.parametrize('shape', list(SHAPES.values()), ids=list(SHAPES))
def test_fused_tail_grid_invariant_small(shape, accumulate):
    """max_ctas 1 / 3 / 7 put 1..16 tiles on a CTA; the result must be bit-identical to the full grid's."""
    import torch
    assert torch.cuda.is_available(), 'pytest -m gpu needs a GPU'
    import gpu_checks
    from test_fused_tail_gpu import _tail_once
    L, ops, rand, DEV = gpu_checks.L, gpu_checks.ops, gpu_checks.rand, gpu_checks.DEV
    (n, h, w), scale, seed = shape, 4, 780
    x = rand(seed, n, 64, h, w, lo=-1, hi=1)
    up = ops.PackedConv(rand(seed + 1, 64, 64, 3, 3, lo=-0.08, hi=0.08).to(DEV),
                        rand(seed + 2, 64, lo=-0.2, hi=0.2).to(DEV), L.CONVT_3X3_S2, L.ACT_RELU)
    oc = ops.PackedConv(rand(seed + 3, 3, 64, 3, 3, lo=-0.08, hi=0.08).to(DEV),
                        rand(seed + 4, 3, lo=-0.2, hi=0.2).to(DEV), L.CONV_3X3, L.ACT_NONE, L.EPI_OUT_NCHW_F32)
    lr = rand(seed + 5, n, 3, 2 * h // scale, 2 * w // scale).to(DEV)
    xg = gpu_checks.nhwc(x)
    ref, ref_u8 = _tail_once(up, oc, xg, lr, scale, L.UP_BICUBIC, accumulate, 0)
    for max_ctas in (1, 3, 7):
        got, got_u8 = _tail_once(up, oc, xg, lr, scale, L.UP_BICUBIC, accumulate, max_ctas)
        assert torch.equal(got, ref), (max_ctas, float((got - ref).abs().max()))
        assert torch.equal(got_u8, ref_u8), max_ctas
