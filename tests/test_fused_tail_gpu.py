"""pytest -m gpu: the fused SRNet tail (last transposed conv + ReLU + conv_out + residual in one launch) at the
frame size the bench runs, where every CTA takes many tiles (so both consumer warpgroups and the wrap of their
halo rings are exercised), and its output is independent of the grid size."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('scale,accumulate', [(4, True), (4, False), (2, True)],
                         ids=['bd4_accumulate', 'bd4_lr_uint8', 'bi2_accumulate'])
def test_fused_tail_full_frame(scale, accumulate):
    import torch
    assert torch.cuda.is_available(), 'pytest -m gpu needs a GPU'
    import gpu_checks
    print(gpu_checks.check_fused_tail(scale=scale, n=2, h=268, w=640, with_lr=True, accumulate=accumulate,
                                      seed=700 + scale))


def _tail_once(up, oc, xg, lr, scale, mode, accumulate, max_ctas):
    """One fused-tail launch into fresh output buffers; returns (fp32 NCHW, uint8 NHWC)."""
    import torch
    import gpu_checks
    ops = gpu_checks.ops
    n, h, w = xg.shape[0], 2 * xg.shape[1], 2 * xg.shape[2]
    y = torch.full((n, 3, h, w), float('nan'), device=gpu_checks.DEV)
    y_u8 = torch.full((n, h, w, 3), 77, dtype=torch.uint8, device=gpu_checks.DEV)
    if accumulate:
        ops.upsample(lr, scale, mode, y=y)
        ops.fused_tail(up, oc, xg, None, scale, mode, y=y, accumulate=True, max_ctas=max_ctas)
        ops.float_to_uint8_nhwc(y, y_u8)
    else:
        ops.fused_tail(up, oc, xg, lr, scale, mode, y=y, y_u8=y_u8, max_ctas=max_ctas)
    torch.cuda.synchronize()
    assert not torch.isnan(y).any(), f'max_ctas={max_ctas}: output pixels left unwritten'
    return y, y_u8


@pytest.mark.parametrize('accumulate', [True, False], ids=['accumulate', 'lr_uint8'])
def test_fused_tail_grid_invariant(accumulate):
    """max_ctas 1 / 3 / 7 give odd tile counts per CTA and leave the second consumer idle on some CTAs; the
    result must be bit-identical to the full grid's, and a second launch into fresh buffers too."""
    import torch
    assert torch.cuda.is_available(), 'pytest -m gpu needs a GPU'
    import gpu_checks
    L, ops, rand, DEV = gpu_checks.L, gpu_checks.ops, gpu_checks.rand, gpu_checks.DEV
    n, h, w, scale, seed = 2, 268, 640, 4, 720
    x = rand(seed, n, 64, h, w, lo=-1, hi=1)
    up = ops.PackedConv(rand(seed + 1, 64, 64, 3, 3, lo=-0.08, hi=0.08).to(DEV),
                        rand(seed + 2, 64, lo=-0.2, hi=0.2).to(DEV), L.CONVT_3X3_S2, L.ACT_RELU)
    oc = ops.PackedConv(rand(seed + 3, 3, 64, 3, 3, lo=-0.08, hi=0.08).to(DEV),
                        rand(seed + 4, 3, lo=-0.2, hi=0.2).to(DEV), L.CONV_3X3, L.ACT_NONE, L.EPI_OUT_NCHW_F32)
    lr = rand(seed + 5, n, 3, 2 * h // scale, 2 * w // scale).to(DEV)
    xg = gpu_checks.nhwc(x)
    ref, ref_u8 = _tail_once(up, oc, xg, lr, scale, L.UP_BICUBIC, accumulate, 0)
    for max_ctas in (0, 1, 3, 7):
        got, got_u8 = _tail_once(up, oc, xg, lr, scale, L.UP_BICUBIC, accumulate, max_ctas)
        assert torch.equal(got, ref), (max_ctas, float((got - ref).abs().max()))
        assert torch.equal(got_u8, ref_u8), max_ctas
