"""pytest -m gpu: the forward halo conv with its output channels split over CTAs (cout 128 / 256 from a
64-channel input) and a residual, where each CTA reads and writes one 64-channel slice of the NHWC tile
through the residual and output tensor maps."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('cout,act,h,w,n', [(128, 'none', 33, 29, 2), (256, 'lrelu', 20, 45, 1)])
def test_halo_nsplit_residual(cout, act, h, w, n):
    import torch
    assert torch.cuda.is_available(), 'pytest -m gpu needs a GPU'
    import gpu_checks
    L = gpu_checks.L
    a = {'none': L.ACT_NONE, 'lrelu': L.ACT_LRELU02}[act]
    res = gpu_checks.check_conv('tcgen05', L.AMODE_HALO, cin=64, cout=cout, h=h, w=w, n=n, act=a, residual=True,
                                seed=610 + cout)
    print(res)


def test_halo_nsplit_residual_vs_simt():
    import torch
    assert torch.cuda.is_available(), 'pytest -m gpu needs a GPU'
    import gpu_checks
    print(gpu_checks.check_conv_vs_simt(gpu_checks.L.AMODE_HALO, cin=64, cout=128, h=70, w=43, n=2))
