"""CPU tests (no GPU): argument checks of the streamed output's resize -- FRNet.stream(out_size=, resize_filter=)
refuses bad sizes, ratios and filters with ValueError; tg_resample_nchw_f32, tg_resample_taps and tg_resample_table
reject bad arguments with the documented codes before any device work; the ops wrappers refuse before calling."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402

L = sys.modules['tecogan-pytorch_b200.lib']
ops = sys.modules['tecogan-pytorch_b200.ops']
P = ctypes.c_void_p(16)                        # a non-null, aligned pointer that is never dereferenced
INVALID, UNSUPPORTED = -1, -2


def _net():
    return T.FRNet(3, 3, 64, 2, 'BD', 4).eval()        # 16x24 LR -> 64x96 HR


@pytest.mark.parametrize('kw', [
    dict(out_size=(48, 0)), dict(out_size=(-48, 72)), dict(out_size=(48.0, 72)), dict(out_size=(48, '72')),
    dict(out_size=48), dict(out_size=(48, 72, 3)), dict(out_size=(True, 72)), dict(out_size=[48]),
    dict(out_size=(15, 72)), dict(out_size=(129, 72)), dict(out_size=(48, 23)), dict(out_size=(48, 193)),
    dict(out_size=(49, 72), out_format='nv12'), dict(out_size=(48, 71), out_format='p010'),
    dict(out_size=(48, 72), resize_filter='bilinear'), dict(out_size=(48, 72), resize_filter='Lanczos'),
    dict(out_size=(48, 72), resize_filter=None), dict(resize_filter='lanczos'),
])
def test_stream_refuses_bad_resize_options(kw):
    with pytest.raises(ValueError):
        _net().stream(2, 16, 24, device='cuda', **kw)


def test_stream_accepts_resize_options():
    net = _net()
    for size, fmt, filt in (((48, 72), 'rgb', 'bicubic'), ((16, 24), 'nv12', 'lanczos'), ((128, 192), 'p010', 'bicubic'),
                            ([49, 71], 'rgb', 'lanczos'), ((np.int64(64), 96), 'i420_10', 'lanczos')):
        s = net.stream(2, 16, 24, device='cuda', out_format=fmt, out_size=size, resize_filter=filt)
        assert s.out_size == tuple(int(v) for v in size) and s.resize_filter == filt
    s = net.stream(2, 16, 24, device='cuda')
    assert s.out_size is None and s.resize_filter == 'bicubic'


def _call(x=P, n=1, c=3, H=64, W=96, rf=P, rw=P, rt=7, cf=P, cw=P, ct=7, Ho=48, Wo=72, y8=P, y32=None):
    return L.load().tg_resample_nchw_f32(x, n, c, H, W, rf, rw, rt, cf, cw, ct, Ho, Wo, y8, y32, None)


def _err():
    return L.load().tg_last_error_string()


def test_resample_rejects_bad_arguments_without_a_gpu():
    for kw in (dict(x=None), dict(rf=None), dict(rw=None), dict(cf=None), dict(cw=None)):
        assert _call(**kw) == INVALID
        assert b'null' in _err()
    assert _call(y8=None) == INVALID                                  # neither output
    assert b'exactly one' in _err()
    assert _call(y32=P) == INVALID                                    # both
    for kw in (dict(n=0), dict(c=0), dict(H=-1), dict(W=0), dict(Ho=0), dict(Wo=-4)):
        assert _call(**kw) == INVALID
        assert b'bad size' in _err()
    assert _call(c=5) == INVALID
    assert b'channels' in _err()
    assert _call(rt=0) == INVALID and _call(ct=-1) == INVALID
    for kw in (dict(x=ctypes.c_void_p(18)), dict(rw=ctypes.c_void_p(17)), dict(cf=ctypes.c_void_p(2)),
               dict(y8=None, y32=ctypes.c_void_p(21))):
        assert _call(**kw) == INVALID
        assert b'aligned' in _err()
    for kw in (dict(Ho=15), dict(Ho=129), dict(Wo=23), dict(Wo=193)):  # outside [1/4, 2] of 64x96
        assert _call(**kw) == UNSUPPORTED
        assert b'ratio' in _err()
    assert _call(rt=26) == UNSUPPORTED and _call(ct=26) == UNSUPPORTED
    assert b'taps' in _err()
    assert _call(n=1 << 20, H=1 << 14, W=1 << 14, Ho=1 << 15, Wo=1 << 15) == UNSUPPORTED
    assert b'grid' in _err()


def test_resample_table_rejects_bad_arguments():
    lib = L.load()
    taps = ctypes.c_int(0)
    assert lib.tg_resample_taps(64, 48, L.RESAMPLE_BICUBIC, None) == INVALID
    assert lib.tg_resample_taps(0, 48, L.RESAMPLE_BICUBIC, ctypes.byref(taps)) == INVALID
    assert lib.tg_resample_taps(64, 48, 2, ctypes.byref(taps)) == UNSUPPORTED
    assert b'filter' in _err()
    assert lib.tg_resample_taps(64, 15, L.RESAMPLE_LANCZOS3, ctypes.byref(taps)) == UNSUPPORTED
    assert lib.tg_resample_taps(64, 129, L.RESAMPLE_LANCZOS3, ctypes.byref(taps)) == UNSUPPORTED
    assert lib.tg_resample_taps(64, 16, L.RESAMPLE_LANCZOS3, ctypes.byref(taps)) == 0 and taps.value == 25
    first = (ctypes.c_int32 * 48)()
    w = (ctypes.c_float * (48 * 7))()
    assert lib.tg_resample_table(64, 48, L.RESAMPLE_BICUBIC, 7, None, w) == INVALID
    assert lib.tg_resample_table(64, 48, L.RESAMPLE_BICUBIC, 7, first, None) == INVALID
    assert lib.tg_resample_table(64, 48, L.RESAMPLE_BICUBIC, 6, first, w) == INVALID
    assert b'needs 7' in _err()
    assert lib.tg_resample_table(64, 48, L.RESAMPLE_BICUBIC, 7, first, w) == 0


def test_ops_wrappers_refuse_before_device_work():
    with pytest.raises(T.TecoganB200Error, match='filter'):
        ops.resample_table(64, 48, 'area')
    with pytest.raises(T.TecoganB200Error, match='ratio'):
        ops.resample_table(64, 15)
    rows, cols = ops.resample_table(64, 48), ops.resample_table(96, 72)
    with pytest.raises(T.TecoganB200Error, match='CUDA'):
        ops.resample(torch.zeros(1, 3, 64, 96), rows, cols)
