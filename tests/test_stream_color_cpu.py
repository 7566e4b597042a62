"""CPU tests (no GPU): argument checks of the streaming interface's colours and 10-bit layouts -- FRNet.stream refuses
unknown colours, a colour on an RGB side and odd sizes; VideoStream.push refuses uint8 frames into a 10-bit stream and
uint16 frames into an 8-bit one before any device work; tg_stream_frame_in_yuv, tg_rgb_to_yuv and tg_yuv_coefficients
reject bad arguments with the documented codes; the device colour table is oracle/yuv_color.py's."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402
from oracle import yuv_color as C              # noqa: E402

L = sys.modules['tecogan-pytorch_b200.lib']
ops = sys.modules['tecogan-pytorch_b200.ops']
P = ctypes.c_void_p(16)                        # a non-null pointer that is never dereferenced


def _net():
    return T.FRNet(3, 3, 64, 2, 'BD', 4).eval()


def _fmt(layout=L.YUV_P010, matrix=709, full=0, reserved=0):
    return ctypes.byref(L.YuvFormat(layout, matrix, full, reserved))


@pytest.mark.parametrize('layout', C.LAYOUTS)
@pytest.mark.parametrize('color', C.COLORS)
def test_device_table_is_the_oracle(layout, color):
    assert ops.yuv_coefficients(layout, color) == C.coefficients(color, C.depth_of(layout))


@pytest.mark.parametrize('kw', [
    dict(input='p010', in_color='bt2020'), dict(out_format='nv12', out_color='BT709'),
    dict(input='nv12', in_color=None), dict(input='i420_10', in_color='709'),
    dict(in_color='bt709'), dict(input='float32', in_color='bt601-full'),              # colour on an RGB side
    dict(out_color='bt709'), dict(input='p010', out_color='bt709-full'),
    dict(input='p010', h=15), dict(out_format='i420_10', w=9),
    dict(input='p010', channel_order='bgr'), dict(input='p016'), dict(out_format='yuv420p10le'),
    dict(input='yuv420p'), dict(out_format='yuyv'), dict(out_format='bgr'),
])
def test_stream_refuses_bad_color_options(kw):
    h, w = kw.pop('h', 16), kw.pop('w', 24)
    with pytest.raises(ValueError):
        _net().stream(2, h, w, device='cuda', **kw)


def test_stream_accepts_every_layout_and_colour_pair():
    net = _net()
    ins = ('uint8', 'float32', *C.LAYOUTS)
    for inp in ins:
        for fmt in ('rgb', *C.LAYOUTS):
            for ic in (C.COLORS if inp in C.LAYOUTS else ('bt601',)):
                oc = 'bt709' if fmt in C.LAYOUTS else 'bt601'
                s = net.stream(2, 16, 24, device='cuda', input=inp, out_format=fmt, in_color=ic, out_color=oc)
                assert (s.input, s.out_format, s.in_color, s.out_color) == (inp, fmt, ic, oc)


@pytest.mark.parametrize('inp,frames,match', [
    ('p010', np.zeros((2, 3, 24, 24), np.uint8), 'expects torch.uint16'),           # uint8 into a 10-bit stream
    ('i420_10', torch.zeros(2, 3, 24, 24, dtype=torch.uint8), 'expects torch.uint16'),
    ('nv12', np.zeros((2, 3, 24, 24), np.uint16), 'expects torch.uint8'),            # uint16 into an 8-bit stream
    ('i420', torch.zeros(2, 3, 24, 24, dtype=torch.uint16), 'expects torch.uint8'),
    ('p010', np.zeros((2, 3, 16, 24), np.uint16), 'do not match'),                   # Y plane only
    ('p010', np.zeros((3, 3, 24, 24), np.uint16), 'do not match'),                   # wrong slot count
    ('i420_10', np.zeros((3, 24, 24), np.uint16), 'do not match'),                   # [k,3h/2,w] needs n == 1
    ('p010', torch.zeros(2, 3, 24, 48, dtype=torch.uint16)[..., :24], 'contiguous'),
])
def test_push_refuses_bad_10bit_frames(inp, frames, match):
    s = _net().stream(2, 16, 24, device='cuda', input=inp, in_color='bt709')
    with pytest.raises(T.TecoganB200Error, match=match):
        s.push(frames)


def test_push_of_a_single_slot_takes_three_dim_10bit_frames():
    s = _net().stream(1, 16, 24, device='cuda', input='p010', out_format='p010', in_color='bt709',
                      out_color='bt709')
    got = s._check_frames(np.zeros((4, 24, 24), np.uint16))
    assert tuple(got.shape) == (1, 4, 24, 24) and got.dtype == torch.uint16


def test_stream_frame_in_yuv_rejects_bad_arguments_without_a_gpu():
    lib = L.load()
    f = lib.tg_stream_frame_in_yuv
    assert f(P, None, None, P, P, P, 1, 8, 8, 4, None) == -1                          # null format
    assert f(P, _fmt(reserved=1), None, P, P, P, 1, 8, 8, 4, None) == -1
    assert b'reserved' in lib.tg_last_error_string()
    assert f(P, _fmt(full=2), None, P, P, P, 1, 8, 8, 4, None) == -1
    assert f(P, _fmt(matrix=2020), None, P, P, P, 1, 8, 8, 4, None) == -2
    assert b'matrix' in lib.tg_last_error_string()
    assert f(P, _fmt(layout=7), None, P, P, P, 1, 8, 8, 4, None) == -2
    assert b'layout' in lib.tg_last_error_string()
    for layout in (L.YUV_NV12, L.YUV_I420, L.YUV_P010, L.YUV_I420_10):
        fm = _fmt(layout)
        assert f(None, fm, None, P, P, P, 1, 8, 8, 4, None) == -1                     # nothing to do
        assert b'both NULL' in lib.tg_last_error_string()
        assert f(P, fm, None, None, P, P, 1, 8, 8, 4, None) == -1                     # null lr_curr
        for n, h, w in ((0, 8, 8), (1, 0, 8), (1, 8, -2)):
            assert f(P, fm, P, P, P, P, n, h, w, 4, None) == -1
            assert b'bad size' in lib.tg_last_error_string()
        for h, w in ((7, 8), (8, 9)):
            assert f(P, fm, P, P, P, P, 1, h, w, 4, None) == -2
            assert b'even' in lib.tg_last_error_string()
        assert f(P, fm, P, P, P, P, 1, 8, 8, 3, None) == -2
        assert b'scale' in lib.tg_last_error_string()
    assert f(ctypes.c_void_p(17), _fmt(L.YUV_P010), P, P, P, P, 1, 8, 8, 4, None) == -1    # odd address, words
    assert b'aligned' in lib.tg_last_error_string()


def test_rgb_to_yuv_rejects_bad_arguments_without_a_gpu():
    lib = L.load()
    f = lib.tg_rgb_to_yuv
    assert f(P, None, P, None, 1, 8, 8, None) == -1
    assert f(P, None, P, _fmt(L.YUV_NV12, reserved=3), 1, 8, 8, None) == -1
    assert f(P, None, P, _fmt(L.YUV_NV12, matrix=0), 1, 8, 8, None) == -2
    assert f(P, None, P, _fmt(layout=-1), 1, 8, 8, None) == -2
    for layout in (L.YUV_NV12, L.YUV_I420):                   # 8 bit: rgb_u8 only
        assert f(None, P, P, _fmt(layout), 1, 8, 8, None) == -1
        assert b'rgb_u8' in lib.tg_last_error_string()
        assert f(P, P, P, _fmt(layout), 1, 8, 8, None) == -1
        assert f(P, None, None, _fmt(layout), 1, 8, 8, None) == -1
        assert f(P, None, P, _fmt(layout), 1, 7, 8, None) == -2
        assert f(P, None, P, _fmt(layout), 0, 8, 8, None) == -1
    for layout in (L.YUV_P010, L.YUV_I420_10):               # 10 bit: rgb_f32 only
        assert f(P, None, P, _fmt(layout), 1, 8, 8, None) == -1
        assert b'rgb_f32' in lib.tg_last_error_string()
        assert f(P, P, P, _fmt(layout), 1, 8, 8, None) == -1
        assert f(None, ctypes.c_void_p(18), P, _fmt(layout), 1, 8, 8, None) == -1   # misaligned fp32
        assert f(None, P, ctypes.c_void_p(17), _fmt(layout), 1, 8, 8, None) == -1  # misaligned words
        assert f(None, P, P, _fmt(layout), 1, 8, 10 - 1, None) == -2
        assert b'even' in lib.tg_last_error_string()


def test_yuv_coefficients_rejects_bad_arguments():
    lib = L.load()
    out = (ctypes.c_int32 * 16)()
    assert lib.tg_yuv_coefficients(None, out) == -1
    assert lib.tg_yuv_coefficients(_fmt(), None) == -1
    assert lib.tg_yuv_coefficients(_fmt(matrix=2020), out) == -2
    assert lib.tg_yuv_coefficients(_fmt(reserved=1), out) == -1


def test_ops_wrappers_refuse_before_device_work():
    lr = torch.zeros(1, 3, 8, 8)
    hr = torch.zeros(1, 3, 32, 32)
    with pytest.raises(T.TecoganB200Error, match='colour'):
        ops.stream_frame_in_yuv(None, 'p010', 'bt2020', None, lr, lr.clone(), hr, 4)
    with pytest.raises(T.TecoganB200Error, match='layout'):
        ops.stream_frame_in_yuv(None, 'p016', 'bt709', None, lr, lr.clone(), hr, 4)
    with pytest.raises(T.TecoganB200Error, match='CUDA'):
        ops.stream_frame_in_yuv(torch.zeros(1, 12, 8, dtype=torch.uint16), 'p010', 'bt709', None, lr, lr.clone(),
                                hr, 4)
    with pytest.raises(T.TecoganB200Error, match='rgb_f32'):
        ops.rgb_to_yuv('p010', 'bt709', rgb_u8=torch.zeros(1, 8, 8, 3, dtype=torch.uint8))
    with pytest.raises(T.TecoganB200Error, match='rgb_u8'):
        ops.rgb_to_yuv('nv12', 'bt709', rgb_f32=torch.zeros(1, 3, 8, 8))
    with pytest.raises(T.TecoganB200Error, match='CUDA'):
        ops.rgb_to_yuv('i420_10', 'bt709-full', rgb_f32=torch.zeros(1, 3, 8, 8))
