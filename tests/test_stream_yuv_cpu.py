"""CPU tests (no GPU): argument checks of the streaming interface's YUV 4:2:0 formats -- FRNet.stream refuses odd
sizes, BGR with YUV input and unknown formats; VideoStream.push refuses YUV frames of the wrong shape or dtype
before any device work; tg_stream_frame_in_yuv420 and tg_rgb_u8_to_yuv420 reject null pointers and unsupported
sizes with the documented codes."""
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
P = ctypes.c_void_p(16)                        # a non-null pointer that is never dereferenced


def _net():
    return T.FRNet(3, 3, 64, 2, 'BD', 4).eval()


@pytest.mark.parametrize('kw', [
    dict(input='nv12', h=15), dict(input='i420', w=25), dict(out_format='nv12', h=17),
    dict(out_format='i420', w=9), dict(input='float32', out_format='nv12', h=3),
    dict(input='nv12', channel_order='bgr'), dict(input='i420', channel_order='bgr'),
    dict(input='yuv420p'), dict(out_format='bgr'), dict(out_format='yuyv'), dict(out_format=None),
])
def test_stream_refuses_bad_yuv_options(kw):
    h, w = kw.pop('h', 16), kw.pop('w', 24)
    with pytest.raises(ValueError):
        _net().stream(2, h, w, device='cuda', **kw)


def test_stream_refuses_yuv_for_a_net_without_three_channels():
    with pytest.raises(ValueError, match='3 colour channels'):
        T.FRNet(1, 1, 64, 2, 'BD', 4).eval().stream(1, 16, 24, device='cuda', out_format='i420')


def test_stream_accepts_every_input_with_every_out_format():
    net = _net()
    for inp in ('uint8', 'float32', 'nv12', 'i420'):
        for fmt in ('rgb', 'nv12', 'i420'):
            s = net.stream(2, 16, 24, device='cuda', input=inp, out_format=fmt)
            assert (s.input, s.out_format) == (inp, fmt)
    # odd sizes remain fine for the RGB formats
    net.stream(2, 15, 25, device='cuda', input='uint8', out_format='rgb')


@pytest.mark.parametrize('layout', ['nv12', 'i420'])
@pytest.mark.parametrize('frames,match', [
    (torch.zeros(2, 3, 24, 24, dtype=torch.float32), 'expects torch.uint8'),          # fp32 into a YUV stream
    (torch.zeros(2, 3, 16, 24, 3, dtype=torch.uint8), 'do not match'),                # RGB HWC into a YUV stream
    (torch.zeros(2, 3, 16, 24, dtype=torch.uint8), 'do not match'),                   # Y plane only
    (torch.zeros(2, 3, 24, 26, dtype=torch.uint8), 'do not match'),                   # wrong width
    (torch.zeros(3, 3, 24, 24, dtype=torch.uint8), 'do not match'),                   # wrong slot count
    (torch.zeros(2, 0, 24, 24, dtype=torch.uint8), 'do not match'),                   # no frames
    (torch.zeros(3, 24, 24, dtype=torch.uint8), 'do not match'),                      # [k,3h/2,w] needs n == 1
    (torch.zeros(2, 3, 24, 48, dtype=torch.uint8)[..., :24], 'contiguous'),           # strided view
    (np.zeros((2, 3, 24, 24), np.uint8)[..., ::-1], 'negative strides'),
])
def test_push_refuses_bad_yuv_frames(layout, frames, match):
    s = _net().stream(2, 16, 24, device='cuda', input=layout)
    with pytest.raises(T.TecoganB200Error, match=match):
        s.push(frames)


def test_push_of_a_single_slot_takes_three_dim_yuv_frames():
    s = _net().stream(1, 16, 24, device='cuda', input='nv12', out_format='i420')
    assert tuple(s._check_frames(np.zeros((4, 24, 24), np.uint8)).shape) == (1, 4, 24, 24)
    with pytest.raises(T.TecoganB200Error, match='do not match'):
        s.push(np.zeros((4, 16, 24), np.uint8))


def test_stream_frame_in_yuv420_rejects_bad_arguments_without_a_gpu():
    lib = L.load()
    f = lib.tg_stream_frame_in_yuv420
    for nv12 in (0, 1):
        assert f(None, nv12, None, P, P, P, 1, 8, 8, 4, None) == -1                  # nothing to do
        assert b'both NULL' in lib.tg_last_error_string()
        assert f(P, nv12, None, None, P, P, 1, 8, 8, 4, None) == -1                  # null lr_curr
        assert b'null' in lib.tg_last_error_string()
        assert f(None, nv12, P, P, None, P, 1, 8, 8, 4, None) == -1                  # null lr_prev
        assert f(None, nv12, P, P, P, None, 1, 8, 8, 4, None) == -1                  # null hr_prev
        for n, h, w in ((0, 8, 8), (1, 0, 8), (1, 8, -2)):
            assert f(P, nv12, P, P, P, P, n, h, w, 4, None) == -1
            assert b'bad size' in lib.tg_last_error_string()
        for h, w in ((7, 8), (8, 9), (5, 5)):
            assert f(P, nv12, P, P, P, P, 1, h, w, 4, None) == -2
            assert b'even' in lib.tg_last_error_string()
        for s in (1, 3, 8):
            assert f(P, nv12, P, P, P, P, 1, 8, 8, s, None) == -2
            assert b'scale' in lib.tg_last_error_string()
        assert f(P, nv12, P, ctypes.c_void_p(18), P, P, 1, 8, 8, 4, None) == -1      # misaligned fp32 buffer
        assert b'aligned' in lib.tg_last_error_string()


def test_rgb_u8_to_yuv420_rejects_bad_arguments_without_a_gpu():
    lib = L.load()
    f = lib.tg_rgb_u8_to_yuv420
    for nv12 in (0, 1):
        assert f(None, P, nv12, 1, 8, 8, None) == -1
        assert b'null' in lib.tg_last_error_string()
        assert f(P, None, nv12, 1, 8, 8, None) == -1
        for n, H, W in ((0, 8, 8), (1, 0, 8), (1, 8, -2)):
            assert f(P, P, nv12, n, H, W, None) == -1
            assert b'bad size' in lib.tg_last_error_string()
        for H, W in ((7, 8), (8, 9)):
            assert f(P, P, nv12, 1, H, W, None) == -2
            assert b'even' in lib.tg_last_error_string()


def test_ops_yuv_wrappers_refuse_cpu_tensors_and_bad_layouts():
    lr = torch.zeros(1, 3, 8, 8)
    with pytest.raises(T.TecoganB200Error, match='CUDA'):
        ops.stream_frame_in_yuv420(torch.zeros(1, 12, 8, dtype=torch.uint8), 'nv12', None, lr, lr.clone(),
                                   torch.zeros(1, 3, 32, 32), 4)
    with pytest.raises(T.TecoganB200Error, match='layout'):
        ops.stream_frame_in_yuv420(None, 'yuv', None, lr, lr.clone(), torch.zeros(1, 3, 32, 32), 4)
    with pytest.raises(T.TecoganB200Error, match='CUDA'):
        ops.rgb_u8_to_yuv420(torch.zeros(1, 8, 8, 3, dtype=torch.uint8), 'i420')
    with pytest.raises(T.TecoganB200Error, match='layout'):
        ops.rgb_u8_to_yuv420(torch.zeros(1, 8, 8, 3, dtype=torch.uint8), 'rgb')
