"""CPU tests (no GPU): argument checks of the streaming interface -- FRNet.stream / VideoStream.push refuse a CPU
device, wrong dtypes, layouts, sizes and reset masks before any device work, and tg_stream_frame_in rejects null
pointers and unsupported sizes with the documented codes."""
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
P = ctypes.c_void_p(16)                        # a non-null pointer that is never dereferenced


def _net():
    return T.FRNet(3, 3, 64, 2, 'BD', 4).eval()


def test_stream_refuses_cpu_device_and_bad_options():
    net = _net()
    with pytest.raises(T.TecoganB200Error):
        net.stream(2, 16, 24, device='cpu')
    with pytest.raises(ValueError):
        net.stream(2, 16, 24, device='cuda', input='float16')
    with pytest.raises(ValueError):
        net.stream(2, 16, 24, device='cuda', channel_order='yuv')
    with pytest.raises(ValueError):
        net.stream(2, 16, 24, device='cuda', input='float32', channel_order='bgr')
    with pytest.raises(ValueError):
        net.stream(0, 16, 24, device='cuda')
    net.train()
    with pytest.raises(T.TecoganB200Error, match='inference only'):
        net.stream(2, 16, 24, device='cuda')


@pytest.mark.parametrize('frames,match', [
    (torch.zeros(2, 3, 16, 24, 3, dtype=torch.float32), 'expects torch.uint8'),       # fp32 into a uint8 stream
    (torch.zeros(2, 3, 3, 16, 24, dtype=torch.uint8), 'do not match'),                # nkchw into a uint8 stream
    (torch.zeros(3, 3, 16, 24, 3, dtype=torch.uint8), 'do not match'),                # wrong slot count
    (torch.zeros(2, 3, 16, 25, 3, dtype=torch.uint8), 'do not match'),                # wrong width
    (torch.zeros(2, 0, 16, 24, 3, dtype=torch.uint8), 'do not match'),                # no frames
    (torch.zeros(3, 16, 24, 3, dtype=torch.uint8), 'do not match'),                   # [k,h,w,c] needs n == 1
    (torch.zeros(2, 3, 16, 24, 4, dtype=torch.uint8)[..., :3], 'contiguous'),          # strided view
    (np.zeros((2, 3, 16, 24, 3), np.uint8)[..., ::-1], 'negative strides'),           # cv2 [..., ::-1] view
])
def test_push_refuses_bad_uint8_frames(frames, match):
    s = _net().stream(2, 16, 24, device='cuda')
    with pytest.raises(T.TecoganB200Error, match=match):
        s.push(frames)


def test_push_refuses_bad_float_frames_reset_and_out():
    net = _net()
    s = net.stream(2, 16, 24, device='cuda', input='float32')
    with pytest.raises(T.TecoganB200Error, match='expects torch.float32'):
        s.push(torch.zeros(2, 3, 3, 16, 24, dtype=torch.float64))
    with pytest.raises(T.TecoganB200Error, match='do not match'):
        s.push(torch.zeros(2, 3, 16, 24, 3))                                   # nkhwc into a float32 stream
    good = torch.zeros(2, 3, 3, 16, 24)
    with pytest.raises(ValueError, match='reset has 3 entries'):
        s.push(good, reset=[True, False, False])
    with pytest.raises(ValueError, match='out must be'):
        s.push(good, out='cpu')
    with pytest.raises(IndexError):
        s.reset([2])
    with pytest.raises(TypeError):
        s.push([[0.0]])
    # valid arguments reach the device step, which needs a GPU and the net on it
    if not torch.cuda.is_available():
        with pytest.raises(T.TecoganB200Error):
            s.push(good)
    net.train()
    with pytest.raises(T.TecoganB200Error, match='inference only'):
        s.push(good)
    s.close()
    with pytest.raises(T.TecoganB200Error, match='closed'):
        s.push(good)


def test_stream_frame_in_rejects_bad_arguments_without_a_gpu():
    lib = L.load()
    f = lib.tg_stream_frame_in
    assert f(None, None, P, P, P, 1, 3, 8, 8, 4, 0, None) == -1                   # nothing to do
    assert b'both NULL' in lib.tg_last_error_string()
    assert f(P, None, None, P, P, 1, 3, 8, 8, 4, 0, None) == -1                   # null lr_curr
    assert b'null' in lib.tg_last_error_string()
    assert f(None, P, P, None, P, 1, 3, 8, 8, 4, 0, None) == -1                   # null lr_prev
    assert f(None, P, P, P, None, 1, 3, 8, 8, 4, 0, None) == -1                   # null hr_prev
    for n, c, h, w in ((0, 3, 8, 8), (1, 0, 8, 8), (1, 3, 0, 8), (1, 3, 8, -1)):
        assert f(P, P, P, P, P, n, c, h, w, 4, 0, None) == -1
        assert b'bad size' in lib.tg_last_error_string()
    assert f(P, P, P, P, P, 1, 5, 8, 8, 4, 0, None) == -2                         # c > 4
    assert b'channels' in lib.tg_last_error_string()
    for s in (1, 3, 8):
        assert f(P, P, P, P, P, 1, 3, 8, 8, s, 0, None) == -2
        assert b'scale' in lib.tg_last_error_string()
    assert f(P, P, ctypes.c_void_p(18), P, P, 1, 3, 8, 8, 4, 0, None) == -1       # misaligned fp32 buffer
    assert b'aligned' in lib.tg_last_error_string()


def test_ops_stream_frame_in_refuses_cpu_and_mismatched_tensors():
    ops = sys.modules['tecogan-pytorch_b200.ops']
    lr = torch.zeros(1, 3, 8, 8)
    with pytest.raises(T.TecoganB200Error, match='CUDA'):
        ops.stream_frame_in(torch.zeros(1, 8, 8, 3, dtype=torch.uint8), None, lr, lr.clone(),
                            torch.zeros(1, 3, 32, 32), 4)
