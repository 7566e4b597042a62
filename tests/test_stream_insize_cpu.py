"""CPU checks of streams at any input resolution (FRNet.stream(in_size=, in_filter=)): the ValueErrors, the engine a
stream builds with and without a resize of its input, and the argument checks of tg_stream_frame_in_resample (they run
before any device work, so fake pointers never reach a launch)."""
import ctypes
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402

L = sys.modules['tecogan-pytorch_b200.lib']
ops = sys.modules['tecogan-pytorch_b200.ops']
engine = sys.modules['tecogan-pytorch_b200.engine']


class _Net:
    """What VideoStream reads of an FRNet before its first push."""
    scale = 4
    training = False

    class fnet:
        in_nc = 3

    def parameters(self):
        return iter(())


@pytest.mark.parametrize('kw', [
    dict(in_size=(540,)),                                   # types and values
    dict(in_size=(540, 960, 1)),
    dict(in_size=540),
    dict(in_size=(540.0, 960)),
    dict(in_size=(540, True)),
    dict(in_size=(0, 960)),
    dict(in_size=(540, -960)),
    dict(in_size=(269, 960)),                               # below 1/4 of 1080
    dict(in_size=(540, 479)),                               # below 1/4 of 1920
    dict(in_size=(2161, 960)),                              # above 2x
    dict(in_size=(540, 3841)),
    dict(crop=(140, 0, 800, 1920), in_size=(199, 960)),    # the ratios refer to the crop box: 800 / 4 = 200
    dict(crop=(140, 0, 800, 1920), in_size=(1601, 960)),
    dict(crop=(0, 240, 1080, 1440), in_size=(540, 2881)),
    dict(in_filter='lanczos'),                              # a filter without in_size
    dict(in_filter='nearest', in_size=(540, 960)),
    dict(in_filter=None, in_size=(540, 960)),
    dict(input='float32', in_size=(540, 960)),
    dict(in_size=(540, 960), out_size=(539, 3840)),        # out_size against 4 * in_size = 2160 x 3840
    dict(in_size=(540, 960), out_size=(4321, 3840)),
    dict(in_size=(540, 960), out_frame=(2000, 3840)),      # out_frame against 2160 x 3840
    dict(in_size=(540, 960), out_frame=(2160, 3839)),
    dict(in_size=(540, 960), out_frame=(2160, 3840), out_origin=(1, 0)),
    dict(in_size=(541, 960), out_format='nv12'),           # the output layout's grid applies to the net's picture
    dict(in_size=(540, 961), out_format='yuy2'),
])
def test_in_size_value_errors(kw):
    with pytest.raises(ValueError):
        T.VideoStream(_Net(), 2, 1080, 1920, **kw)


def test_in_size_sets_the_hr_size():
    s = T.VideoStream(_Net(), 1, 1080, 1920, input='nv12', in_size=(540, 960), out_format='nv12',
                      out_frame=(2400, 3840))
    assert s.in_size == (540, 960) and s.out_origin == (120, 0)
    # out_size within 1/4 .. 2 of 2160 x 3840, not of 4320 x 7680
    T.VideoStream(_Net(), 1, 1080, 1920, in_size=(540, 960), out_size=(1080, 1920))
    T.VideoStream(_Net(), 1, 1080, 1920, in_size=(540, 960), out_size=(4320, 7680))
    # the limits: 1/4 and 2 times the picture, on each axis, and of the crop box
    T.VideoStream(_Net(), 1, 1080, 1920, in_size=(270, 3840), in_filter='lanczos')
    T.VideoStream(_Net(), 1, 1080, 1920, crop=(140, 0, 800, 1920), in_size=(200, 480))
    T.VideoStream(_Net(), 1, 1080, 1920, crop=(140, 0, 800, 1920), in_size=(1600, 3840))
    # an odd LR size is fine for YUV input: the input layout's grid applies to the pushed frames
    T.VideoStream(_Net(), 1, 1080, 1920, input='nv12', in_size=(541, 961))


def _args(**kw):
    cls, args, kwargs = T.VideoStream(_Net(), 2, 1080, 1920, **kw)._engine_args()
    return cls, args[1:], kwargs          # args[0] is the net


@pytest.mark.parametrize('kw', [
    dict(),
    dict(input='nv12', out_format='nv12', out_size=(2160, 3840)),
    dict(crop=(140, 0, 800, 1920), out_frame=(4320, 7680)),
    dict(input='p010', scene_cut=10.0, pad_front=5),
    dict(channel_order='bgr', pad_front=3, padding_mode='replicate'),
])
def test_in_size_of_the_picture_is_the_stream_without_it(kw):
    ph, pw = kw['crop'][2:] if 'crop' in kw else (1080, 1920)
    plain = _args(**kw)
    for filt in ('bicubic', 'lanczos'):
        assert _args(in_size=(ph, pw), in_filter=filt, **kw) == plain
        assert _args(in_size=[ph, pw], in_filter=filt, **kw) == plain


def test_in_size_engine_arguments():
    cls, args, kw = _args(input='nv12', in_size=(540, 960), in_filter='lanczos', out_format='nv12')
    plain_cls, plain_args, plain_kw = _args(input='nv12', out_format='nv12')
    assert cls is plain_cls is engine.StreamEngine
    assert args == (2, 3, 540, 960, plain_args[4]) and plain_args[2:4] == (1080, 1920)
    assert kw == dict(plain_kw, in_picture=(1080, 1920), in_filter='lanczos')
    # with a crop the picture is the box, and the engine reads it out of the whole frames
    cls, args, kw = _args(crop=(140, 0, 800, 1920), in_size=(400, 960), pad_front=2)
    assert cls is engine.PaddedStreamEngine
    assert args[2:4] == (400, 960) and kw['in_picture'] == (800, 1920) and kw['crop'] == (1080, 1920, 140, 0)
    assert kw['in_filter'] == 'bicubic' and kw['pad_front'] == 2


# ------------------------------------------------------------------------------------------------- C ABI
def _fmt(layout='nv12', color='bt601', reserved=0):
    f = ops.yuv_format(layout, color)
    f.reserved = reserved
    return ctypes.byref(f)


def _win(fh, fw, top, left):
    return ctypes.byref(L.FrameWindow(fh, fw, top, left))


P = 1 << 12     # a fake, well-aligned device address: every call below is refused before it is used
INV, UNS = L.TG_OK - 1, L.TG_OK - 2


def _call(in_=P, fmt=None, bgr=0, win=None, h=16, w=16, rt=9, ct=9, n=1, c=3, hn=8, wn=8, s=4, rf=P, rw=P, cf=P,
          cw=P, reset=None, lr=P, lp=P, hp=P):
    """tg_stream_frame_in_resample with a 16 x 16 -> 8 x 8 bicubic resize (9 taps an axis) unless overridden;
    every test call below breaks at least one rule."""
    return L.load().tg_stream_frame_in_resample(in_, fmt, bgr, win, h, w, rf, rw, rt, cf, cw, ct, reset, lr, lp, hp,
                                                 n, c, hn, wn, s, None)


def test_frame_in_resample_is_exported():
    assert hasattr(L.load(), 'tg_stream_frame_in_resample')
    assert 'tg_stream_frame_in_resample' in L.exported_symbols()


def test_frame_in_resample_refuses_what_the_windowed_frame_input_refuses():
    # the refusals of tg_stream_frame_in_window / tg_stream_frame_in_yuv_window (test_stream_window_cpu)
    assert _call(win=_win(18, 16, 1, 0), fmt=_fmt('nv12')) == UNS          # off the 4:2:0 grid
    assert _call(win=_win(20, 20, 0, 3), fmt=_fmt('p010')) == UNS
    assert _call(win=_win(17, 16, 0, 0), fmt=_fmt('i420')) == UNS
    assert _call(win=_win(16, 18, 0, 1), fmt=_fmt('yuy2')) == UNS          # off the 4:2:2 grid
    assert _call(win=_win(17, 17, 1, 0), fmt=_fmt('uyvy')) == UNS
    assert _call(win=_win(16, 16, 10, 0), fmt=_fmt('nv12')) == INV         # the picture outside the frame
    assert _call(win=_win(16, 8, 0, 0)) == INV
    assert _call(win=_win(32, 32, 0, -1)) == INV
    assert _call(win=_win(0, 16, 0, 0)) == INV
    assert _call(in_=P + 1, fmt=_fmt('p010')) == INV                       # misaligned 10-bit frames
    assert _call(in_=P + 2, fmt=_fmt('yuy2')) == INV                       # misaligned packed frames
    assert _call(fmt=_fmt('nv12'), h=15) == UNS                             # odd 4:2:0 picture
    assert _call(fmt=_fmt('yuy2'), w=15) == UNS
    assert _call(fmt=_fmt('nv12', reserved=1)) == INV
    fmt = L.YuvFormat(7, 601, 0, 0)                                         # 7 is not a layout
    assert _call(fmt=ctypes.byref(fmt)) == UNS
    fmt = L.YuvFormat(L.YUV_NV12, 2020, 0, 0)
    assert _call(fmt=ctypes.byref(fmt)) == UNS
    fmt = L.YuvFormat(L.YUV_NV12, 601, 2, 0)
    assert _call(fmt=ctypes.byref(fmt)) == INV
    assert _call(lr=None) == INV                                            # null pointers
    assert _call(lp=None) == INV
    assert _call(hp=None) == INV
    assert _call(in_=None) == INV                                           # in is required here
    assert _call(lr=P + 2) == INV                                           # misaligned fp32 buffers
    assert _call(hp=P + 1) == INV
    assert _call(n=0) == INV
    assert _call(h=0) == INV
    assert _call(c=0) == INV
    assert _call(c=5) == UNS                                                # HWC: at most 4 channels
    assert _call(fmt=_fmt('nv12'), c=4) == INV                              # YUV decodes to 3
    assert _call(fmt=_fmt('i444'), bgr=1) == INV                            # bgr is for HWC frames
    assert _call(s=3) == UNS


def test_frame_in_resample_refuses_tables_that_do_not_match():
    assert _call(rf=None) == INV
    assert _call(cw=None) == INV
    assert _call(rw=P + 2) == INV
    assert _call(cf=P + 1) == INV
    assert _call(hn=0) == INV
    assert _call(wn=-8) == INV
    # ratios outside 1/4 .. 2 on either axis (16 -> 3, 16 -> 33)
    assert _call(hn=3, rt=25) == UNS
    assert _call(wn=33, ct=5) == UNS
    # tap counts: 16 -> 8 takes 9 (bicubic) or 13 (lanczos), 16 -> 32 takes 5 or 7
    assert _call(rt=13, ct=10) == INV
    assert _call(rt=8) == INV
    assert _call(ct=0) == INV
    assert _call(rt=26) == INV
    assert _call(hn=32, rt=9) == INV
    assert _call(wn=32, rt=13, ct=9) == INV
    # the tables of another size: 8 x 8 -> 16 x 16 tables (5 taps) for a 16 x 16 -> 8 x 8 resize
    assert _call(rt=5, ct=5) == INV
    for layout in ('nv12', 'i420_10', 'yuy2', 'i444'):
        assert _call(fmt=_fmt(layout), rt=13, ct=7) == INV


def test_frame_in_resample_ops_wrapper_checks_shapes():
    # the torch front end refuses CPU tensors before any call (no CPU fallback)
    import torch
    t = torch.zeros(1, 3, 8, 8)
    tabs = ops.resample_table(16, 8, 'bicubic')
    with pytest.raises(L.TecoganB200Error):
        ops.stream_frame_in_resample(torch.zeros(1, 16, 16, 3, dtype=torch.uint8), None, 'bt601', None, t, t,
                                     torch.zeros(1, 3, 32, 32), 4, tabs, tabs, (16, 16))
