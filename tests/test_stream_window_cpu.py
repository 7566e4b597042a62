"""CPU checks of picture windows in streamed video (crop / letterbox / pillarbox): the oracle/frame_window.py
specification against the YUV oracles, the black words of every format, tecogan_b200.fit_size, the detect_bars rule,
the ValueErrors of FRNet.stream(crop=, out_frame=, out_origin=), and the new C ABI entry points' error codes (their
argument checks run before any device work)."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402
from oracle import frame_window as FW          # noqa: E402
from oracle import yuv_422_444 as Y            # noqa: E402

L = sys.modules['tecogan-pytorch_b200.lib']
ops = sys.modules['tecogan-pytorch_b200.ops']
COLORS = Y.COLORS


def _frames(layout, h, w, seed):
    rng = np.random.default_rng(seed)
    if layout == 'rgb':
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    top = 1024 if Y.depth_of(layout) == 10 else 256
    v = rng.integers(0, top, Y.frame_shape(layout, h, w)).astype(Y.word_dtype(layout))
    return (v << 6).astype(np.uint16) if layout == 'p010' else v


def _decode(frame, layout, color):
    return frame if layout == 'rgb' else Y.yuv_to_rgb(frame, layout, color)


@pytest.mark.parametrize('layout', FW.LAYOUTS)
@pytest.mark.parametrize('color', COLORS)
def test_windowed_decode_is_the_cropped_frames_decode(layout, color):
    if layout == 'rgb' and color != 'bt601':
        pytest.skip('RGB frames have no colour')
    gy, gx = FW.grid(layout)
    Hf, Wf = 12, 20
    frame = _frames(layout, Hf, Wf, 3)
    full = _decode(frame, layout, color)
    for top, left, h, w in ((0, 0, Hf, Wf), (2, 4, 6, 8), (Hf - 4, Wf - 6, 4, 6), (0, Wf - 2, 2, 2),
                            (gy, gx, 2 * gy, 2 * gx)):
        pic = FW.crop_words(frame, layout, top, left, h, w)
        assert pic.shape == FW.frame_shape(layout, h, w)
        # nearest chroma on the chroma grid: the picture's decode is the frame's decode cropped
        np.testing.assert_array_equal(_decode(pic, layout, color), full[top:top + h, left:left + w])
        # and placing it back into a frame of the same size restores its words there
        back = FW.place_words(pic, layout, color, Hf, Wf, top, left)
        np.testing.assert_array_equal(FW.crop_words(back, layout, top, left, h, w), pic)
    if gy == 2:
        with pytest.raises(ValueError):
            FW.crop_words(frame, layout, 1, 0, 2, 2)
    if gx == 2:
        with pytest.raises(ValueError):
            FW.crop_words(frame, layout, 0, 1, 2, 2)


@pytest.mark.parametrize('layout', Y.ALL_LAYOUTS)
@pytest.mark.parametrize('color', COLORS)
def test_black_words_decode_to_black(layout, color):
    d = Y.depth_of(layout)
    yb, cb = FW.black_words(layout, color)
    sh = 6 if layout == 'p010' else 0
    assert cb == (128 << (d - 8)) << sh
    assert yb == ((0 if color.endswith('-full') else 16 << (d - 8)) << sh)
    want = {('bt601', 8): (16, 128), ('bt601-full', 8): (0, 128), ('bt601', 10): (64, 512),
            ('bt601-full', 10): (0, 512)}[(color.replace('709', '601'), d)]
    assert (yb >> sh, cb >> sh) == want
    frame = FW.black_frame(layout, color, 4, 6)
    assert frame.shape == Y.frame_shape(layout, 4, 6) and frame.dtype == Y.word_dtype(layout)
    assert not _decode(frame, layout, color).any()


def test_rgb_black_is_zero():
    assert FW.black_words('rgb') == (0, 0)
    assert not FW.black_frame('rgb', 'bt601', 3, 5).any()


def test_place_words_pads_with_black():
    pic = _frames('nv12', 4, 6, 1)
    out = FW.place_words(pic, 'nv12', 'bt601', 8, 10, 2, 4)
    y, u, v = Y.split_planes(out, 'nv12')
    mask = np.zeros((8, 10), bool)
    mask[2:6, 4:10] = True
    assert (y[~mask] == 16).all()
    cm = mask[::2, ::2]
    assert (u[~cm] == 128).all() and (v[~cm] == 128).all()


# ------------------------------------------------------------------------------------------------- fit_size
@pytest.mark.parametrize('picture, frame, sar, fmt, want', [
    ((536, 1280), (720, 1280), (1, 1), 'rgb', (536, 1280)),      # 2.39:1 into 16:9: letterbox, full width
    ((480, 640), (720, 1280), (1, 1), 'rgb', (720, 960)),         # 4:3 into 16:9: pillarbox
    ((480, 640), (720, 1280), (1, 1), 'nv12', (720, 960)),
    ((480, 720), (1080, 1920), (8, 9), 'rgb', (960, 1280)),       # anamorphic 4:3 DVD, height capped at 2x
    ((480, 720), (720, 1280), (32, 27), 'rgb', (720, 1280)),      # anamorphic 16:9 DVD fills a 16:9 frame
    ((480, 720), (720, 1280), (8, 9), 'rgb', (720, 960)),
    ((135, 241), (720, 1280), (1, 1), 'rgb', (270, 482)),         # 2x cap on both sides
    ((134, 321), (720, 1280), (1, 1), 'nv12', (268, 642)),        # rounded down to the 4:2:0 grid
    ((101, 101), (150, 303), (1, 1), 'yuy2', (150, 150)),
])
def test_fit_size(picture, frame, sar, fmt, want):
    got = T.fit_size(picture, frame, sar=sar, out_format=fmt)
    assert got == want
    h, w = got
    assert h <= frame[0] and w <= frame[1]
    assert ops.resample_ratio_ok(picture[0], h) and ops.resample_ratio_ok(picture[1], w)
    gy, gx = FW.grid(fmt)
    assert h % gy == 0 and w % gx == 0


def test_fit_size_refuses():
    with pytest.raises(ValueError):
        T.fit_size((1000, 1000), (100, 1000))     # 1/10 of the picture: below the resize's 1/4
    for bad in ((0, 5), (5,), (1.5, 2), None):
        with pytest.raises(ValueError):
            T.fit_size(bad, (10, 10))
    with pytest.raises(ValueError):
        T.fit_size((10, 10), (10, 10), out_format='yuv')


# ------------------------------------------------------------------------------------------------- detect_bars rule
def _letterboxed(k, h, w, box, seed, noise=10):
    rng = np.random.default_rng(seed)
    f = rng.integers(0, noise + 1, (k, h, w, 3), dtype=np.uint8)      # bars: noise below the limit
    t, l, ch, cw = box
    f[:, t:t + ch, l:l + cw] = rng.integers(40, 256, (k, ch, cw, 3), dtype=np.uint8)
    return f


def test_detect_bars_rule_letterbox_and_pillarbox():
    f = _letterboxed(3, 40, 64, (6, 0, 28, 64), 0)
    assert FW.detect_bars(f, 'rgb') == (6, 0, 28, 64)
    f = _letterboxed(2, 40, 64, (0, 9, 40, 45), 1)
    assert FW.detect_bars(f, 'rgb') == (0, 9, 40, 45)
    # 4:2:0 rounds inward: rows [7, 34) -> [8, 34), columns [9, 54) -> [10, 54)
    f = _letterboxed(2, 40, 64, (7, 9, 27, 45), 2)
    l8 = FW.luma8(f, 'rgb')
    assert FW.detect_bars(l8[..., None].repeat(3, -1).astype(np.uint8), 'rgb') == (7, 9, 27, 45)
    y = np.zeros((2, 60, 64), np.uint8)
    y[:, :40] = l8
    y[:, 40:] = 128
    assert FW.detect_bars(y, 'nv12') == (8, 10, 26, 44)


def test_detect_bars_rule_logo_in_a_bar_and_black_frames():
    f = _letterboxed(2, 40, 64, (8, 0, 24, 64), 3)
    # a bright logo in the top bar of one frame: 6 x 8 pixels of 255 give row means of 8 * 255 / 64 = 31.9 > 24
    f[1, 2:8, 50:58] = 255
    assert FW.detect_bars(f, 'rgb') == (2, 0, 30, 64)
    # a dimmer logo (row mean 8 * 150 / 64 = 18.75) stays below the limit
    f[1, 2:8, 50:58] = 150
    assert FW.detect_bars(f, 'rgb') == (8, 0, 24, 64)
    assert FW.detect_bars(np.zeros((2, 40, 64, 3), np.uint8), 'rgb') == (0, 0, 40, 64)
    # noise that reaches the limit in the mean is picture
    assert FW.detect_bars(np.full((1, 40, 64, 3), 25, np.uint8), 'rgb') == (0, 0, 40, 64)
    assert FW.detect_bars(np.full((1, 40, 64, 3), 24, np.uint8), 'rgb') == (0, 0, 40, 64)


def test_detect_bars_package_rule_matches_oracle():
    engine = sys.modules['tecogan-pytorch_b200.engine']
    for seed, box, layout in ((0, (7, 9, 27, 45), 'rgb'), (1, (7, 9, 27, 45), 'nv12'), (2, (3, 5, 30, 41), 'yuy2')):
        f = _letterboxed(2, 40, 64, box, seed)
        l8 = FW.luma8(f, 'rgb')
        rows, cols = l8.sum(-1), l8.sum(-2)
        got = engine.bars_box((rows > 24 * 64).any(0), (cols > 24 * 40).any(0), layout)
        gy, gx = FW.grid(layout)
        y = np.zeros((2, *Y.frame_shape(layout, 40, 64)) if layout != 'rgb' else f.shape, np.uint8)
        if layout == 'rgb':
            y = f
        elif layout == 'yuy2':
            y[..., 0::2] = l8
        else:
            y[:, :40] = l8
        assert got == FW.detect_bars(y, layout)


def test_luma8_10_bit_and_bgr():
    f = np.zeros((1, 6, 4), np.uint16)
    f[0, :4] = 1023 << 6
    assert (FW.luma8(f, 'p010')[0] == 255).all()
    g = np.zeros((1, 2, 2, 3), np.uint8)
    g[..., 2] = 255
    assert FW.luma8(g, 'rgb')[0, 0, 0] == (3735 * 255 + 16384) >> 15
    assert FW.luma8(g, 'rgb', 'bgr')[0, 0, 0] == (9798 * 255 + 16384) >> 15


# ------------------------------------------------------------------------------------------------- ValueErrors
class _Net:
    """What VideoStream reads of an FRNet before its first push."""
    scale = 4
    training = False

    class fnet:
        in_nc = 3

    def parameters(self):
        return iter(())


@pytest.mark.parametrize('kw', [
    dict(crop=(0, 0, 181, 320)),                    # outside the frame
    dict(crop=(-2, 0, 100, 320)),
    dict(crop=(0, 0, 0, 320)),
    dict(crop=(22, 0, 134)),
    dict(crop=(22.0, 0, 134, 320)),
    dict(crop=(21, 0, 134, 320), input='nv12'),     # odd top for 4:2:0
    dict(crop=(22, 0, 133, 320), input='p010'),
    dict(crop=(22, 1, 134, 318), input='i420'),
    dict(crop=(22, 0, 134, 319), input='i420_10'),
    dict(crop=(22, 1, 134, 318), input='yuy2'),     # odd left / cw for 4:2:2
    dict(crop=(22, 0, 134, 319), input='uyvy'),
    dict(crop=(22, 0, 134, 320), input='float32'),
    dict(out_frame=(500, 1280)),                    # the 720x1280 picture does not fit
    dict(crop=(22, 0, 134, 320), out_frame=(535, 1280)),
    dict(out_frame=(720, 1280), out_origin=(1, 0)),
    dict(out_frame=(800, 1280), out_origin=(81, 0), out_format='nv12'),   # odd origin for 4:2:0
    dict(out_frame=(800, 1281), out_format='nv12'),
    dict(out_frame=(800, 1282), out_origin=(0, 1), out_format='yuy2'),
    dict(out_frame=(800, 1281), out_format='uyvy'),
    dict(out_origin=(0, 0)),                        # an origin without a frame
    dict(out_frame=(720,)),
    dict(out_frame=(720, 1280), out_origin=(0, -1)),
    dict(crop=(22, 0, 134, 320), out_size=(2000, 1280)),   # ratio limits apply to the picture
])
def test_stream_window_value_errors(kw):
    with pytest.raises(ValueError):
        T.VideoStream(_Net(), 2, 180, 320, **kw)


def test_output_layout_grid_applies_to_the_picture():
    # the picture the net runs on decides the output layout's grid: an odd frame height is fine once cropped
    s = T.VideoStream(_Net(), 1, 181, 320, crop=(0, 0, 180, 320), out_format='nv12')
    assert s.crop == (0, 0, 180, 320)
    T.VideoStream(_Net(), 1, 180, 321, crop=(0, 0, 180, 320), out_format='yuy2')
    for kw in (dict(out_format='nv12'), dict(crop=(0, 0, 181, 320), out_format='nv12'),
               dict(crop=(0, 0, 180, 321), out_format='uyvy')):
        with pytest.raises(ValueError):
            T.VideoStream(_Net(), 1, 181, 321, **kw)
    with pytest.raises(ValueError):           # the input layout still checks the pushed frames
        T.VideoStream(_Net(), 1, 181, 320, input='nv12', crop=(0, 0, 180, 320))


def test_stream_window_defaults():
    s = T.VideoStream(_Net(), 2, 180, 320, crop=(22, 0, 134, 320), out_frame=(720, 1280))
    assert s.crop == (22, 0, 134, 320) and s.out_frame == (720, 1280) and s.out_origin == (92, 0)
    s = T.VideoStream(_Net(), 1, 180, 320, out_format='nv12', out_frame=(722, 1286), out_size=(356, 640))
    assert s.out_origin == (182, 322)
    s = T.VideoStream(_Net(), 1, 180, 320, out_format='yuy2', out_frame=(723, 1283 + 1), out_size=(357, 640))
    assert s.out_origin == (183, 322)
    s = T.VideoStream(_Net(), 1, 180, 320, crop=(22, 0, 134, 320), out_size=(268, 640))   # 1/2 of 536 x 1280
    assert s.out_size == (268, 640)


# ------------------------------------------------------------------------------------------------- C ABI
def _fmt(layout='nv12', color='bt601'):
    return ctypes.byref(ops.yuv_format(layout, color))


def _win(fh, fw, top, left):
    return ctypes.byref(L.FrameWindow(fh, fw, top, left))


P = 1 << 12     # a fake, well-aligned device address: every call below is refused before it is used


def test_window_entry_points_are_exported():
    lib = L.load()
    for name in ('tg_stream_frame_in_window', 'tg_stream_frame_in_yuv_window', 'tg_rgb_to_yuv_window',
                 'tg_float_to_uint8_nhwc_window', 'tg_resample_nchw_f32_window', 'tg_fill_black',
                 'tg_luma_line_sums'):
        assert hasattr(lib, name)
    assert ctypes.sizeof(L.FrameWindow) == 16
    assert lib.tg_version() == 2


def test_window_error_codes():
    lib = L.load()
    INV, UNS = L.TG_OK - 1, L.TG_OK - 2
    s = None
    # frame in, HWC: null window, picture outside the frame
    assert lib.tg_stream_frame_in_window(P, None, None, P, P, P, 1, 3, 8, 8, 4, 0, s) == INV
    assert lib.tg_stream_frame_in_window(P, _win(8, 8, 1, 0), None, P, P, P, 1, 3, 8, 8, 4, 0, s) == INV
    assert lib.tg_stream_frame_in_window(P, _win(16, 8, 0, -1), None, P, P, P, 1, 3, 8, 8, 4, 0, s) == INV
    assert lib.tg_stream_frame_in_window(P, _win(0, 8, 0, 0), None, P, P, P, 1, 3, 8, 8, 4, 0, s) == INV
    # frame in, YUV: off the chroma grid
    args = (None, P, P, P, 1, 8, 8, 4, s)
    assert lib.tg_stream_frame_in_yuv_window(P, _fmt('nv12'), _win(16, 16, 1, 0), *args) == UNS
    assert lib.tg_stream_frame_in_yuv_window(P, _fmt('p010'), _win(16, 16, 0, 3), *args) == UNS
    assert lib.tg_stream_frame_in_yuv_window(P, _fmt('i420'), _win(15, 16, 0, 0), *args) == UNS
    assert lib.tg_stream_frame_in_yuv_window(P, _fmt('yuy2'), _win(16, 16, 0, 1), *args) == UNS
    assert lib.tg_stream_frame_in_yuv_window(P, _fmt('uyvy'), _win(16, 15, 1, 0), *args) == UNS
    assert lib.tg_stream_frame_in_yuv_window(P, _fmt('nv12'), _win(16, 16, 10, 0), *args) == INV
    assert lib.tg_stream_frame_in_yuv_window(P, _fmt('nv12'), None, *args) == INV
    assert lib.tg_stream_frame_in_yuv_window(P + 1, _fmt('p010'), _win(16, 16, 0, 0), *args) == INV
    # encodes
    assert lib.tg_rgb_to_yuv_window(P, None, P, _fmt('nv12'), None, 1, 8, 8, s) == INV
    assert lib.tg_rgb_to_yuv_window(P, None, P, _fmt('nv12'), _win(16, 16, 2, 9), 1, 8, 8, s) == INV
    assert lib.tg_rgb_to_yuv_window(P, None, P, _fmt('nv12'), _win(16, 16, 1, 2), 1, 8, 8, s) == UNS
    assert lib.tg_rgb_to_yuv_window(P, None, P, _fmt('i444'), _win(16, 16, 9, 0), 1, 8, 8, s) == INV
    assert lib.tg_rgb_to_yuv_window(P, None, P, _fmt('yuy2'), _win(16, 16, 1, 1), 1, 8, 8, s) == UNS
    assert lib.tg_rgb_to_yuv_window(P, None, P, _fmt('p010'), _win(16, 16, 0, 0), 1, 8, 8, s) == INV   # 10 bit: f32
    assert lib.tg_float_to_uint8_nhwc_window(P, P, None, 1, 3, 8, 8, s) == INV
    assert lib.tg_float_to_uint8_nhwc_window(P, P, _win(8, 16, 1, 0), 1, 3, 8, 8, s) == INV
    assert lib.tg_resample_nchw_f32_window(P, 1, 3, 8, 8, P, P, 9, P, P, 9, 16, 16, P, None, s) == INV
    assert lib.tg_resample_nchw_f32_window(P, 1, 3, 8, 8, P, P, 9, P, P, 9, 16, 16, P, _win(16, 16, 0, 1), s) == INV
    assert lib.tg_resample_nchw_f32_window(P, 1, 3, 8, 8, P, P, 9, P, P, 9, 16, 16, None, _win(16, 16, 0, 0),
                                           s) == INV
    # fill and luma sums
    assert lib.tg_fill_black(None, None, 1, 3, 8, 8, s) == INV
    assert lib.tg_fill_black(P, None, 1, 3, 0, 8, s) == INV
    assert lib.tg_fill_black(P, _fmt('nv12'), 1, 3, 7, 8, s) == UNS
    assert lib.tg_fill_black(P, _fmt('yuy2'), 1, 3, 8, 7, s) == UNS
    assert lib.tg_fill_black(P, _fmt('nv12'), 1, 4, 8, 8, s) == INV
    assert lib.tg_fill_black(P + 1, _fmt('i420_10'), 1, 3, 8, 8, s) == INV
    assert lib.tg_luma_line_sums(None, None, 0, 1, 3, 8, 8, P, P, s) == INV
    assert lib.tg_luma_line_sums(P, None, 0, 1, 3, 8, 8, P + 4, P, s) == INV
    assert lib.tg_luma_line_sums(P, None, 0, 1, 4, 8, 8, P, P, s) == INV
    assert lib.tg_luma_line_sums(P, _fmt('i420'), 0, 1, 3, 7, 8, P, P, s) == UNS
