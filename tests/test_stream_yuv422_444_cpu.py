"""CPU tests (no GPU): packed 4:2:2 (YUY2, UYVY) and planar 4:4:4 (I444, I444_10) frame I/O of streamed inference.

- oracle/yuv_422_444.py reproduces cv2's COLOR_RGB2YUV_YUY2 / _UYVY and COLOR_YUV2RGB_YUY2 / _UYVY byte for byte
  on tests/golden/yuv422_cv2.npz (oracle/gen_yuv422_golden.py), including the pairs on the chroma average's rounding
  boundary, and against a live cv2 when it imports;
- its decode of I444 with chroma replicated from NV12 / I420_10 is the 4:2:0 decode, and YUY2's is I444's;
- tg_yuv_coefficients gives the 4:2:0 row of the same depth for the new layouts;
- the C ABI, the ops wrappers and FRNet.stream refuse what they cannot serve before any device work."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402
from oracle import yuv_422_444 as C            # noqa: E402

L = T.lib
ops = sys.modules['tecogan-pytorch_b200.ops']
P = ctypes.c_void_p(16)                        # a non-null pointer that is never dereferenced
NEW = C.LAYOUTS_422 + C.LAYOUTS_444
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'yuv422_cv2.npz')
CODES = {'yuy2': L.YUV_YUY2, 'uyvy': L.YUV_UYVY, 'i444': L.YUV_I444, 'i444_10': L.YUV_I444_10}


@pytest.fixture(scope='module')
def golden():
    return dict(np.load(GOLDEN))


def _fmt(layout, matrix=601, full=0):
    return ctypes.byref(L.YuvFormat(layout, matrix, full, 0))


def _sets(golden):
    return sorted(k[len('rgb_'):] for k in golden if k.startswith('rgb_') and not k.startswith(('rgb_yuy2_',
                                                                                                'rgb_uyvy_')))


# ------------------------------------------------------------------------------------------------ oracle vs cv2
@pytest.mark.parametrize('layout', C.LAYOUTS_422)
def test_oracle_encode_is_cv2_on_the_golden_sets(golden, layout):
    names = _sets(golden)
    assert {'extremes', 'ties', 'random_1x2', 'random_5x54'} <= set(names)
    for name in names:
        got = C.rgb_to_yuv(golden[f'rgb_{name}'], layout)
        assert got.dtype == np.uint8 and np.array_equal(got, golden[f'{layout}_{name}']), name


@pytest.mark.parametrize('layout', C.LAYOUTS_422)
def test_oracle_decode_is_cv2_on_the_golden_sets(golden, layout):
    keys = [k[len('yuv_'):] for k in golden if k.startswith('yuv_')]
    assert len(keys) >= 4
    for key in keys:
        assert np.array_equal(C.yuv_to_rgb(golden[f'yuv_{key}'], layout), golden[f'rgb_{layout}_{key}']), key


def test_tie_set_pins_the_rounding_of_the_average(golden):
    """On the tie pairs, rounding the pair's mean half down (or averaging the two rounded per-pixel chroma
    values) gives other bytes than cv2's: the fixture tells the rules apart."""
    rgb = golden['rgb_ties'].astype(np.int64)
    want = golden['yuy2_ties'].reshape(*rgb.shape[:-2], -1, 4).astype(np.int64)
    s = rgb[..., 0::2, :] + rgb[..., 1::2, :]
    for k, col in ((C.CV2_422[1], 1), (C.CV2_422[2], 3)):
        dot = k[0] * s[..., 0] + k[1] * s[..., 1] + k[2] * s[..., 2]
        up = ((dot + 8192) >> 14) + 128
        down = ((dot + 8191) >> 14) + 128
        assert np.array_equal(up, want[..., col])
        assert (down != want[..., col]).sum() > 100


def test_oracle_is_cv2_live():
    cv2 = pytest.importorskip('cv2')
    rng = np.random.default_rng(8)
    rgb = rng.integers(0, 256, size=(97, 512, 3), dtype=np.uint8)
    yuv = rng.integers(0, 256, size=(97, 1024), dtype=np.uint8)
    for layout, code in (('yuy2', 'YUY2'), ('uyvy', 'UYVY')):
        enc = cv2.cvtColor(rgb, getattr(cv2, f'COLOR_RGB2YUV_{code}')).reshape(97, 1024)
        assert np.array_equal(C.rgb_to_yuv(rgb, layout), enc)
        dec = cv2.cvtColor(yuv.reshape(97, 512, 2), getattr(cv2, f'COLOR_YUV2RGB_{code}'))
        assert np.array_equal(C.yuv_to_rgb(yuv, layout), dec)


# ------------------------------------------------------------------------------------------------ oracle identities
def _up420(a):
    return np.repeat(np.repeat(a, 2, axis=-2), 2, axis=-1)


@pytest.mark.parametrize('color', C.COLORS)
@pytest.mark.parametrize('src,dst', [('nv12', 'i444'), ('i420_10', 'i444_10')])
def test_i444_with_replicated_4_2_0_chroma_decodes_as_4_2_0(src, dst, color):
    if src == 'nv12':
        frame = C.yuv_triples_pattern('nv12')[:1536]                          # 1024 rows of every (U, V)
    else:
        frame = C.yuv10_pattern('i420_10')[0][:4]
    y, u, v = C.split_planes(frame, src)
    f444 = C.join_planes(y, _up420(u), _up420(v), dst)
    assert np.array_equal(C.yuv_to_rgb(f444, dst, color), C.yuv_to_rgb(frame, src, color))


@pytest.mark.parametrize('color', C.COLORS)
@pytest.mark.parametrize('layout', C.LAYOUTS_422)
def test_4_2_2_decodes_as_i444_with_the_pair_chroma(layout, color):
    frame = C.yuv_triples_pattern(layout)[:1024]
    y, u, v = C.split_planes(frame, layout)
    f444 = C.join_planes(y, np.repeat(u, 2, axis=-1), np.repeat(v, 2, axis=-1), 'i444')
    assert np.array_equal(C.yuv_to_rgb(frame, layout, color), C.yuv_to_rgb(f444, 'i444', color))


def test_triple_patterns_cover_every_triple():
    for layout in ('yuy2', 'uyvy', 'i444'):
        frame = C.yuv_triples_pattern(layout)
        assert frame.shape == C.frame_shape(layout, 4096, 4096)
        y, u, v = C.split_planes(frame, layout)
        if layout != 'i444':
            u, v = np.repeat(u, 2, axis=-1), np.repeat(v, 2, axis=-1)
        assert np.unique((y << 16) | (u << 8) | v).size == 1 << 24, layout
    frames, h, w = C.yuv10_pattern('i444_10')
    y, u, v = C.split_planes(frames, 'i444_10')
    m = C.samples10().size
    keys = np.unique(((y << 20) | (u << 10) | v)[(frames[:, :h] < 1024) & (frames[:, h:2 * h] < 1024)
                                                  & (frames[:, 2 * h:] < 1024)])
    assert keys.size > 0.8 * m ** 3 and int((frames > 1023).sum()) > 0


@pytest.mark.parametrize('color', C.COLORS)
def test_i444_encode_is_the_per_pixel_4_2_0_encode(color):
    rng = np.random.default_rng(45)
    for layout, src, top in (('i444', 'i420', 255), ('i444_10', 'i420_10', 1023)):
        rgb = rng.integers(0, top + 1, size=(7, 9, 3))
        y, u, v = C.split_planes(C.rgb_to_yuv(rgb, layout, color), layout)
        dt = np.uint8 if top == 255 else np.uint16
        block = np.repeat(np.repeat(rgb, 2, axis=0), 2, axis=1).astype(dt)
        y4, u4, v4 = C.split_planes(C.rgb_to_yuv(block, src, color), src)
        assert np.array_equal(y, y4[::2, ::2]) and np.array_equal(u, u4) and np.array_equal(v, v4), layout


@pytest.mark.parametrize('color', ['bt709', 'bt601-full', 'bt709-full'])
def test_derived_4_2_2_chroma_is_the_pair_mean(color):
    """Derived colours: a pair of equal pixels gets the per-pixel chroma, and any pair is within one code value of
    the float64 H.273 chroma of the pair's mean."""
    rng = np.random.default_rng(46)
    rgb = rng.integers(0, 256, size=(64, 256, 3)).astype(np.uint8)
    same = np.repeat(rgb[:, ::2], 2, axis=1)
    _, u, v = C.split_planes(C.rgb_to_yuv(same, 'yuy2', color), 'yuy2')
    _, u4, v4 = C.split_planes(C.rgb_to_yuv(same, 'i444', color), 'i444')
    assert np.array_equal(u, u4[:, ::2]) and np.array_equal(v, v4[:, ::2])
    _, u, v = C.split_planes(C.rgb_to_yuv(rgb, 'uyvy', color), 'uyvy')
    mean = (rgb[:, 0::2].astype(np.float64) + rgb[:, 1::2]) / 2
    enc, (_, coff), _ = C.float_matrices(color, 8)
    f = mean @ np.asarray(enc).T + np.array([0, coff, coff])
    assert np.abs(u - np.rint(f[..., 1])).max() <= 1 and np.abs(v - np.rint(f[..., 2])).max() <= 1


def test_frame_shapes_and_depths():
    for layout in C.ALL_LAYOUTS:
        assert ops.yuv_frame_shape(layout, 6, 10) == C.frame_shape(layout, 6, 10)
        assert ops.yuv_depth(layout) == C.depth_of(layout)
    assert ops.yuv_frame_shape('yuy2', 5, 10) == (5, 20) and ops.yuv_frame_shape('i444_10', 5, 9) == (15, 9)
    with pytest.raises(ValueError):
        C.frame_shape('uyvy', 4, 9)
    with pytest.raises(ValueError):
        C.split_planes(np.zeros((4, 18), np.uint8), 'yuy2')                      # 2w bytes with w odd
    with pytest.raises(ValueError):
        C.split_planes(np.zeros((9, 4), np.uint16), 'i444')                      # wrong word type


# ------------------------------------------------------------------------------------------------ the C ABI
def test_enum_values_and_exports():
    assert (L.YUV_NV12, L.YUV_I420, L.YUV_P010, L.YUV_I420_10) == (0, 1, 2, 3)
    assert (L.YUV_YUY2, L.YUV_UYVY, L.YUV_I444, L.YUV_I444_10) == (4, 5, 6, 8)
    lib = L.load()
    for sym in ('tg_stream_frame_in_yuv', 'tg_rgb_to_yuv', 'tg_yuv_coefficients', 'tg_stream_frame_in_yuv420',
                'tg_rgb_u8_to_yuv420'):
        assert hasattr(lib, sym)
    header = open(os.path.join(ROOT, 'include', 'tecogan_b200.h')).read()
    assert 'TG_YUV_YUY2 = 4, TG_YUV_UYVY = 5' in header and 'TG_YUV_I444 = 6, TG_YUV_I444_10 = 8' in header


@pytest.mark.parametrize('layout', NEW)
@pytest.mark.parametrize('color', C.COLORS)
def test_coefficients_are_the_4_2_0_row_of_the_same_depth(layout, color):
    same = 'i420_10' if C.depth_of(layout) == 10 else 'nv12'
    assert ops.yuv_coefficients(layout, color) == ops.yuv_coefficients(same, color)
    assert ops.yuv_coefficients(layout, color) == C.coefficients(color, C.depth_of(layout))


def test_layout_seven_stays_unknown():
    lib = L.load()
    out = (ctypes.c_int32 * 16)()
    assert lib.tg_yuv_coefficients(_fmt(7), out) == -2
    assert lib.tg_rgb_to_yuv(P, None, P, _fmt(7), 1, 8, 8, None) == -2
    assert b'layout' in lib.tg_last_error_string()


def test_frame_in_rejects_bad_arguments_without_a_gpu():
    lib = L.load()
    f = lib.tg_stream_frame_in_yuv
    for layout in NEW:
        fm = _fmt(CODES[layout])
        assert f(None, fm, None, P, P, P, 1, 8, 8, 4, None) == -1
        assert f(P, fm, P, None, P, P, 1, 8, 8, 4, None) == -1
        assert f(P, fm, P, P, P, P, 1, 0, 8, 4, None) == -1
        assert f(P, fm, P, P, P, P, 1, 8, 8, 3, None) == -2
    for layout in C.LAYOUTS_422:
        assert f(P, _fmt(CODES[layout]), P, P, P, P, 1, 8, 9, 4, None) == -2                 # odd w
        assert b'even width' in lib.tg_last_error_string()
        assert f(ctypes.c_void_p(18), _fmt(CODES[layout]), P, P, P, P, 1, 8, 8, 4, None) == -1
        assert b'4-byte aligned' in lib.tg_last_error_string()
    assert f(ctypes.c_void_p(17), _fmt(L.YUV_I444_10), P, P, P, P, 1, 8, 8, 4, None) == -1
    assert b'aligned' in lib.tg_last_error_string()


def test_encode_rejects_bad_arguments_without_a_gpu():
    lib = L.load()
    f = lib.tg_rgb_to_yuv
    for layout in ('yuy2', 'uyvy', 'i444'):                                  # 8 bit: rgb_u8 only
        fm = _fmt(CODES[layout], 709)
        assert f(None, P, P, fm, 1, 8, 8, None) == -1 and b'rgb_u8' in lib.tg_last_error_string()
        assert f(P, P, P, fm, 1, 8, 8, None) == -1
        assert f(P, None, None, fm, 1, 8, 8, None) == -1
        assert f(P, None, P, fm, 1, 8, 0, None) == -1
    fm = _fmt(L.YUV_I444_10)
    assert f(P, None, P, fm, 1, 8, 8, None) == -1 and b'rgb_f32' in lib.tg_last_error_string()
    assert f(None, ctypes.c_void_p(18), P, fm, 1, 8, 8, None) == -1
    assert f(None, P, ctypes.c_void_p(17), fm, 1, 8, 8, None) == -1
    for layout in C.LAYOUTS_422:
        fm = _fmt(CODES[layout])
        assert f(P, None, P, fm, 1, 8, 7, None) == -2 and b'even width' in lib.tg_last_error_string()
        assert f(P, None, ctypes.c_void_p(18), fm, 1, 8, 8, None) == -1
        assert b'4-byte aligned' in lib.tg_last_error_string()


def test_ops_wrappers_refuse_before_device_work():
    lr = torch.zeros(1, 3, 8, 8)
    hr = torch.zeros(1, 3, 32, 32)
    with pytest.raises(T.TecoganB200Error, match='layout'):
        ops.stream_frame_in_yuv(None, 'yuyv', 'bt601', None, lr, lr.clone(), hr, 4)
    with pytest.raises(T.TecoganB200Error, match='CUDA'):
        ops.stream_frame_in_yuv(torch.zeros(1, 8, 16, dtype=torch.uint8), 'yuy2', 'bt601', None, lr, lr.clone(),
                                hr, 4)
    with pytest.raises(T.TecoganB200Error, match='rgb_f32'):
        ops.rgb_to_yuv('i444_10', 'bt709', rgb_u8=torch.zeros(1, 8, 8, 3, dtype=torch.uint8))
    with pytest.raises(T.TecoganB200Error, match='rgb_u8'):
        ops.rgb_to_yuv('uyvy', 'bt709', rgb_f32=torch.zeros(1, 3, 8, 8))
    assert ops.yuv_size_error('yuy2', 7, 9) and not ops.yuv_size_error('yuy2', 7, 10)
    assert ops.yuv_size_error('i444_10', 7, 9) is None and ops.yuv_size_error('nv12', 7, 10)


# ------------------------------------------------------------------------------------------------ FRNet.stream
def _net():
    return T.FRNet(3, 3, 64, 2, 'BD', 4).eval()


def test_stream_accepts_the_new_layouts_with_every_colour():
    net = _net()
    for layout in NEW:
        for color in C.COLORS:
            s = net.stream(2, 15, 24, device='cuda', input=layout, in_color=color, out_format=layout,
                           out_color=color)
            assert (s.input, s.out_format, s.in_color, s.out_color) == (layout, layout, color, color)
    # odd heights for 4:2:2 / 4:4:4, odd widths for 4:4:4, odd out_size where the layout allows it
    net.stream(1, 7, 10, device='cuda', input='yuy2', out_format='uyvy')
    net.stream(1, 7, 9, device='cuda', input='i444', out_format='i444_10')
    net.stream(1, 8, 10, device='cuda', out_format='i444', out_size=(31, 39))
    net.stream(1, 8, 10, device='cuda', out_format='yuy2', out_size=(31, 40))


@pytest.mark.parametrize('kw', [
    dict(input='yuy2', w=9), dict(input='uyvy', w=15), dict(out_format='yuy2', w=9),
    dict(out_format='uyvy', out_size=(32, 39)), dict(out_format='yuy2', out_size=(31, 39)),
    dict(input='i444', out_format='nv12', h=7), dict(input='yuyv'), dict(out_format='i422'),
    dict(input='i444', channel_order='bgr'),
])
def test_stream_refuses_bad_options(kw):
    h, w = kw.pop('h', 8), kw.pop('w', 10)
    with pytest.raises(ValueError):
        _net().stream(1, h, w, device='cuda', **kw)


@pytest.mark.parametrize('inp,frames,match', [
    ('yuy2', np.zeros((2, 3, 15, 48), np.uint16), 'expects torch.uint8'),
    ('i444_10', np.zeros((2, 3, 45, 24), np.uint8), 'expects torch.uint16'),
    ('i444', np.zeros((2, 3, 45, 24), np.uint16), 'expects torch.uint8'),
    ('yuy2', np.zeros((2, 3, 15, 24), np.uint8), 'do not match'),                  # [h, w]: one byte a pixel
    ('uyvy', np.zeros((2, 3, 22, 24), np.uint8), 'n,k,h,2w'),                        # a 4:2:0 shape
    ('i444', np.zeros((2, 3, 30, 24), np.uint8), 'n,k,3h,w'),
    ('i444_10', np.zeros((3, 45, 24), np.uint16), 'do not match'),                 # [k,...] needs n == 1
    ('yuy2', torch.zeros(2, 3, 15, 96, dtype=torch.uint8)[..., :48], 'contiguous'),
])
def test_push_refuses_bad_frames(inp, frames, match):
    s = _net().stream(2, 15, 24, device='cuda', input=inp)
    with pytest.raises(T.TecoganB200Error, match=match):
        s.push(frames)


def test_single_slot_push_takes_three_dim_frames():
    for layout, shape, dt in (('yuy2', (4, 15, 48), np.uint8), ('i444_10', (4, 45, 24), np.uint16)):
        s = _net().stream(1, 15, 24, device='cuda', input=layout)
        got = s._check_frames(np.zeros(shape, dt))
        assert tuple(got.shape) == (1, *shape)
