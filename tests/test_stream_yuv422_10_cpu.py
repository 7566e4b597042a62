"""CPU tests (no GPU): 10-bit 4:2:2 (P210, I422_10, v210) frame I/O of streamed inference.

- oracle/yuv_422_10.py packs v210 as the format defines it: a hand-worked 16-byte group, a partial last group and
  the row padding;
- P210, I422_10 and v210 round-trip through the oracle's pack and unpack, carry the same samples for one RGB frame,
  and its encode and windows follow the stated rules;
- the C ABI exports and enum values, tg_yuv_coefficients' 10-bit row, and the refusals of the ABI, the ops wrappers
  and FRNet.stream before any device work (odd widths, v210 windows off the 6-column grid, 'i422' still refused)."""
import ctypes
import os
import struct
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402
from oracle import yuv_422_10 as V             # noqa: E402
from oracle import yuv_422_444 as Q            # noqa: E402

L = T.lib
ops = sys.modules['tecogan-pytorch_b200.ops']
engine = sys.modules['tecogan-pytorch_b200.engine']
P = ctypes.c_void_p(16)                        # a non-null pointer that is never dereferenced
CODES = {'p210': 9, 'i422_10': 10, 'v210': 11}


def _fmt(layout, matrix=601, full=0):
    return ctypes.byref(L.YuvFormat(layout, matrix, full, 0))


# ------------------------------------------------------------------------------------------------ v210 packing
def test_v210_hand_worked_group_partial_group_and_padding():
    # 8 pixels: one whole group (pixels 0-5) and a partial one (pixels 6, 7), then padding to 128 bytes
    y = [0x3FF, 0x001, 0x2AA, 0x155, 0x040, 0x3AC, 0x200, 0x123]
    u = [0x100, 0x0F0, 0x30F, 0x001]
    v = [0x3C0, 0x00F, 0x2C0, 0x3FE]
    words = [u[0] | y[0] << 10 | v[0] << 20, y[1] | u[1] << 10 | y[2] << 20,       # Cb0 Y0 Cr0, Y1 Cb2 Y2
             v[1] | y[3] << 10 | u[2] << 20, y[4] | v[2] << 10 | y[5] << 20,       # Cr2 Y3 Cb4, Y4 Cr4 Y5
             u[3] | y[6] << 10 | v[3] << 20, y[7], 0, 0]                          # Cb6 Y6 Cr6, Y7 and zeros
    want = struct.pack('<8I', *words) + bytes(128 - 32)
    got = V.pack_v210(np.array([y]), np.array([u]), np.array([v]))
    assert got.shape == (1, 128) and got.tobytes() == want
    # the first word byte for byte: 0x100 | 0x3FF << 10 | 0x3C0 << 20 = 0x3C0FFD00, little endian
    assert got[0, :4].tolist() == [0x00, 0xFD, 0x0F, 0x3C]
    yy, uu, vv = V.unpack_v210(got, 8)
    assert yy.tolist() == [y] and uu.tolist() == [u] and vv.tolist() == [v]
    assert V.frame_shape('v210', 3, 48) == (3, 128) and V.frame_shape('v210', 3, 50) == (3, 256)
    assert V.frame_shape('p210', 3, 50) == V.frame_shape('i422_10', 3, 50) == (6, 50)


def test_v210_decode_ignores_the_top_bits_and_the_padding():
    rng = np.random.default_rng(1)
    y, u, v = rng.integers(0, 1024, (2, 5, 10)), rng.integers(0, 1024, (2, 5, 5)), rng.integers(0, 1024, (2, 5, 5))
    f = V.pack_v210(y, u, v)
    junk = f.copy()
    w32 = junk.view('<u4')
    w32 |= rng.integers(0, 4, w32.shape).astype('<u4') << 30
    junk[..., 32:] = rng.integers(0, 256, junk[..., 32:].shape, dtype=np.uint8)     # past the 2 groups of w = 10
    for a, b in zip(V.unpack_v210(junk, 10), (y, u, v)):
        assert np.array_equal(a, b)


@pytest.mark.parametrize('layout', V.LAYOUTS)
@pytest.mark.parametrize('hw', [(1, 2), (3, 46), (5, 48), (4, 50), (7, 96)])
def test_layouts_round_trip(layout, hw):
    h, w = hw
    rng = np.random.default_rng(h * w)
    y, u, v = rng.integers(0, 1024, (2, h, w)), rng.integers(0, 1024, (2, h, w // 2)), rng.integers(0, 1024, (2, h, w // 2))
    f = V.join_planes(y, u, v, layout)
    assert f.shape == (2, *V.frame_shape(layout, h, w)) and f.dtype == V.word_dtype(layout)
    assert f.shape[1:] == ops.yuv_frame_shape(layout, h, w)
    for a, b in zip(V.split_planes(f, layout, w), (y, u, v)):
        assert np.array_equal(a, b)
    if layout == 'p210':
        assert np.array_equal(f[:, :h] >> 6, y) and np.array_equal(f[:, h:, 0::2] >> 6, u)
    if layout == 'i422_10':
        assert np.array_equal(f[:, h:].reshape(2, -1)[:, :h * w // 2].reshape(2, h, w // 2), u)


@pytest.mark.parametrize('color', V.COLORS)
def test_three_layouts_carry_the_same_samples_and_decode_alike(color):
    rng = np.random.default_rng(7)
    x = rng.random((2, 5, 26, 3)).astype(np.float32)
    x[0, 0, :4] = [[0, 0, 0], [1, 1, 1], [1, 0, 0], [0, 0, 1]]
    enc = {k: V.rgb_f32_to_yuv(x, k, color) for k in V.LAYOUTS}
    samples = [V.split_planes(enc[k], k, 26) for k in V.LAYOUTS]
    for s in samples[1:]:
        for a, b in zip(s, samples[0]):
            assert np.array_equal(a, b)
    rgb = [V.yuv_to_rgb(enc[k], k, color, 26) for k in V.LAYOUTS]
    assert all(np.array_equal(r, rgb[0]) for r in rgb[1:])


@pytest.mark.parametrize('color', V.COLORS)
def test_encode_rule(color):
    rng = np.random.default_rng(3)
    q = rng.integers(0, 1024, (9, 14, 3))
    q[0, :2] = [[0, 0, 0], [1023, 1023, 1023]]
    y, u, v = V.encode_samples(q, color)
    # luma is the I444_10 encode's, per pixel
    y4, _, _ = Q.split_planes(Q.rgb_to_yuv(q, 'i444_10', color), 'i444_10')
    assert np.array_equal(y, y4)
    # chroma of the pair's sum at 19 fraction bits: within half a code of the float64 mean's
    c = V.coefficients(color, 10)
    mean = (q[:, 0::2] + q[:, 1::2]) / 2.0
    for ch, k in ((u, 3), (v, 6)):
        f = mean @ (np.array(c[k:k + 3], np.float64) / (1 << 18)) + 512
        assert np.abs(ch - np.clip(np.rint(f), 0, 1023)).max() <= 1
    # a pair of equal pixels takes the I444_10 chroma of that pixel
    same = np.repeat(q[:, 0::2], 2, axis=1)
    _, u4, v4 = Q.split_planes(Q.rgb_to_yuv(same, 'i444_10', color), 'i444_10')
    _, us, vs = V.encode_samples(same, color)
    assert np.array_equal(us, u4[:, 0::2]) and np.array_equal(vs, v4[:, 0::2])


@pytest.mark.parametrize('layout', V.LAYOUTS)
def test_black_and_windows(layout):
    for color, yb in (('bt709', 64), ('bt601-full', 0)):
        b = V.black(layout, color, 3, 14)
        y, u, v = V.split_planes(b, layout, 14)
        assert (y == yb).all() and (u == 512).all() and (v == 512).all()
    if layout == 'v210':
        b = V.black('v210', 'bt709', 1, 14)
        # group 2 holds pixels 12, 13: its word 1 is Y13 alone, words 2 and 3 and the padding are 0
        assert b[0, 36:40].view('<u4')[0] == 64 and b[0, 40:].tolist() == [0] * 88
    # a windowed encode changes the picture's samples (v210: its groups) and nothing else
    fw = 26
    frames = V.black(layout, 'bt709', 7, fw, (2,))
    rng = np.random.default_rng(5)
    q = rng.integers(0, 1024, (2, 3, 12, 3))
    out = V.encode_window(frames, q, layout, 'bt709', 2, 6, fw)
    got = V.decode_window(out, layout, 'bt709', 2, 6, 3, 12, fw)
    want = V.yuv_to_rgb(V.rgb_to_yuv(q, layout, 'bt709'), layout, 'bt709', 12)
    assert np.array_equal(got, want)
    y, u, v = V.split_planes(out, layout, fw)
    yb, ub, vb = V.split_planes(frames, layout, fw)
    mask = np.ones(y.shape, bool)
    mask[:, 2:5, 6:18] = False
    assert np.array_equal(y[mask], yb[mask])
    mask = np.ones(u.shape, bool)
    mask[:, 2:5, 3:9] = False
    assert np.array_equal(u[mask], ub[mask]) and np.array_equal(v[mask], vb[mask])
    assert V.window_error(layout, 7, fw, 0, 18, 3, 8) is None                        # ends at the right edge
    assert V.window_error(layout, 7, fw, 0, 12, 3, 6) is None                        # ends on a group
    assert V.window_error(layout, 7, fw, 0, 4, 3, 9) and V.window_error(layout, 7, fw, 0, 3, 3, 10)   # odd w / left
    assert V.window_error(layout, 7, fw, 0, 20, 3, 8)                                # outside the frame
    off_grid = [V.window_error(layout, 7, fw, 0, *lw) for lw in ((4, 3, 12), (6, 3, 10), (0, 3, 4))]
    if layout == 'v210':                      # starts off a group, ends off a group short of the right edge
        assert all(e and '6-pixel group' in e for e in off_grid)
    else:
        assert off_grid == [None] * 3


# ------------------------------------------------------------------------------------------------ the C ABI
def test_enum_values_exports_and_coefficients():
    assert (L.YUV_P210, L.YUV_I422_10, L.YUV_V210) == (9, 10, 11)
    header = open(os.path.join(ROOT, 'include', 'tecogan_b200.h')).read()
    assert 'TG_YUV_P210 = 9, TG_YUV_I422_10 = 10, TG_YUV_V210 = 11' in header
    lib = L.load()
    for sym in ('tg_stream_frame_in_yuv', 'tg_stream_frame_in_yuv_window', 'tg_rgb_to_yuv', 'tg_rgb_to_yuv_window',
                'tg_fill_black', 'tg_luma_line_sums', 'tg_stream_frame_in_resample', 'tg_yuv_coefficients'):
        assert hasattr(lib, sym)
    for layout in V.LAYOUTS:
        for color in V.COLORS:
            assert ops.yuv_coefficients(layout, color) == V.coefficients(color, 10)
            assert ops.yuv_coefficients(layout, color) == ops.yuv_coefficients('i444_10', color)
        assert ops.yuv_depth(layout) == 10
    assert ops.yuv_word_dtype('v210') == torch.uint8 and ops.yuv_word_dtype('p210') == torch.uint16
    assert ops.yuv_word_dtype('i422_10') == torch.uint16 and ops.yuv_word_dtype('i444_10') == torch.uint16
    out = (ctypes.c_int32 * 16)()
    assert lib.tg_yuv_coefficients(_fmt(7), out) == -2 and lib.tg_yuv_coefficients(_fmt(12), out) == -2


def test_abi_refuses_bad_arguments_without_a_gpu():
    lib = L.load()
    f = lib.tg_stream_frame_in_yuv
    for layout, code in CODES.items():
        fm = _fmt(code, 709, 1)
        assert f(P, fm, P, P, P, P, 1, 8, 9, 4, None) == -2 and b'even width' in lib.tg_last_error_string()
        assert lib.tg_rgb_to_yuv(None, P, P, fm, 1, 8, 7, None) == -2
        assert lib.tg_rgb_to_yuv(P, None, P, fm, 1, 8, 8, None) == -1 and b'rgb_f32' in lib.tg_last_error_string()
        assert lib.tg_fill_black(P, fm, 1, 3, 8, 9, None) == -2
        assert lib.tg_luma_line_sums(P, fm, 0, 1, 3, 8, 9, P, P, None) == -2
    fm = _fmt(L.YUV_V210)
    assert f(ctypes.c_void_p(24), fm, P, P, P, P, 1, 8, 8, 4, None) == -1
    assert b'16-byte aligned' in lib.tg_last_error_string()
    assert lib.tg_rgb_to_yuv(None, P, ctypes.c_void_p(24), fm, 1, 8, 8, None) == -1
    assert b'16-byte aligned' in lib.tg_last_error_string()
    # v210 windows.  n = 2^31 - 1 slots make every call's grid too large, a refusal that comes after the window
    # check: a window on the group grid reaches it, one off the grid is refused first, and nothing is launched.
    fw = ops.frame_window
    big = 0x7fffffff
    for box, w, ok in (((8, 26, 0, 6), 12, True), ((8, 26, 0, 18), 8, True), ((8, 26, 0, 4), 8, False),
                       ((8, 30, 0, 18), 8, False)):
        rc = lib.tg_stream_frame_in_yuv_window(P, fm, ctypes.byref(fw(*box)), None, P, P, P, big, 8, w, 4, None)
        msg = lib.tg_last_error_string()
        assert rc == -2 and (b'grid too large' in msg if ok else b'6-pixel group' in msg), (box, msg)
        rc = lib.tg_rgb_to_yuv_window(None, P, P, fm, ctypes.byref(fw(*box)), big, 8, w, None)
        msg = lib.tg_last_error_string()
        assert rc == -2 and (b'grid too large' in msg if ok else b'6-pixel group' in msg), (box, msg)


def test_ops_wrappers_refuse_before_device_work():
    with pytest.raises(T.TecoganB200Error, match='rgb_f32'):
        ops.rgb_to_yuv('v210', 'bt709', rgb_u8=torch.zeros(1, 8, 8, 3, dtype=torch.uint8))
    with pytest.raises(T.TecoganB200Error, match='fill_black_v210'):
        ops.fill_black(torch.zeros(1, 8, 128, dtype=torch.uint8), 'v210')
    assert ops.yuv_frame_size('v210', (5, 256), 50) == (5, 50) and ops.yuv_frame_size('p210', (10, 8)) == (5, 8)
    with pytest.raises(T.TecoganB200Error):
        ops.yuv_frame_size('i422_10', (10, 8), 10)
    assert ops.yuv_size_error('v210', 7, 9) and not ops.yuv_size_error('i422_10', 7, 10)


# ------------------------------------------------------------------------------------------------ FRNet.stream
def _net():
    return T.FRNet(3, 3, 64, 2, 'BD', 4).eval()


def test_stream_accepts_the_new_layouts_with_every_colour():
    net = _net()
    for layout in V.LAYOUTS:
        for color in V.COLORS:
            s = net.stream(2, 15, 26, device='cuda', input=layout, in_color=color, out_format=layout,
                           out_color=color)
            assert (s.input, s.out_format, s.in_color, s.out_color) == (layout, layout, color, color)
    net.stream(1, 9, 26, device='cuda', input='v210', crop=(1, 6, 7, 20))            # ends at the right edge
    net.stream(1, 9, 26, device='cuda', input='v210', crop=(0, 6, 9, 12))            # ends on a group
    net.stream(1, 8, 10, device='cuda', out_format='v210', out_size=(31, 40))
    s = net.stream(1, 8, 10, device='cuda', out_format='v210', out_size=(32, 36), out_frame=(40, 48))
    assert s.out_origin == (4, 6)                                                    # 6 + 36 = 42: a group end
    s = net.stream(1, 8, 10, device='cuda', out_format='v210', out_frame=(40, 58), out_origin=(0, 18))
    assert s.out_origin == (0, 18)                                                   # 18 + 40 = 58: the right edge
    # the centred origin (6) would end a 40- or 44-wide picture inside a group: the default is the right edge
    assert net.stream(1, 8, 10, device='cuda', out_format='v210', out_frame=(40, 58)).out_origin == (4, 18)
    s = net.stream(1, 8, 10, device='cuda', out_format='v210', out_size=(32, 44), out_frame=(32, 62))
    assert s.out_origin == (0, 18)
    assert net.stream(1, 8, 10, device='cuda', out_format='p210', out_frame=(40, 58)).out_origin == (4, 8)


@pytest.mark.parametrize('kw', [
    dict(input='p210', w=9), dict(input='v210', w=15), dict(out_format='i422_10', w=9),
    dict(out_format='v210', out_size=(32, 39)), dict(out_format='i422'), dict(input='i422'),
    dict(input='v210', crop=(0, 4, 8, 6)), dict(input='v210', crop=(0, 6, 8, 2)),
    dict(input='p210', crop=(0, 1, 8, 4)), dict(input='v210', channel_order='bgr'),
    dict(out_format='v210', out_frame=(40, 61)), dict(out_format='v210', out_frame=(40, 60), out_origin=(0, 4)),
    dict(out_format='v210', out_frame=(40, 60), out_origin=(0, 6)), dict(out_format='v210', out_frame=(40, 62)),
])
def test_stream_refuses_bad_options(kw):
    h, w = kw.pop('h', 8), kw.pop('w', 10)
    with pytest.raises(ValueError):
        _net().stream(1, h, w, device='cuda', **kw)


@pytest.mark.parametrize('inp,frames,match', [
    ('v210', np.zeros((2, 3, 15, 128), np.uint16), 'expects torch.uint8'),
    ('p210', np.zeros((2, 3, 30, 26), np.uint8), 'expects torch.uint16'),
    ('v210', np.zeros((2, 3, 15, 52), np.uint8), 'n,k,h,128'),                      # [h, 2w] bytes: YUY2's shape
    ('i422_10', np.zeros((2, 3, 45, 26), np.uint16), 'n,k,2h,w'),
    ('p210', np.zeros((3, 30, 26), np.uint16), 'do not match'),                    # [k,...] needs n == 1
])
def test_push_refuses_bad_frames(inp, frames, match):
    s = _net().stream(2, 15, 26, device='cuda', input=inp)
    with pytest.raises(T.TecoganB200Error, match=match):
        s.push(frames)


def test_window_helpers():
    pic = np.zeros(26, bool)
    pic[7:23] = True
    assert engine.bars_box(np.ones(5, bool), pic, 'v210') == (0, 12, 5, 6)           # [12, 18): whole groups
    pic[7:] = True
    assert engine.bars_box(np.ones(5, bool), pic, 'v210') == (0, 12, 5, 14)          # to the right edge
    assert engine.bars_box(np.ones(5, bool), pic, 'p210') == (0, 8, 5, 18)
    h, w = engine.fit_size((480, 720), (1080, 1920), (8, 9), 'v210')
    assert w % 6 == 0 and h <= 1080 and w <= 1920
    with pytest.raises(ValueError, match='width'):
        engine.detect_bars(torch.zeros(1, 4, 128, dtype=torch.uint8), 'v210')
    with pytest.raises(ValueError, match='width'):
        engine.detect_bars(torch.zeros(1, 4, 8, dtype=torch.uint16), 'p210', width=8)
