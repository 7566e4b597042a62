"""CPU tests (no GPU): oracle/yuv_color.py, the specification of the stream's BT.601 / BT.709, limited / full range,
8- and 10-bit YUV 4:2:0 frame I/O.

- its 'bt601' 8-bit conversions are oracle/yuv_oracle.py's (cv2's) on the exhaustive patterns;
- every 8-bit RGB triple and every (Y, U, V) triple, for all four colours, within 1 code value of the float64
  ITU-T H.273 formula ('bt601' decode: with cv2's clamp of Y at 16, which the formula does not have);
- 'bt601-full' within 1 code value of cv2's COLOR_RGB2YCrCb / COLOR_YCrCb2RGB (skipped without cv2);
- 10-bit on a dense sample that includes 0, 64, 512, 940, 960 and 1023 in every channel, against float64;
- the word layouts (P010 high bits, I420_10 low bits and clamp) and the fp32 quantisation."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import yuv_color as C              # noqa: E402
from oracle import yuv_oracle as Y8            # noqa: E402


def _all_rgb():
    i = np.arange(1 << 24, dtype=np.int64)
    return np.stack([(i >> 16) & 255, (i >> 8) & 255, i & 255], axis=-1)


def _per_pixel_encode(rgb, depth, color):
    """The oracle's integer encode of each pixel (as the top-left pixel of its own 2x2 block): [N, 3] -> [N, 3]."""
    layout = 'i420' if depth == 8 else 'i420_10'
    block = np.repeat(np.repeat(rgb.reshape(-1, 1, 1, 3), 2, axis=1), 2, axis=2)          # [N,2,2,3]
    yuv = C.split_planes(C.rgb_to_yuv(block.astype(np.uint8 if depth == 8 else np.uint16), layout, color), layout)
    return np.stack([yuv[0][:, 0, 0], yuv[1][:, 0, 0], yuv[2][:, 0, 0]], axis=-1)


@pytest.mark.parametrize('layout', Y8.LAYOUTS)
def test_bt601_8bit_is_the_cv2_oracle(layout):
    for r in range(0, 4096, 1024):
        rgb = Y8.rgb_triples_pattern(r, 256)
        assert np.array_equal(C.rgb_to_yuv(rgb, layout), Y8.rgb_to_yuv420(rgb, layout)), r
    frame = Y8.yuv_triples_pattern(layout)
    assert np.array_equal(C.yuv_to_rgb(frame, layout), Y8.yuv420_to_rgb(frame, layout))


@pytest.mark.parametrize('color', C.COLORS)
def test_encode_every_rgb_triple_within_one_of_float64(color):
    rgb = _all_rgb()
    for k in range(0, rgb.shape[0], 1 << 22):
        part = rgb[k:k + (1 << 22)]
        got = _per_pixel_encode(part, 8, color)
        want = C.float_rgb_to_yuv(part, 8, color)
        assert int(np.abs(got - want).max()) <= 1, (color, k)


@pytest.mark.parametrize('color', C.COLORS)
def test_decode_every_yuv_triple_within_one_of_float64(color):
    frame = C.yuv_triples_pattern('nv12')
    got = C.yuv_to_rgb(frame, 'nv12', color).astype(np.int64)
    y, u, v = (p.astype(np.int64) for p in C.split_planes(frame, 'nv12'))
    up = lambda a: np.repeat(np.repeat(a, 2, axis=-2), 2, axis=-1)
    if color == 'bt601':
        y = np.maximum(y, 16)               # cv2's clamp, kept in this row only
    want = C.float_yuv_to_rgb(np.stack([y, up(u), up(v)], axis=-1), 8, color)
    assert int(np.abs(got - want).max()) <= 1, color


def test_derived_rows_do_not_clamp_luma_below_the_offset():
    """Y = 0 with a strong chroma: the H.273 rows follow the formula, only cv2's row clamps Y to 16 first."""
    frame = C.join_planes(np.zeros((2, 2), np.uint8), np.full((1, 1), 40, np.uint8), np.full((1, 1), 240, np.uint8),
                          'nv12')
    f = C.float_yuv_to_rgb(np.array([0, 40, 240]), 8, 'bt709')
    assert np.abs(C.yuv_to_rgb(frame, 'nv12', 'bt709')[0, 0].astype(np.int64) - f).max() <= 1
    clamped = C.yuv_to_rgb(frame, 'nv12', 'bt601')[0, 0].astype(np.int64)
    assert np.abs(clamped - C.float_yuv_to_rgb(np.array([0, 40, 240]), 8, 'bt601')).max() > 1


def test_bt601_full_matches_cv2_ycrcb():
    cv2 = pytest.importorskip('cv2')
    rgb = _all_rgb()
    for k in range(0, rgb.shape[0], 1 << 22):
        part = rgb[k:k + (1 << 22)]
        got = _per_pixel_encode(part, 8, 'bt601-full')
        ycrcb = cv2.cvtColor(part.astype(np.uint8).reshape(1, -1, 3), cv2.COLOR_RGB2YCrCb)[0].astype(np.int64)
        assert int(np.abs(got - ycrcb[:, [0, 2, 1]]).max()) <= 1, k
    frame = C.yuv_triples_pattern('i420')
    got = C.yuv_to_rgb(frame, 'i420', 'bt601-full').astype(np.int64)
    y, u, v = C.split_planes(frame, 'i420')
    up = lambda a: np.repeat(np.repeat(a, 2, axis=-2), 2, axis=-1)
    ycrcb = np.stack([y, up(v), up(u)], axis=-1).astype(np.uint8)
    want = cv2.cvtColor(ycrcb, cv2.COLOR_YCrCb2RGB).astype(np.int64)
    assert int(np.abs(got - want).max()) <= 1


@pytest.mark.parametrize('color', C.COLORS)
def test_10bit_dense_sample_within_one_of_float64(color):
    s = C.samples10()
    assert {0, 64, 512, 940, 960, 1023} <= set(s.tolist())
    trip = np.stack(np.meshgrid(s, s, s, indexing='ij'), axis=-1).reshape(-1, 3)
    got = _per_pixel_encode(trip, 10, color)
    assert int(np.abs(got - C.float_rgb_to_yuv(trip, 10, color)).max()) <= 1
    # decode: each triple as a 2x2 block of one Y
    n = trip.shape[0]
    y = np.repeat(np.repeat(trip[:, 0].reshape(n, 1, 1), 2, 1), 2, 2)
    frame = C.join_planes(y, trip[:, 1].reshape(n, 1, 1), trip[:, 2].reshape(n, 1, 1), 'i420_10')
    rgb = C.yuv_to_rgb(frame, 'i420_10', color)[:, 0, 0].astype(np.int64)
    assert int(np.abs(rgb - C.float_yuv_to_rgb(trip, 10, color)).max()) <= 1


def test_10bit_pattern_covers_every_sample_triple():
    frames, h, w = C.yuv10_pattern('p010')
    assert frames.dtype == np.uint16 and frames.shape[1:] == (3 * h // 2, w)
    y, u, v = C.split_planes(frames, 'p010')
    up = lambda a: np.repeat(np.repeat(a, 2, axis=-2), 2, axis=-1)
    key = (y << 20) | (up(u) << 10) | up(v)
    m = C.samples10().size
    assert np.unique(key).size == m ** 3


def test_word_layouts_and_quantisation():
    y = np.array([[0, 64], [940, 1023]], np.int64)
    u, v = np.array([[512]]), np.array([[960]])
    p010 = C.join_planes(y, u, v, 'p010')
    assert p010.dtype == np.uint16 and p010[0].tolist() == [0, 64 << 6] and p010[2].tolist() == [512 << 6, 960 << 6]
    i10 = C.join_planes(y, u, v, 'i420_10')
    assert i10[1].tolist() == [940, 1023] and i10[2].tolist() == [512, 960]
    assert [a.tolist() for a in C.split_planes(p010 | 0x3f, 'p010')] == [y.tolist(), [[512]], [[960]]]
    big = i10.copy()
    big[0, 0] = 40000
    assert int(C.split_planes(big, 'i420_10')[0][0, 0]) == 1023
    x = np.array([-0.5, 0.0, 0.5 / 1023, 1.5 / 1023, 2.5 / 1023, 1.0, 1.7], np.float32)
    want = np.clip(np.rint(x * np.float32(1023)), 0, 1023)
    assert C.quantize10(x).tolist() == want.astype(np.int64).tolist()
    with pytest.raises(ValueError):
        C.split_planes(p010.astype(np.uint8), 'p010')
    with pytest.raises(ValueError):
        C.parse_color('bt2020')
    with pytest.raises(ValueError):
        C.depth_of('p016')


def test_fixed_point_fits_int32_and_extremes():
    for depth in (8, 10):
        top = (1 << depth) - 1
        for color in C.COLORS:
            c = C.coefficients(color, depth)
            assert c[14] == C.SHIFT[depth]
            # the largest decode sum: (top - yoff) * CY + max chroma term
            worst = (top - c[15]) * c[9] + (top - (1 << (depth - 1))) * max(abs(c[10]), abs(c[13])) + (1 << c[14])
            assert worst < 1 << 31, (color, depth)
            black = C.rgb_to_yuv(np.zeros((2, 2, 3), np.int64), 'i420' if depth == 8 else 'i420_10', color)
            white = C.rgb_to_yuv(np.full((2, 2, 3), top, np.int64), 'i420' if depth == 8 else 'i420_10', color)
            full = color.endswith('-full')
            assert int(black[0, 0]) == (0 if full else 16 << (depth - 8))
            assert int(white[0, 0]) == (top if full else 235 << (depth - 8))
            assert int(black[2, 0]) == int(white[2, 0]) == 1 << (depth - 1)
