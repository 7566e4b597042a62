"""CPU tests (no GPU): oracle/yuv_oracle.py, the specification of the stream's NV12 / I420 frame I/O, is
cv2.cvtColor byte for byte.

- against a live cv2 when it imports: every RGB triple as the top-left pixel of a 2x2 block (all Y and all (U, V)
  results of RGB -> I420 / NV12), and every (Y, U, V) triple of a 4096x4096 frame (YUV -> RGB, NV12 and I420);
- always against tests/golden/yuv420_cv2.npz (oracle/gen_yuv_golden.py), so the pin holds without cv2;
- the properties the kernels rely on: BT.601 limited range, chroma from the top-left pixel only, nearest chroma on
  decode, odd sizes rejected."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import yuv_oracle as Y             # noqa: E402

GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'yuv420_cv2.npz')


def _cv2():
    return pytest.importorskip('cv2')


def test_encode_every_rgb_triple_matches_cv2():
    cv2 = _cv2()
    for r in range(0, 4096, 512):                  # 512 x 4096 blocks per chunk: 2^24 top-left pixels in all
        rgb = Y.rgb_triples_pattern(r, 512)
        want = cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV_I420)
        got = Y.rgb_to_yuv420(rgb, 'i420')
        assert np.array_equal(got, want), (r, int((got != want).sum()))
        y, u, v = Y.split_planes(want, 'i420')
        assert np.array_equal(Y.rgb_to_yuv420(rgb, 'nv12'), Y.join_planes(y, u, v, 'nv12'))


@pytest.mark.parametrize('layout', Y.LAYOUTS)
def test_decode_every_yuv_triple_matches_cv2(layout):
    cv2 = _cv2()
    frame = Y.yuv_triples_pattern(layout)
    code = cv2.COLOR_YUV2RGB_NV12 if layout == 'nv12' else cv2.COLOR_YUV2RGB_I420
    want = cv2.cvtColor(frame, code)
    got = Y.yuv420_to_rgb(frame, layout)
    assert np.array_equal(got, want), int((got != want).sum())


def test_exhaustive_patterns_cover_every_triple():
    y, u, v = Y.split_planes(Y.yuv_triples_pattern('nv12'), 'nv12')
    up = lambda a: np.repeat(np.repeat(a.astype(np.int64), 2, 0), 2, 1)
    assert np.unique((y.astype(np.int64) << 16) | (up(u) << 8) | up(v)).size == 1 << 24
    tl = Y.rgb_triples_pattern(4095, 1)[0, ::2].astype(np.int64)           # the last row of blocks
    assert int((tl[-1, 0] << 16) | (tl[-1, 1] << 8) | tl[-1, 2]) == (1 << 24) - 1


def test_oracle_matches_cv2_golden():
    g = np.load(GOLDEN)
    sizes = sorted({k.split('_')[-1] for k in g.files if k.startswith('yuv_')})
    assert len(sizes) >= 3
    for key in sizes:
        assert np.array_equal(Y.rgb_to_yuv420(g[f'rgb_{key}'], 'i420'), g[f'i420_{key}']), key
        yy, u, v = Y.split_planes(g[f'i420_{key}'], 'i420')
        assert np.array_equal(Y.rgb_to_yuv420(g[f'rgb_{key}'], 'nv12'), Y.join_planes(yy, u, v, 'nv12')), key
        for layout in Y.LAYOUTS:
            assert np.array_equal(Y.yuv420_to_rgb(g[f'yuv_{key}'], layout), g[f'rgb_{layout}_{key}']), (key, layout)


def test_bt601_limited_range_and_chroma_siting():
    black, white = np.zeros((2, 2, 3), np.uint8), np.full((2, 2, 3), 255, np.uint8)
    assert Y.rgb_to_yuv420(black, 'i420').ravel().tolist() == [16] * 4 + [128, 128]
    assert Y.rgb_to_yuv420(white, 'i420').ravel().tolist() == [235] * 4 + [128, 128]
    rng = np.random.default_rng(3)
    rgb = rng.integers(0, 256, size=(6, 8, 3), dtype=np.uint8)
    other = rng.integers(0, 256, size=rgb.shape, dtype=np.uint8)
    other[::2, ::2] = rgb[::2, ::2]                                       # same top-left pixels
    for layout in Y.LAYOUTS:
        a, b = Y.rgb_to_yuv420(rgb, layout), Y.rgb_to_yuv420(other, layout)
        assert np.array_equal(a[6:], b[6:])                                # chroma rows: top-left pixel only
    yuv = rng.integers(0, 256, size=(9, 8), dtype=np.uint8)
    rgb_nv12 = Y.yuv420_to_rgb(yuv, 'nv12')
    y, u, v = Y.split_planes(yuv, 'nv12')
    assert np.array_equal(Y.yuv420_to_rgb(Y.join_planes(y, u, v, 'i420'), 'i420'), rgb_nv12)
    # nearest chroma: the RGB of a pixel depends on its own Y and its block's (U, V) only
    flat = Y.join_planes(np.full_like(y, 100), u, v, 'nv12')
    rgb_flat = Y.yuv420_to_rgb(flat, 'nv12')
    assert np.array_equal(rgb_flat[0::2, 0::2], rgb_flat[1::2, 1::2])


def test_odd_sizes_and_unknown_layouts_are_rejected():
    with pytest.raises(ValueError):
        Y.rgb_to_yuv420(np.zeros((4, 5, 3), np.uint8), 'i420')
    with pytest.raises(ValueError):
        Y.rgb_to_yuv420(np.zeros((3, 4, 3), np.uint8), 'nv12')
    with pytest.raises(ValueError):
        Y.yuv420_to_rgb(np.zeros((6, 5), np.uint8), 'nv12')
    with pytest.raises(ValueError):
        Y.yuv420_to_rgb(np.zeros((6, 4), np.uint8), 'yuyv')
    cv2 = pytest.importorskip('cv2')
    with pytest.raises(cv2.error):                                         # cv2 refuses them too
        cv2.cvtColor(np.zeros((4, 5, 3), np.uint8), cv2.COLOR_RGB2YUV_I420)
