"""Generate tests/golden/yuv422_cv2.npz: cv2.cvtColor's packed YUV 4:2:2 conversions (YUY2 and UYVY, both
directions), so that oracle/yuv_422_444.py's 4:2:2 rules stay pinned to cv2 where cv2 is not installed.

    python oracle/gen_yuv422_golden.py

RGB sets (each an RGB uint8 frame [h, w, 3], w even, encoded with COLOR_RGB2YUV_YUY2 / _UYVY):
  rgb_<name>, yuy2_<name>, uyvy_<name>  ([h, 2w] each)
  random_<h>x<w>   seeded random frames, odd heights included
  extremes         every ordered pair of the 8 corners of the RGB cube side by side, and pairs (x, 255 - x)
  ties             pairs whose chroma sum lands on a rounding boundary of cv2's 14-bit rule, for U or for V:
                   (k . (rgb0 + rgb1) + 8192) mod 16384 in {0, 16384 - g}, i.e. the pair's mean at or just below .5
                   (g = gcd of the channel's coefficients and 16384: 4 for U, 1 for V)
YUV sets (random bytes [h, 2w] decoded with COLOR_YUV2RGB_YUY2 / _UYVY):
  yuv_<h>x<w>, rgb_yuy2_<h>x<w>, rgb_uyvy_<h>x<w>
"""
import math
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import yuv_422_444 as C           # noqa: E402

SIZES = ((1, 2), (5, 54), (16, 30), (64, 96))


def _encode(rgb, code):
    h, w = rgb.shape[:2]
    return cv2.cvtColor(rgb, getattr(cv2, 'COLOR_RGB2YUV_' + code)).reshape(h, 2 * w)


def _decode(yuv, code):
    h, w2 = yuv.shape
    return cv2.cvtColor(yuv.reshape(h, w2 // 2, 2), getattr(cv2, 'COLOR_YUV2RGB_' + code))


def extremes(rng):
    corners = np.array([[(i >> 2) & 1, (i >> 1) & 1, i & 1] for i in range(8)], np.int64) * 255
    pairs = [np.stack([a, b]) for a in corners for b in corners]                   # 64 pairs
    x = rng.integers(0, 256, size=(64, 3))
    pairs += [np.stack([a, 255 - a]) for a in x]                                     # 64 more
    return np.stack(pairs).reshape(8, 32, 3).astype(np.uint8)


def ties(rng, per_set=512):
    """Pairs whose U or V sum sits on cv2's rounding boundary; per_set of each (channel, residue)."""
    ku, kv = C.CV2_422[1], C.CV2_422[2]
    s = np.arange(511, dtype=np.int64)
    sg, sb = (a.reshape(-1) for a in np.meshgrid(s, s, indexing='ij'))
    below = [16384 - math.gcd(*k, 16384) for k in (ku, kv)]
    found = {(c, r): [] for c in range(2) for r in (0, below[c])}
    for sr in range(511):
        for c, k in enumerate((ku, kv)):
            m = (k[0] * sr + k[1] * sg + k[2] * sb + 8192) & 16383
            for r in (0, below[c]):
                idx = np.flatnonzero(m == r)
                if idx.size:
                    found[(c, r)].append(np.stack([np.full(idx.size, sr), sg[idx], sb[idx]], axis=-1))
    sums = []
    for key, parts in found.items():
        allp = np.concatenate(parts)
        sums.append(allp[rng.choice(allp.shape[0], size=min(per_set, allp.shape[0]), replace=False)])
    sums = np.concatenate(sums)
    # split each sum into two code values at a random point of its range
    lo, hi = np.maximum(sums - 255, 0), np.minimum(sums, 255)
    p0 = lo + (rng.random(sums.shape) * (hi - lo + 1)).astype(np.int64)
    pairs = np.stack([p0, sums - p0], axis=1)                                         # [N, 2, 3]
    return pairs.reshape(-1, 64, 3).astype(np.uint8)


def main():
    rng = np.random.default_rng(422)
    arrays = {'cv2_version': np.array(cv2.__version__)}
    sets = {f'random_{h}x{w}': rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in SIZES}
    sets['extremes'] = extremes(rng)
    sets['ties'] = ties(rng)
    for name, rgb in sets.items():
        arrays[f'rgb_{name}'] = rgb
        arrays[f'yuy2_{name}'] = _encode(rgb, 'YUY2')
        arrays[f'uyvy_{name}'] = _encode(rgb, 'UYVY')
    for h, w in SIZES:
        key = f'{h}x{w}'
        yuv = rng.integers(0, 256, size=(h, 2 * w), dtype=np.uint8)
        arrays[f'yuv_{key}'] = yuv
        arrays[f'rgb_yuy2_{key}'] = _decode(yuv, 'YUY2')
        arrays[f'rgb_uyvy_{key}'] = _decode(yuv, 'UYVY')
    path = os.path.join(ROOT, 'tests', 'golden', 'yuv422_cv2.npz')
    np.savez_compressed(path, **arrays)
    print(path, os.path.getsize(path))


if __name__ == '__main__':
    main()
