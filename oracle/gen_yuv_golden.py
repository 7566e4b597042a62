"""Generate tests/golden/yuv420_cv2.npz: cv2.cvtColor's YUV 4:2:0 conversions of small seeded random frames, so
that oracle/yuv_oracle.py stays pinned to cv2 where cv2 is not installed.

    python oracle/gen_yuv_golden.py

For each size (h, w) the file holds
  rgb_<h>x<w>            RGB uint8 [h, w, 3]
  i420_<h>x<w>           cv2.cvtColor(rgb, COLOR_RGB2YUV_I420)            [3h/2, w]
  yuv_<h>x<w>            random YUV bytes                                 [3h/2, w]
  rgb_nv12_<h>x<w>       cv2.cvtColor(yuv, COLOR_YUV2RGB_NV12)            [h, w, 3]
  rgb_i420_<h>x<w>       cv2.cvtColor(yuv, COLOR_YUV2RGB_I420)            [h, w, 3]
"""
import os

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = ((2, 2), (38, 54), (16, 30), (64, 96))


def main():
    rng = np.random.default_rng(420)
    arrays = {'cv2_version': np.array(cv2.__version__)}
    for h, w in SIZES:
        key = f'{h}x{w}'
        rgb = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        yuv = rng.integers(0, 256, size=(3 * h // 2, w), dtype=np.uint8)
        arrays[f'rgb_{key}'] = rgb
        arrays[f'i420_{key}'] = cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV_I420)
        arrays[f'yuv_{key}'] = yuv
        arrays[f'rgb_nv12_{key}'] = cv2.cvtColor(yuv, cv2.COLOR_YUV2RGB_NV12)
        arrays[f'rgb_i420_{key}'] = cv2.cvtColor(yuv, cv2.COLOR_YUV2RGB_I420)
    path = os.path.join(ROOT, 'tests', 'golden', 'yuv420_cv2.npz')
    np.savez_compressed(path, **arrays)
    print(path)


if __name__ == '__main__':
    main()
