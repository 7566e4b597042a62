"""Generate tests/golden/resample_pil.npz: Pillow's antialiased bicubic and Lanczos resizes of small seeded random
'F' (float32) images, so that oracle/resample.py stays pinned to Pillow where Pillow is not installed.

    python oracle/gen_resample_golden.py

The file holds
  x_<H>x<W>                          the float32 input [H, W], uniform in [-0.1, 1.1]
  <filter>_<H>x<W>_<Ho>x<Wo>         Image.fromarray(x, 'F').resize((Wo, Ho), filter, reducing_gap=None)
for a downscale, an upscale and an anamorphic case (different x and y ratios) per filter.
"""
import os

import numpy as np
import PIL
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {(30, 64): ((22, 48), (8, 16), (60, 128), (40, 85)),           # about 3/4, 1/4, 2, 4/3
         (24, 45): ((27, 60), (18, 23))}                                 # anamorphic: 9/8 x 4/3, 3/4 x 1/2
FILTERS = {'bicubic': Image.BICUBIC, 'lanczos': Image.LANCZOS}


def main():
    rng = np.random.default_rng(2024)
    arrays = {'pil_version': np.array(PIL.__version__)}
    for (H, W), outs in CASES.items():
        x = rng.uniform(-0.1, 1.1, size=(H, W)).astype(np.float32)
        arrays[f'x_{H}x{W}'] = x
        for Ho, Wo in outs:
            for name, filt in FILTERS.items():
                y = Image.fromarray(x, 'F').resize((Wo, Ho), filt, reducing_gap=None)
                arrays[f'{name}_{H}x{W}_{Ho}x{Wo}'] = np.asarray(y, dtype=np.float32)
    path = os.path.join(ROOT, 'tests', 'golden', 'resample_pil.npz')
    np.savez_compressed(path, **arrays)
    print(path)


if __name__ == '__main__':
    main()
