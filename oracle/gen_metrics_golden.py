"""Generate tests/golden/metrics_cv2.npz: cv2's Farneback flows and tOF on small seeded frame pairs, cv2's
COLOR_RGB2GRAY, and the Y of the reference's data_utils.rgb_to_ycbcr for the colours whose Y sits on or near a .5
rounding tie, so that oracle/farneback.py and oracle/metrics_oracle.py stay pinned to cv2 and the reference on
machines that have neither.

    python oracle/gen_metrics_golden.py

The file holds, per flow case <name>:
  <name>_prev, <name>_next    uint8 [H, W] gray frames
  <name>_flow                 cv2.calcOpticalFlowFarneback(prev, next, None, 0.5, 3, 15, 3, 5, 1.2, 0), float32
                              [H, W, 2], or every <name>_rows-th row of it (rows 0, k, 2k, ...)
and
  tof_true, tof_pred          uint8 RGB [2, H, W, 3] two-frame sequences; tof_value: compute_tOF's value for them
  gray_rgb, gray_cv2          uint8 colours [N, 3] and cv2.cvtColor(..., COLOR_RGB2GRAY) of them
  tie_rgb, tie_y              the colours whose float64 Y is within 1e-9 of a .5 tie, and rgb_to_ycbcr's Y of them
"""
import os
import sys

import cv2
import numpy as np
import scipy.ndimage as nd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import refimport  # noqa: E402

ARGS = (None, 0.5, 3, 15, 3, 5, 1.2, 0)


def textured(h, w, seed, sigma=2.0):
    r = np.random.default_rng(seed)
    base = nd.gaussian_filter(r.uniform(0, 255, (h, w)), sigma)
    return (base - base.min()) / (base.max() - base.min()) * 255


def shifted_pair(h, w, dy, dx, seed):
    pad = int(max(abs(dy), abs(dx))) + 4
    base = textured(h + 2 * pad, w + 2 * pad, seed)
    a = base[pad:pad + h, pad:pad + w]
    b = nd.shift(base, (dy, dx), order=3, mode='nearest')[pad:pad + h, pad:pad + w]
    return np.clip(a, 0, 255).round().astype(np.uint8), np.clip(b, 0, 255).round().astype(np.uint8)


def cases():
    out = {}
    out['small'] = shifted_pair(128, 136, 1.0, 2.0, 1) + (3,)            # L = 2
    out['odd'] = shifted_pair(67, 101, -0.7, 1.3, 2) + (1,)              # L = 1, level 33.5 -> 34
    out['tiny'] = shifted_pair(40, 31, 0.5, 0.5, 3) + (1,)               # L = 0
    out['large'] = shifted_pair(96, 128, 9.0, -11.0, 4) + (2,)           # flow leaves the frame
    a, b = shifted_pair(96, 128, 1.5, 1.0, 5)
    a[:, :64] = 90                                                       # flat half: the 1e-3 regulariser
    b[:, :64] = 90
    out['flat'] = (a, b, 2)
    out['deep'] = shifted_pair(259, 270, 2.5, -3.5, 6) + (16,)           # L = 3, 32.375 x 33.75 -> 32 x 34
    return out


def main():
    arrays = {'cv2_version': np.array(cv2.__version__)}
    for name, (a, b, step) in cases().items():
        f = cv2.calcOpticalFlowFarneback(a, b, *ARGS)
        arrays[f'{name}_prev'], arrays[f'{name}_next'] = a, b
        arrays[f'{name}_flow'] = f[::step]
        arrays[f'{name}_rows'] = np.int64(step)
    rng = np.random.default_rng(7)
    seq = [np.stack([textured(60, 80, 10 + c, 3.0) for c in range(3)], -1)]
    seq.append(nd.shift(seq[0], (1.0, -2.0, 0), order=1, mode='nearest'))
    true = np.clip(np.stack(seq), 0, 255).round().astype(np.uint8)
    pred = np.clip(true.astype(np.int64) + rng.integers(-12, 13, true.shape), 0, 255).astype(np.uint8)
    g = [cv2.cvtColor(x, cv2.COLOR_RGB2GRAY) for x in (true[0], true[1], pred[0], pred[1])]
    d = cv2.calcOpticalFlowFarneback(g[0], g[1], *ARGS) - cv2.calcOpticalFlowFarneback(g[2], g[3], *ARGS)
    arrays['tof_true'], arrays['tof_pred'] = true, pred
    arrays['tof_value'] = np.float64(np.mean(np.sqrt(np.sum(d ** 2, axis=-1))))
    colours = rng.integers(0, 256, (4096, 3)).astype(np.uint8)
    # near-tie colours of Y (below), plus the extremes
    c = np.arange(1 << 24, dtype=np.int64)
    rgb = np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8)
    f = rgb.astype(np.float64)
    s = f[:, 0] * 0.256788235294118 + f[:, 1] * 0.504129411764706 + f[:, 2] * 0.097905882352941 + 16.0
    tie = rgb[np.abs(s - np.floor(s) - 0.5) < 1e-9]
    colours = np.concatenate([colours, tie, np.uint8([[0, 0, 0], [255, 255, 255]])])
    arrays['gray_rgb'] = colours
    arrays['gray_cv2'] = cv2.cvtColor(colours[None], cv2.COLOR_RGB2GRAY)[0]
    _, _, du = refimport.import_generator()
    arrays['tie_rgb'] = tie
    arrays['tie_y'] = du.rgb_to_ycbcr(tie[None])[0, :, 0]
    path = os.path.join(ROOT, 'tests', 'golden', 'metrics_cv2.npz')
    np.savez_compressed(path, **arrays)
    print(path, os.path.getsize(path), 'bytes;', len(tie), 'near-tie colours')


if __name__ == '__main__':
    main()
