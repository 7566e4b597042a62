"""PSNR and tOF of TecoGAN's MetricCalculator (codes/metrics/metric_calculator.py), restated in numpy.

This is the specification of tecogan_b200.metrics.sequence_metrics:

  crop   each frame pair is cropped to the smaller height and width (top-left corner)
  PSNR   'rgb': over the three channels; 'y': over the Y of data_utils.rgb_to_ycbcr.  RMSE = sqrt(mean((t - p)^2))
         in float64, PSNR = 20 log10(255 / RMSE), inf for RMSE == 0
  tOF    for t >= 1: the mean over pixels of |F(gt[t-1], gt[t]) - F(pr[t-1], pr[t])|, F = oracle.farneback on the
         gray frames (cv2 COLOR_RGB2GRAY) with pyr_scale=0.5, levels=3, winsize=15, iterations=3, poly_n=5,
         poly_sigma=1.2, flags=0.  compute_tOF always uses gray, whatever the configured tOF colorspace.

Two integer rules make the device's frame input exact:
  gray   cv2's COLOR_RGB2GRAY on uint8 is (9798 R + 19235 G + 3735 B + 16384) >> 15, for all 2^24 colours.
  Y      rgb_to_ycbcr computes np.matmul(rgb, T) + 16 in float64, clips and rounds half to even.  A left-to-right
         float64 sum r*T0 + g*T1 + b*T2 + 16 (no FMA) gives the same Y except for three colours, listed in
         Y_EXCEPTIONS, where the matmul lands on the other side of a .5 tie and the reference's Y is one lower.
"""
import numpy as np

from . import farneback as F

T_Y = (0.256788235294118, 0.504129411764706, 0.097905882352941)
Y_EXCEPTIONS = ((1, 173, 225), (12, 174, 191), (24, 46, 73))
TOF_ARGS = dict(pyr_scale=0.5, levels=3, winsize=15, iterations=3, poly_n=5, poly_sigma=1.2, flags=0)


def rgb_to_gray(u8):
    x = np.asarray(u8).astype(np.int64)
    return ((9798 * x[..., 0] + 19235 * x[..., 1] + 3735 * x[..., 2] + 16384) >> 15).astype(np.uint8)


def rgb_to_y(u8):
    """Y of data_utils.rgb_to_ycbcr, by the left-to-right rule and its exception list (uint8)"""
    x = np.asarray(u8).astype(np.float64)
    s = x[..., 0] * T_Y[0] + x[..., 1] * T_Y[1] + x[..., 2] * T_Y[2] + 16.0
    y = np.clip(s, 0, 255).round().astype(np.int64)
    c = np.asarray(u8).astype(np.int64)
    code = (c[..., 0] << 16) | (c[..., 1] << 8) | c[..., 2]
    for r, g, b in Y_EXCEPTIONS:
        y[code == ((r << 16) | (g << 8) | b)] -= 1
    return y.astype(np.uint8)


def crop_pair(t, p):
    h, w = min(t.shape[0], p.shape[0]), min(t.shape[1], p.shape[1])
    return t[:h, :w], p[:h, :w]


def psnr(true_img, pred_img, colorspace='y'):
    t, p = crop_pair(np.asarray(true_img), np.asarray(pred_img))
    if colorspace != 'rgb':
        t, p = rgb_to_y(t), rgb_to_y(p)
    diff = t.astype(np.float64) - p.astype(np.float64)
    rmse = np.sqrt(np.mean(np.power(diff, 2)))
    return np.inf if rmse == 0 else 20 * np.log10(255.0 / rmse)


def tof(true_pre, true_cur, pred_pre, pred_cur):
    flows = [F.farneback(rgb_to_gray(a), rgb_to_gray(b), **TOF_ARGS)
             for a, b in ((true_pre, true_cur), (pred_pre, pred_cur))]
    d = flows[0] - flows[1]
    return float(np.mean(np.sqrt(np.sum(d * d, axis=-1))))


def sequence_metrics(true_seq, pred_seq, psnr_colorspace='y', with_tof=True, frames=None):
    """{'PSNR': float64 [T], 'tOF': float64 [T-1]} of uint8 THWC sequences; `frames` restricts tOF to the listed
    frame indices t (pairs t-1 -> t), the others are NaN"""
    T = len(true_seq)
    crops = [crop_pair(np.asarray(true_seq[i]), np.asarray(pred_seq[i])) for i in range(T)]
    out = {}
    if psnr_colorspace is not None:
        out['PSNR'] = np.array([psnr(t, p, psnr_colorspace) for t, p in crops])
    if with_tof:
        v = np.full(max(T - 1, 0), np.nan)
        for i in range(1, T):
            if frames is None or i in frames:
                v[i - 1] = tof(crops[i - 1][0], crops[i][0], crops[i - 1][1], crops[i][1])
        out['tOF'] = v
    return out
