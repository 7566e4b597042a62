"""TecoGAN's official metric script (codes/official_metrics/metrics.py, the script behind the paper's tables),
restated in float64 numpy + scipy + cv2, without LPIPS / tLP.

This is the specification of tecogan_b200.metrics.official_sequence_metrics / official_averages:

  to_uint8   x.astype(float32) / 255 * 255, rounded and clipped: the identity on uint8 frames
  Y          the Y row of _rgb2ycbcr(maxVal=255): float64 0.256788235294118 R + 0.504129411764706 G
             + 0.097905882352941 B + 16, never rounded
  crop_8x8   per side n: the largest multiple of 32 that is <= n - 16, at offset (n - size) // 2
  PSNR       20 log10(255 / sqrt(mean((Yt - Yp)^2))) on the crop_8x8 of the frames; inf on equal frames
  SSIM       skimage 0.16 compare_ssim(Yt, Yp, data_range=Yp.max() - Yp.min()) on the crop: 7x7 uniform_filter
             moments, covariances scaled by 49/48, C1 = (0.01 R)^2, C2 = (0.03 R)^2, mean of S[3:-3, 3:-3]
  tOF        the mean per-pixel L2 norm of the difference of the crop_8x8 of two cv2 Farneback flows (0.5, 3, 15, 3,
             5, 1.2, 0), computed on the uncropped gray frames (cv2 COLOR_RGB2GRAY), in float32 as the script does
  frames     both frames are first cut to their common top-left size; frames cutfr .. T - cutfr - 1 are scored,
             tOF from frame cutfr + 1 on (pair i - 1 -> i)
  totals     per sequence the float32 cast of each list, its sum and mean; FrameAvg = all sums / all lengths,
             FolderAvg = mean of the per-sequence means, Avg = float32 [per-sequence means]

skimage is not needed: ssim() is the formula, checked against a direct 7x7 window sum.
"""
import cv2
import numpy as np
import scipy.ndimage as nd

T_Y = (0.256788235294118, 0.504129411764706, 0.097905882352941)
FLOW_ARGS = (None, 0.5, 3, 15, 3, 5, 1.2, 0)
KEYS = ('PSNR', 'SSIM', 'tOF')


def to_uint8(x, vmin, vmax):
    x = x.astype('float32')
    x = (x - vmin) / (vmax - vmin) * 255
    return np.clip(np.round(x), 0, 255)


def rgb_to_y(img):
    """float64 Y of _rgb2ycbcr(img, 255), left to right, no FMA"""
    x = np.asarray(img).astype(np.float64)
    return x[..., 0] * T_Y[0] + x[..., 1] * T_Y[1] + x[..., 2] * T_Y[2] + 16.0


def crop_8x8(n):
    """(offset, size) along one side of n pixels; the slice [offset:offset + size] is crop_8x8's"""
    size = (n // 32) * 32
    while size > n - 16:
        size -= 32
    return (n - size) // 2, size


def crop(img):
    (y, h), (x, w) = crop_8x8(img.shape[0]), crop_8x8(img.shape[1])
    return img[y:y + h, x:x + w]


def psnr(yt, yp):
    diff = yt - yp
    rmse = np.sqrt(np.mean(np.power(diff, 2)))
    with np.errstate(divide='ignore'):
        return 20 * np.log10(255. / rmse)


def ssim(x, y, data_range):
    """skimage.measure.compare_ssim(x, y, data_range=data_range) with its defaults (skimage 0.16)"""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    ux, uy = nd.uniform_filter(x, size=7), nd.uniform_filter(y, size=7)
    uxx, uyy, uxy = (nd.uniform_filter(a, size=7) for a in (x * x, y * y, x * y))
    cov_norm = 49 / 48
    vx, vy, vxy = cov_norm * (uxx - ux * ux), cov_norm * (uyy - uy * uy), cov_norm * (uxy - ux * uy)
    c1, c2 = (0.01 * data_range) ** 2, (0.03 * data_range) ** 2
    with np.errstate(divide='ignore', invalid='ignore'):
        s = ((2 * ux * uy + c1) * (2 * vxy + c2)) / ((ux ** 2 + uy ** 2 + c1) * (vx + vy + c2))
    return s[3:-3, 3:-3].mean()


def ssim_direct(x, y, data_range):
    """ssim() by explicit 7x7 window sums (sliding_window_view), the independent restatement it is checked against"""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    win = np.lib.stride_tricks.sliding_window_view

    def mean7(a):
        return win(a, (7, 7)).sum(axis=(-2, -1)) / 49
    ux, uy = mean7(x), mean7(y)
    vx = (mean7(x * x) - ux * ux) * 49 / 48
    vy = (mean7(y * y) - uy * uy) * 49 / 48
    vxy = (mean7(x * y) - ux * uy) * 49 / 48
    c1, c2 = (0.01 * data_range) ** 2, (0.03 * data_range) ** 2
    with np.errstate(divide='ignore', invalid='ignore'):
        s = (2 * ux * uy + c1) * (2 * vxy + c2) / ((ux * ux + uy * uy + c1) * (vx + vy + c2))
    return s.mean()


def ssim_y(true_img, pred_img):
    yt, yp = rgb_to_y(to_uint8(true_img, 0, 255)), rgb_to_y(to_uint8(pred_img, 0, 255))
    return ssim(yt, yp, data_range=yp.max() - yp.min())


def sequence_metrics(true_seq, pred_seq, cutfr=2, keys=KEYS):
    """{key: float64 array} of uint8 RGB sequences [T, H, W, 3], as the script's frame loop computes them"""
    lists = {k: [] for k in keys}
    T = len(true_seq)
    pre = None
    for i in range(cutfr, T - cutfr):
        out, tar = np.asarray(pred_seq[i]), np.asarray(true_seq[i])
        h, w = min(out.shape[0], tar.shape[0]), min(out.shape[1], tar.shape[1])
        out, tar = out[:h, :w], tar[:h, :w]
        if 'tOF' in keys:
            grey = (cv2.cvtColor(np.ascontiguousarray(tar), cv2.COLOR_RGB2GRAY),
                    cv2.cvtColor(np.ascontiguousarray(out), cv2.COLOR_RGB2GRAY))
            if i > cutfr:
                t_of = cv2.calcOpticalFlowFarneback(pre[0], grey[0], *FLOW_ARGS)
                o_of = cv2.calcOpticalFlowFarneback(pre[1], grey[1], *FLOW_ARGS)
                d = np.absolute(crop(t_of) - crop(o_of))
                lists['tOF'].append(np.sqrt(np.sum(d * d, axis=-1)).mean())
            pre = grey
        tar, out = crop(tar), crop(out)
        if 'PSNR' in keys:
            lists['PSNR'].append(psnr(rgb_to_y(to_uint8(tar, 0, 255)), rgb_to_y(to_uint8(out, 0, 255))))
        if 'SSIM' in keys:
            lists['SSIM'].append(ssim_y(tar, out))
    return {k: np.asarray(v, np.float64) for k, v in lists.items()}


def averages(per_sequence):
    """the script's totals over sequences (its folders): FrameAvg_*, FolderAvg_*, Avg_*"""
    keys = list(per_sequence[0])
    sums, lens, folder, avg = dict.fromkeys(keys, 0), dict.fromkeys(keys, 0), dict.fromkeys(keys, 0), {}
    for d in per_sequence:
        for k in keys:
            cur = np.float32(d[k])
            s = cur.sum()
            mean = s / cur.shape[0]
            avg.setdefault(k, []).append(mean)
            sums[k] += s
            lens[k] += cur.shape[0]
            folder[k] += mean
    out = {}
    for k in keys:
        out['FrameAvg_' + k] = sums[k] / lens[k]
        out['FolderAvg_' + k] = folder[k] / len(per_sequence)
        out['Avg_' + k] = np.float32(avg[k])
    return out
