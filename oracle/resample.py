"""Antialiased bicubic / Lanczos-3 resize of fp32 NCHW frames, restated in float64 numpy.

This is the specification of tg_resample_table and tg_resample_nchw_f32 (the streamed output's resize).  The
filters are Pillow's: Image.resize(size, BICUBIC | LANCZOS) on mode 'F' images (reducing_gap=None, no box).  For
one axis, in -> out:

  scale   = in / out;  fs = max(scale, 1);  support = S * fs       S = 2 (bicubic), 3 (lanczos)
  center  = (o + 0.5) * scale
  xmin    = max(int(center - support + 0.5), 0);  xmax = min(int(center + support + 0.5), in)
  w[x]    = K((x - center + 0.5) / fs) for x in [xmin, xmax), then w /= sum(w)
  bicubic K(x), a = -0.5:  |x| < 1: ((a+2)|x| - (a+3))x^2 + 1;  1 <= |x| < 2: a(|x|^3 - 5x^2 + 8|x| - 4);  else 0
  lanczos K(x):            |x| < 3: sinc(x) sinc(x/3);  else 0

A downscale widens the kernel by the ratio (antialiasing); an upscale uses it as is.  The resize is separable,
horizontal then vertical, summed in float64 (Pillow rounds the intermediate and the result to float32).

Table form (what the kernel reads): per output index o a window start first[o] and taps = 2 * ceil(support) + 1
weights, the window's weights at offset xmin - first and zeros elsewhere.  The window is placed so that it ends
inside the axis (first = max(0, min(xmin, in - taps))), so a padding tap never indexes outside the image; on an axis
shorter than taps the kernel clamps the index.  The kernel's weights are the float32 rounding of these.

Each axis needs in/4 <= out <= 2*in, which bounds taps at 17 (bicubic) and 25 (lanczos).

torch.nn.functional.interpolate(antialias=True) is not this specification: it differs from Pillow by up to 1.4e-5
at non-integer ratios and only serves as a loose cross-check for bicubic.  ffmpeg's `scale` filter uses other
parameters (swscale's bicubic is B=0, C=0.6) and does not give the same values either.

uint8 output: float32_to_uint8 of the float32 resized value, clip(rint_half_even(x * 255), 0, 255).  10-bit YUV
output: oracle/yuv_color.py's encode of the float32 resized frame.
"""
import math

import numpy as np

FILTERS = ('bicubic', 'lanczos')
SUPPORT = {'bicubic': 2.0, 'lanczos': 3.0}
MAX_TAPS = 25


def _bicubic(x):
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1.0
    if x < 2.0:
        return (((x - 5.0) * x + 8.0) * x - 4.0) * a
    return 0.0


def _sinc(x):
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _lanczos(x):
    return _sinc(x) * _sinc(x / 3.0) if -3.0 <= x < 3.0 else 0.0


_KERNEL = {'bicubic': _bicubic, 'lanczos': _lanczos}


def check_ratio(n_in, n_out):
    """True when in/4 <= out <= 2*in (both positive)."""
    return n_in > 0 and n_out > 0 and 4 * n_out >= n_in and n_out <= 2 * n_in


def taps(n_in, n_out, filt):
    """Table width of one axis: 2 * ceil(support) + 1."""
    if filt not in FILTERS:
        raise ValueError(f'filter must be one of {FILTERS}, got {filt!r}')
    return 2 * math.ceil(SUPPORT[filt] * max(n_in / n_out, 1.0)) + 1


def windows(n_in, n_out, filt):
    """Per output index: (xmin, normalised float64 weights of [xmin, xmax)), Pillow's precompute_coeffs.
    Scalar Python floats throughout, so the arithmetic is the C library's double arithmetic term for term."""
    kern = _KERNEL[filt]
    scale = n_in / n_out
    fs = max(scale, 1.0)
    support = SUPPORT[filt] * fs
    ss = 1.0 / fs
    out = []
    for o in range(n_out):
        center = (o + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), n_in)
        w = [kern((x - center + 0.5) * ss) for x in range(xmin, xmax)]
        tot = 0.0
        for v in w:
            tot += v
        if tot != 0.0:
            w = [v / tot for v in w]
        out.append((xmin, w))
    return out


def table(n_in, n_out, filt):
    """(first int32 [out], weights float64 [out, taps]) with the window placed to end inside the axis."""
    k = taps(n_in, n_out, filt)
    first = np.zeros(n_out, np.int32)
    wt = np.zeros((n_out, k), np.float64)
    for o, (xmin, w) in enumerate(windows(n_in, n_out, filt)):
        f = max(0, min(xmin, n_in - k))
        first[o] = f
        wt[o, xmin - f:xmin - f + len(w)] = w
    return first, wt


def table_f32(n_in, n_out, filt):
    """The kernel's table: the float32 rounding of table()'s weights."""
    first, wt = table(n_in, n_out, filt)
    return first, wt.astype(np.float32)


def matrix(n_in, n_out, filt):
    """Dense float64 [out, in] resampling matrix of one axis."""
    m = np.zeros((n_out, n_in), np.float64)
    for o, (xmin, w) in enumerate(windows(n_in, n_out, filt)):
        m[o, xmin:xmin + len(w)] = w
    return m


def resize(x, out_hw, filt='bicubic'):
    """float [..., H, W] -> float64 [..., Ho, Wo]: horizontal, then vertical, in float64."""
    x = np.asarray(x, dtype=np.float64)
    H, W = x.shape[-2:]
    Ho, Wo = out_hw
    if not (check_ratio(H, Ho) and check_ratio(W, Wo)):
        raise ValueError(f'resize {H}x{W} -> {Ho}x{Wo}: each axis needs in/4 <= out <= 2*in')
    return matrix(H, Ho, filt) @ (x @ matrix(W, Wo, filt).T)


def to_uint8(y):
    """float32_to_uint8 of the float32 value: clip(rint(float32(y) * 255), 0, 255), round half to even."""
    return np.clip(np.rint(np.asarray(y, dtype=np.float32) * np.float32(255.0)), 0, 255).astype(np.uint8)


def resize_u8_nhwc(x_nchw, out_hw, filt='bicubic'):
    """fp32 NCHW [n,c,H,W] -> the uint8 NHWC [n,Ho,Wo,c] the kernel writes."""
    return np.ascontiguousarray(to_uint8(resize(x_nchw, out_hw, filt)).transpose(0, 2, 3, 1))


def near_boundary(y, tol=1e-3):
    """True where y * 255 lies within tol of a rounding boundary (k + 0.5): float32 sums may round either way."""
    v = np.asarray(y, dtype=np.float64) * 255.0
    return np.abs(v - np.floor(v) - 0.5) < tol
