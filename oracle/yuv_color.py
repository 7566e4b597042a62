"""YUV 4:2:0 <-> RGB for every colour the stream supports, restated in integer numpy.

This is the specification of tg_stream_frame_in_yuv and tg_rgb_to_yuv: the kernels match it bit for bit.
oracle/yuv_oracle.py (cv2.cvtColor restated) stays the specification of the 8-bit BT.601 limited-range case,
and the 'bt601' 8-bit row here reproduces it exactly.

Colours:  'bt601', 'bt709' (limited range), 'bt601-full', 'bt709-full'.
Layouts:  'nv12' / 'i420' (uint8), 'p010' (NV12 planes, uint16 words, sample in the high 10 bits: v << 6),
          'i420_10' (I420 planes, uint16 words, sample in the low 10 bits; ffmpeg's yuv420p10le).
Frames are [..., 3h/2, w] of the layout's word type, planes as in yuv_oracle.py.

Coefficients are derived from (Kr, Kb) with the quantisation of ITU-T H.273 for bit depth n:
  limited  Y = 16*2^(n-8) + 219*2^(n-8)*E'Y,   C = 128*2^(n-8) + 224*2^(n-8)*E'C
  full     Y = (2^n-1)*E'Y,                    C = 2^(n-1) + (2^n-1)*E'C
and rounded to SHIFT[n]-bit fixed point (20 bits at 8 bits, 18 at 10 bits, so that every intermediate fits in
int32).  Encode of an RGB code triple (r, g, b) at depth n:
  Y = clip((cRY*r + cGY*g + cBY*b + HALF + (yoff << S)) >> S, 0, 2^n-1), likewise U, V with the offset 2^(n-1)
Decode:
  R = clip(((Y - yoff)*CY + CVR*(V - coff) + HALF) >> S, 0, 2^n-1), and so on.
The 'bt601' 8-bit row keeps cv2's constants and its clamp max(Y - 16, 0) before the multiply; the derived rows
leave Y - yoff unclamped and clamp only the result, as H.273 does.

Chroma siting as in yuv_oracle.py: nearest chroma on decode, the top-left pixel of each 2x2 block on encode.
10-bit decode reads P010 words as v >> 6 and I420_10 words as min(v, 1023); the stream's input is then
float32(RGB10) / 1023.  10-bit encode takes the fp32 RGB frame: q = clip(rint(float32(x) * 1023), 0, 1023)
(round half to even), then the integer matrix; P010 stores the result << 6.
"""
import math

import numpy as np

from . import yuv_oracle as Y8

COLORS = ('bt601', 'bt709', 'bt601-full', 'bt709-full')      # index = table row, as in tg_stream.cu
LAYOUTS = ('nv12', 'i420', 'p010', 'i420_10')
KRKB = {601: (0.299, 0.114), 709: (0.2126, 0.0722)}
SHIFT = {8: 20, 10: 18}
# tg_yuv_coefficients order
NAMES = ('cRY', 'cGY', 'cBY', 'cRU', 'cGU', 'cBU', 'cRV', 'cGV', 'cBV', 'CY', 'CUB', 'CUG', 'CVG', 'CVR',
         'shift', 'yoff')


def parse_color(color):
    """'bt709-full' -> (709, True)."""
    if color not in COLORS:
        raise ValueError(f'colour must be one of {COLORS}, got {color!r}')
    return (709 if color.startswith('bt709') else 601), color.endswith('-full')


def depth_of(layout):
    if layout not in LAYOUTS:
        raise ValueError(f'layout must be one of {LAYOUTS}, got {layout!r}')
    return 10 if layout in ('p010', 'i420_10') else 8


def word_dtype(layout):
    return np.uint16 if depth_of(layout) == 10 else np.uint8


def _rnd(x):
    """Round half away from zero (the C side's rule; ties do not occur in the table)."""
    return int(math.floor(abs(x) + 0.5)) * (1 if x >= 0 else -1)


def float_matrices(color, depth):
    """float64 (enc [3,3] per RGB code value, offsets (yoff, coff), dec (CY, CUB, CUG, CVG, CVR)) of H.273."""
    matrix, full = parse_color(color)
    kr, kb = KRKB[matrix]
    kg = 1.0 - kr - kb
    d = float((1 << depth) - 1)
    sc = float(1 << (depth - 8))
    ky, kc, yoff = (d, d, 0) if full else (219.0 * sc, 224.0 * sc, 16 << (depth - 8))
    enc = [[kr * ky / d, kg * ky / d, kb * ky / d],
           [-kr / (2.0 * (1.0 - kb)) * kc / d, -kg / (2.0 * (1.0 - kb)) * kc / d, 0.5 * kc / d],
           [0.5 * kc / d, -kg / (2.0 * (1.0 - kr)) * kc / d, -kb / (2.0 * (1.0 - kr)) * kc / d]]
    dec = [d / ky, d * 2.0 * (1.0 - kb) / kc, -d * 2.0 * (1.0 - kb) * kb / (kg * kc),
           -d * 2.0 * (1.0 - kr) * kr / (kg * kc), d * 2.0 * (1.0 - kr) / kc]
    return enc, (yoff, 1 << (depth - 1)), dec


def coefficients(color, depth):
    """The 16 int32 of tg_yuv_coefficients (NAMES order) for a colour at bit depth 8 or 10."""
    if depth not in SHIFT:
        raise ValueError(f'bit depth must be 8 or 10, got {depth}')
    if color == 'bt601' and depth == 8:
        return [Y8.CRY, Y8.CGY, Y8.CBY, Y8.CRU, Y8.CGU, Y8.CBU, Y8.CRV, Y8.CGV, Y8.CBV,
                Y8.CY, Y8.CUB, Y8.CUG, Y8.CVG, Y8.CVR, Y8.SHIFT, 16]
    enc, (yoff, _), dec = float_matrices(color, depth)
    one = float(1 << SHIFT[depth])
    return [_rnd(c * one) for row in enc for c in row] + [_rnd(c * one) for c in dec] + [SHIFT[depth], yoff]


def _check_int32(*arrays):
    for a in arrays:
        if a.size and (int(a.max()) >= 1 << 31 or int(a.min()) < -(1 << 31)):
            raise AssertionError('fixed-point intermediate outside int32')


# ------------------------------------------------------------------------------------------------- planes
def split_planes(frame, layout):
    """[..., 3h/2, w] words -> (Y, U, V) samples (int64) at the layout's depth."""
    frame = np.asarray(frame)
    if frame.dtype != word_dtype(layout):
        raise ValueError(f'{layout} frames are {np.dtype(word_dtype(layout)).name}, got {frame.dtype}')
    v = frame.astype(np.int64)
    if layout == 'p010':
        v = v >> 6
    elif layout == 'i420_10':
        v = np.minimum(v, 1023)
    return Y8.split_planes(v, 'nv12' if layout in ('nv12', 'p010') else 'i420')


def join_planes(y, u, v, layout):
    """Inverse of split_planes for in-range samples: the layout's words."""
    h, w = y.shape[-2:]
    Y8._check(h, w, 'nv12')
    lead = y.shape[:-2]
    if layout in ('nv12', 'p010'):
        c = np.stack([u, v], axis=-1).reshape(*lead, h // 2, w)
    else:
        c = np.concatenate([u.reshape(*lead, -1), v.reshape(*lead, -1)], axis=-1).reshape(*lead, h // 2, w)
    out = np.concatenate([y, c], axis=-2).astype(np.int64)
    if layout == 'p010':
        out = out << 6
    return np.ascontiguousarray(out.astype(word_dtype(layout)))


# ------------------------------------------------------------------------------------------------- conversions
def yuv_to_rgb(frame, layout, color='bt601'):
    """frame [..., 3h/2, w] -> RGB code values [..., h, w, 3] (uint8 at 8 bits, uint16 0..1023 at 10 bits)."""
    depth = depth_of(layout)
    cy, cub, cug, cvg, cvr, s, yoff = coefficients(color, depth)[9:]
    coff, top, half = 1 << (depth - 1), (1 << depth) - 1, 1 << (s - 1)
    y, u, v = split_planes(frame, layout)
    uu, vv = u - coff, v - coff
    ruv, guv, buv = half + cvr * vv, half + cvg * vv + cug * uu, half + cub * uu
    up = lambda a: np.repeat(np.repeat(a, 2, axis=-2), 2, axis=-1)            # nearest chroma
    yy = y - yoff
    if color == 'bt601' and depth == 8:
        yy = np.maximum(yy, 0)                                                  # cv2's clamp
    yy = yy * cy
    sums = [yy + up(c) for c in (ruv, guv, buv)]
    _check_int32(yy, ruv, guv, buv, *sums)
    rgb = np.stack([np.clip(a >> s, 0, top) for a in sums], axis=-1)
    return rgb.astype(np.uint8 if depth == 8 else np.uint16)


def quantize10(x):
    """fp32 [...] -> RGB10 code values: clip(rint(float32(x) * 1023f), 0, 1023), round half to even."""
    q = np.rint(np.asarray(x, dtype=np.float32) * np.float32(1023.0))
    return np.clip(q, 0, 1023).astype(np.int64)


def rgb_to_yuv(rgb, layout, color='bt601'):
    """RGB code values [..., h, w, 3] at the layout's depth -> frame [..., 3h/2, w] of the layout's words.
    10-bit layouts take RGB10 codes (quantize10 of the fp32 frame)."""
    depth = depth_of(layout)
    c = coefficients(color, depth)
    s, yoff = c[14], c[15]
    coff, top, half = 1 << (depth - 1), (1 << depth) - 1, 1 << (s - 1)
    rgb = np.asarray(rgb)
    if rgb.shape[-1] != 3:
        raise ValueError(f'expected RGB [..., h, w, 3], got {rgb.shape}')
    h, w = rgb.shape[-3:-1]
    Y8._check(h, w, 'nv12')
    r, g, b = (rgb[..., k].astype(np.int64) for k in range(3))
    if int(np.max(rgb, initial=0)) > top or int(np.min(rgb, initial=0)) < 0:
        raise ValueError(f'RGB code values outside [0, {top}]')
    ys = c[0] * r + c[1] * g + c[2] * b + half + (yoff << s)
    y = np.clip(ys >> s, 0, top)
    r, g, b = (a[..., ::2, ::2] for a in (r, g, b))                            # top-left pixel of each 2x2 block
    us = c[3] * r + c[4] * g + c[5] * b + half + (coff << s)
    vs = c[6] * r + c[7] * g + c[8] * b + half + (coff << s)
    _check_int32(ys, us, vs)
    return join_planes(y, np.clip(us >> s, 0, top), np.clip(vs >> s, 0, top), layout)


def rgb_f32_to_yuv(rgb_f32, layout, color='bt601'):
    """The 10-bit encode of an fp32 RGB frame [..., h, w, 3]."""
    if depth_of(layout) != 10:
        raise ValueError('the fp32 encode is the 10-bit one')
    return rgb_to_yuv(quantize10(rgb_f32), layout, color)


# ------------------------------------------------------------------------------------------------- float64 H.273
def float_rgb_to_yuv(rgb, depth, color):
    """float64 H.273 encode of per-pixel RGB codes [..., 3] -> YUV codes [..., 3] (rounded, clipped)."""
    enc, (yoff, coff), _ = float_matrices(color, depth)
    x = np.asarray(rgb, dtype=np.float64) @ np.asarray(enc).T + np.array([yoff, coff, coff], np.float64)
    return np.clip(np.rint(x), 0, (1 << depth) - 1).astype(np.int64)


def float_yuv_to_rgb(yuv, depth, color):
    """float64 H.273 decode of per-pixel YUV codes [..., 3] -> RGB codes [..., 3] (rounded, clipped)."""
    _, (yoff, coff), (cy, cub, cug, cvg, cvr) = float_matrices(color, depth)
    yuv = np.asarray(yuv, dtype=np.float64)
    yy, uu, vv = yuv[..., 0] - yoff, yuv[..., 1] - coff, yuv[..., 2] - coff
    rgb = np.stack([cy * yy + cvr * vv, cy * yy + cug * uu + cvg * vv, cy * yy + cub * uu], axis=-1)
    return np.clip(np.rint(rgb), 0, (1 << depth) - 1).astype(np.int64)


# ------------------------------------------------------------------------------------------------- test patterns
def yuv_triples_pattern(layout):
    """yuv_oracle.yuv_triples_pattern in any 8-bit layout: every (Y, U, V) triple once in a 4096x4096 frame."""
    if depth_of(layout) != 8:
        raise ValueError('the exhaustive pattern is 8-bit')
    return Y8.yuv_triples_pattern(layout)


def samples10():
    """The dense 10-bit sample values: every multiple of 31 and the edges 0, 1, 63, 64, 65, 511, 512, 513, 939,
    940, 941, 959, 960, 961, 1022, 1023."""
    edges = [0, 1, 63, 64, 65, 511, 512, 513, 939, 940, 941, 959, 960, 961, 1022, 1023]
    return np.unique(np.concatenate([np.arange(0, 1024, 31), edges])).astype(np.int64)


def yuv10_pattern(layout):
    """10-bit frames [m, 3h/2, w] that hold every (Y, U, V) of samples10()^3 (Y per pixel, (U, V) per 2x2 block) as
    words of the layout; returns (frames, h, w).  P010 words carry junk in their low 6 bits (the decode ignores it);
    5 % of the I420_10 words are replaced by values above 1023 (the decode clamps them), so only P010 covers every
    triple exactly."""
    s = samples10()
    m = s.size
    uu, vv = np.meshgrid(s, s, indexing='ij')                       # m x m chroma blocks
    uu, vv = uu.reshape(-1), vv.reshape(-1)
    nb = uu.size
    per_row = 64                                                    # blocks per chroma row
    rows = -(-nb // per_row)
    ub = np.full(rows * per_row, 512, np.int64)
    vb = ub.copy()
    ub[:nb], vb[:nb] = uu, vv
    u, v = ub.reshape(rows, per_row), vb.reshape(rows, per_row)
    h, w = 2 * rows, 2 * per_row
    # luma cycles through samples10 (7 is coprime with m); frame k shifts that cycle by k pixels, so over the m
    # frames every pixel of every block takes every Y
    y = s[(np.arange(h * w).reshape(h, w) * 7) % m]
    frames = [join_planes(np.roll(y.reshape(-1), k).reshape(h, w), u, v, layout) for k in range(m)]
    f = np.stack(frames).astype(np.int64)
    rng = np.random.default_rng(10)
    if layout == 'p010':
        f |= rng.integers(0, 64, size=f.shape)
    else:
        hi = rng.random(f.shape) < 0.05
        f[hi] = rng.integers(1024, 65536, size=int(hi.sum()))
    return np.ascontiguousarray(f.astype(np.uint16)), h, w
