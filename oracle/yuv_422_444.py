"""YUV 4:2:2 and 4:4:4 <-> RGB for every colour the stream supports, restated in integer numpy.

This is the specification of tg_stream_frame_in_yuv and tg_rgb_to_yuv for the layouts
  'yuy2' / 'uyvy'  packed 4:2:2, uint8 [..., h, 2w], w even: each pixel pair one 4-byte group Y0 U Y1 V (YUY2,
                   V4L2 YUYV) or U Y0 V Y1 (UYVY, SDI "2vuy")
  'i444'           planar 4:4:4, uint8 [..., 3h, w]: the Y, U and V planes of h x w (ffmpeg yuv444p)
  'i444_10'        the same in uint16 words, sample in the low 10 bits (ffmpeg yuv444p10le); read as min(v, 1023)
The kernels match it bit for bit.  It builds on oracle/yuv_color.py, the specification of the 4:2:0 layouts: the
colour table (coefficients), the colours, the 10-bit quantisation of the fp32 frame and the per-pixel integer
matrices are that module's.  Every function here also accepts the 4:2:0 layouts and hands them to yuv_color.py
unchanged, so a caller can use one module for every layout.

Decode: the per-pixel rule of yuv_color.yuv_to_rgb with nearest chroma (both pixels of a 4:2:2 pair take its U and
V; 4:4:4 has a sample per pixel).  The 'bt601' 8-bit decode is cv2's COLOR_YUV2RGB_YUY2 / _UYVY.

Encode, 4:4:4: the per-pixel integer matrix, no subsampling (I444_10 from the fp32 frame, as P010).

Encode, 4:2:2: U and V of the pair's mean, rounded half up, from the sum of its two pixels (sr = r0 + r1, ...):
  Y = clip((kY . rgb + 2^(sy-1) + (yoff << sy)) >> sy, 0, 255)                     per pixel
  C = clip((kC . (sr, sg, sb) + 2^(sc-1) + (128 << sc)) >> sc, 0, 255)             per pair
The derived colours take the table's encode row with sy = 20, sc = 21.  The 'bt601' row is cv2's
COLOR_RGB2YUV_YUY2 / _UYVY (cv2 4.13), whose 14-bit constants CV2_422 -- luma included -- differ from its 4:2:0
ones: Y = ((4211 R + 8258 G + 1606 B + 8192) >> 14) + 16, C = ((kC . (sr, sg, sb) + 8192) >> 14) + 128.  This
reproduces cv2 on every chroma sum (511^3) and every colour's luma (2^24); tests/golden/yuv422_cv2.npz
(oracle/gen_yuv422_golden.py) pins it.
"""
import numpy as np

from . import yuv_color as C

COLORS = C.COLORS
LAYOUTS_420 = C.LAYOUTS                                          # 'nv12', 'i420', 'p010', 'i420_10'
LAYOUTS_422 = ('yuy2', 'uyvy')                                  # packed 4:2:2, 8 bit
LAYOUTS_444 = ('i444', 'i444_10')                               # planar 4:4:4
LAYOUTS = LAYOUTS_422 + LAYOUTS_444
ALL_LAYOUTS = LAYOUTS_420 + LAYOUTS
# cv2's 4:2:2 encode: (luma per RGB code value, U and V per sum of the pair's two code values, luma shift,
# chroma shift)
CV2_422 = ((4211, 8258, 1606), (-1212, -2384, 3596), (3596, -3015, -582), 14, 14)
_PACKED = {'yuy2': (0, 1), 'uyvy': (1, 0)}                     # byte of Y0 and of U in a 4-byte group

coefficients = C.coefficients
float_matrices = C.float_matrices
quantize10 = C.quantize10
samples10 = C.samples10


def depth_of(layout):
    if layout not in ALL_LAYOUTS:
        raise ValueError(f'layout must be one of {ALL_LAYOUTS}, got {layout!r}')
    return 10 if layout in ('p010', 'i420_10', 'i444_10') else 8


def word_dtype(layout):
    return np.uint16 if depth_of(layout) == 10 else np.uint8


def _check_size(h, w, layout):
    if h <= 0 or w <= 0:
        raise ValueError(f'frame size must be positive, got {h}x{w}')
    if layout in LAYOUTS_422 and w % 2:
        raise ValueError(f'YUV 4:2:2 needs an even width, got {w}')
    if layout in LAYOUTS_420 and (h % 2 or w % 2):
        raise ValueError(f'YUV 4:2:0 needs an even height and width, got {h}x{w}')


def frame_shape(layout, h, w):
    """The [rows, cols] words of one h x w frame: [3h/2, w] (4:2:0), [h, 2w] (4:2:2) or [3h, w] (4:4:4)."""
    depth_of(layout)
    _check_size(h, w, layout)
    if layout in LAYOUTS_422:
        return (h, 2 * w)
    return (3 * h, w) if layout in LAYOUTS_444 else (3 * h // 2, w)


def enc422_coefficients(color):
    """The 4:2:2 encode row: ((kRY, kGY, kBY), (kRU, kGU, kBU), (kRV, kGV, kBV), luma shift, chroma shift); the
    chroma coefficients multiply the sum of a pair's two RGB code values."""
    if color == 'bt601':
        return CV2_422
    c = coefficients(color, 8)
    return tuple(c[0:3]), tuple(c[3:6]), tuple(c[6:9]), c[14], c[14] + 1


def _check_int32(*arrays):
    for a in arrays:
        if a.size and (int(a.max()) >= 1 << 31 or int(a.min()) < -(1 << 31)):
            raise AssertionError('fixed-point intermediate outside int32')


# ------------------------------------------------------------------------------------------------- planes
def split_planes(frame, layout):
    """Frame words ([..., *frame_shape]) -> (Y [..., h, w], U, V) samples (int64) at the layout's depth; U and V are
    [..., h, w/2] (4:2:2), [..., h, w] (4:4:4) or, for 4:2:0, as yuv_color.split_planes."""
    if layout in LAYOUTS_420:
        return C.split_planes(frame, layout)
    frame = np.asarray(frame)
    if frame.dtype != word_dtype(layout):
        raise ValueError(f'{layout} frames are {np.dtype(word_dtype(layout)).name}, got {frame.dtype}')
    v = frame.astype(np.int64)
    if layout == 'i444_10':
        v = np.minimum(v, 1023)
    if layout in LAYOUTS_422:
        w2 = v.shape[-1]
        if w2 % 4:
            raise ValueError(f'a {layout} frame has 2w bytes per row with w even, got {w2}')
        y0, u0 = _PACKED[layout]
        g = v.reshape(*v.shape[:-1], w2 // 4, 4)
        y = np.stack([g[..., y0], g[..., y0 + 2]], axis=-1).reshape(*v.shape[:-1], w2 // 2)
        return y, g[..., u0], g[..., u0 + 2]
    h3 = v.shape[-2]
    if h3 % 3:
        raise ValueError(f'a {layout} frame has 3h rows, got {h3}')
    h = h3 // 3
    return v[..., :h, :], v[..., h:2 * h, :], v[..., 2 * h:, :]


def join_planes(y, u, v, layout):
    """Inverse of split_planes for in-range samples: the layout's words."""
    if layout in LAYOUTS_420:
        return C.join_planes(y, u, v, layout)
    h, w = y.shape[-2:]
    depth_of(layout)
    _check_size(h, w, layout)
    lead = y.shape[:-2]
    if layout in LAYOUTS_422:
        y0, u0 = _PACKED[layout]
        g = np.empty((*lead, h, w // 2, 4), np.int64)
        yy = np.asarray(y).reshape(*lead, h, w // 2, 2)
        g[..., y0], g[..., y0 + 2], g[..., u0], g[..., u0 + 2] = yy[..., 0], yy[..., 1], u, v
        return np.ascontiguousarray(g.reshape(*lead, h, 2 * w).astype(np.uint8))
    return np.ascontiguousarray(np.concatenate([y, u, v], axis=-2).astype(word_dtype(layout)))


# ------------------------------------------------------------------------------------------------- conversions
def yuv_to_rgb(frame, layout, color='bt601'):
    """frame [..., *frame_shape] -> RGB code values [..., h, w, 3] (uint8 at 8 bits, uint16 0..1023 at 10 bits)."""
    if layout in LAYOUTS_420:
        return C.yuv_to_rgb(frame, layout, color)
    depth = depth_of(layout)
    cy, cub, cug, cvg, cvr, s, yoff = coefficients(color, depth)[9:]
    coff, top, half = 1 << (depth - 1), (1 << depth) - 1, 1 << (s - 1)
    y, u, v = split_planes(frame, layout)
    if layout in LAYOUTS_422:                                               # nearest chroma
        u, v = np.repeat(u, 2, axis=-1), np.repeat(v, 2, axis=-1)
    uu, vv = u - coff, v - coff
    ruv, guv, buv = half + cvr * vv, half + cvg * vv + cug * uu, half + cub * uu
    yy = y - yoff
    if color == 'bt601' and depth == 8:
        yy = np.maximum(yy, 0)                                              # cv2's clamp
    yy = yy * cy
    sums = [yy + c for c in (ruv, guv, buv)]
    _check_int32(yy, ruv, guv, buv, *sums)
    rgb = np.stack([np.clip(a >> s, 0, top) for a in sums], axis=-1)
    return rgb.astype(np.uint8 if depth == 8 else np.uint16)


def rgb_to_yuv(rgb, layout, color='bt601'):
    """RGB code values [..., h, w, 3] at the layout's depth -> frame [..., *frame_shape] of the layout's words.
    10-bit layouts take RGB10 codes (quantize10 of the fp32 frame)."""
    if layout in LAYOUTS_420:
        return C.rgb_to_yuv(rgb, layout, color)
    depth = depth_of(layout)
    c = coefficients(color, depth)
    s, yoff = c[14], c[15]
    coff, top, half = 1 << (depth - 1), (1 << depth) - 1, 1 << (s - 1)
    rgb = np.asarray(rgb)
    if rgb.shape[-1] != 3:
        raise ValueError(f'expected RGB [..., h, w, 3], got {rgb.shape}')
    h, w = rgb.shape[-3:-1]
    _check_size(h, w, layout)
    if int(np.max(rgb, initial=0)) > top or int(np.min(rgb, initial=0)) < 0:
        raise ValueError(f'RGB code values outside [0, {top}]')
    r, g, b = (rgb[..., k].astype(np.int64) for k in range(3))
    if layout in LAYOUTS_422:
        ky, ku, kv, sy, sc = enc422_coefficients(color)
        ys = ky[0] * r + ky[1] * g + ky[2] * b + (1 << (sy - 1)) + (yoff << sy)
        sr, sg, sb = (a[..., 0::2] + a[..., 1::2] for a in (r, g, b))            # the pair's sum
        us = ku[0] * sr + ku[1] * sg + ku[2] * sb + (1 << (sc - 1)) + (coff << sc)
        vs = kv[0] * sr + kv[1] * sg + kv[2] * sb + (1 << (sc - 1)) + (coff << sc)
    else:
        ys = c[0] * r + c[1] * g + c[2] * b + half + (yoff << s)
        us = c[3] * r + c[4] * g + c[5] * b + half + (coff << s)
        vs = c[6] * r + c[7] * g + c[8] * b + half + (coff << s)
        sy = sc = s
    _check_int32(ys, us, vs)
    return join_planes(np.clip(ys >> sy, 0, top), np.clip(us >> sc, 0, top), np.clip(vs >> sc, 0, top), layout)


def rgb_f32_to_yuv(rgb_f32, layout, color='bt601'):
    """The 10-bit encode of an fp32 RGB frame [..., h, w, 3]."""
    if depth_of(layout) != 10:
        raise ValueError('the fp32 encode is the 10-bit one')
    return rgb_to_yuv(quantize10(rgb_f32), layout, color)


# ------------------------------------------------------------------------------------------------- test patterns
def yuv_triples_pattern(layout):
    """Every 8-bit (Y, U, V) triple once in a 4096x4096 frame.  4:2:2: pair (r, c) carries
    (U, V) = divmod((r % 32) * 2048 + c, 256) and Y = 2 * (r // 32) + dx; 4:4:4: pixel i holds the triple
    (i >> 16, i >> 8, i) & 255; 4:2:0: yuv_color.yuv_triples_pattern."""
    if depth_of(layout) != 8:
        raise ValueError('the exhaustive pattern is 8-bit')
    if layout in LAYOUTS_422:
        r = np.arange(4096, dtype=np.int64)[:, None]
        c = np.arange(2048, dtype=np.int64)[None, :]
        pair = (r % 32) * 2048 + c
        y = np.stack([np.broadcast_to(2 * (r // 32) + dx, (4096, 2048)) for dx in range(2)], axis=-1)
        return join_planes(y.reshape(4096, 4096), pair >> 8, pair & 255, layout)
    if layout in LAYOUTS_444:
        i = np.arange(1 << 24, dtype=np.int64).reshape(4096, 4096)
        return join_planes((i >> 16) & 255, (i >> 8) & 255, i & 255, layout)
    return C.yuv_triples_pattern(layout)


def yuv10_pattern(layout):
    """'i444_10': one frame [1, 3h, w] with each triple of samples10()^3 at one pixel and 5 % of the words replaced
    by values above 1023 (the decode clamps them); returns (frames, h, w).  4:2:0: yuv_color.yuv10_pattern."""
    if layout != 'i444_10':
        return C.yuv10_pattern(layout)
    s = samples10()
    trip = np.stack(np.meshgrid(s, s, s, indexing='ij'), axis=-1).reshape(-1, 3)
    w = 256
    h = -(-trip.shape[0] // w)
    pad = np.full((h * w - trip.shape[0], 3), 512, np.int64)
    trip = np.concatenate([trip, pad]).reshape(h, w, 3)
    f = join_planes(trip[..., 0], trip[..., 1], trip[..., 2], layout)[None].astype(np.int64)
    rng = np.random.default_rng(10)
    hi = rng.random(f.shape) < 0.05
    f[hi] = rng.integers(1024, 65536, size=int(hi.sum()))
    return np.ascontiguousarray(f.astype(np.uint16)), h, w
