"""10-bit YUV 4:2:2 <-> RGB for every colour the stream supports, restated in integer numpy.

This is the specification of tg_stream_frame_in_yuv, tg_rgb_to_yuv, tg_fill_black and tg_luma_line_sums (and their
window variants) for the layouts
  'p210'     uint16 [..., 2h, w]: the h x w Y plane, then a full-height interleaved UV plane (U0 V0 U1 V1 ... per
             row, one (U, V) per pixel pair); each sample in the high 10 bits (v << 6), as P010
  'i422_10'  uint16 [..., 2h, w]: the Y plane, then the U and V planes of h x w/2; each sample in the low 10 bits,
             read as min(v, 1023), as I420_10 and I444_10 (ffmpeg yuv422p10le)
  'v210'     uint8 [..., h, S] with S = v210_stride(w) = 128 * ceil(w / 48) bytes a row (SDI, ffmpeg v210).  Each
             16-byte group holds 6 pixels as four little-endian 32-bit words Cb0 Y0 Cr0 | Y1 Cb2 Y2 | Cr2 Y3 Cb4 |
             Y4 Cr4 Y5, the 10-bit fields at bits 0, 10 and 20, bits 30-31 zero.  A row's ceil(w / 6) groups hold its
             pixels; the unused fields of a partial last group and the padding up to S are 0 in encoded frames and
             ignored on decode.  S does not give w, so every function here takes it.
All three need an even w; h may be odd.  The kernels match this module bit for bit.

It builds on oracle/yuv_color.py (the colour table, the colours, the 10-bit quantisation of the fp32 frame) and
oracle/yuv_422_444.py (the 4:2:2 rules):
  Decode: the 10-bit row's per-pixel rule with nearest chroma, both pixels of a pair take its U and V
          (yuv_422_444.yuv_to_rgb's rule at 10 bits).
  Encode: q = clip(rint(x * 1023), 0, 1023) of the fp32 frame; Y per pixel with the 10-bit row, as the I444_10
          encode; U and V from the pair's sum q0 + q1 with one more fraction bit, rounded half up:
            C = clip((kC . (q0 + q1) + 2^18 + (512 << 19)) >> 19, 0, 1023)
          the rule the derived 8-bit 4:2:2 rows use (enc422_coefficients: shift + 1), on the 10-bit row.
  Black:  Y = the colour's luma offset (64 limited, 0 full), U = V = 512.
  Windows: a picture of h x w at (top, left) of an fh x fw frame; 4:2:2 needs fw and left even, and a v210 picture
          starts on a group (left % 6 == 0) and ends on one unless it reaches the frame's right edge.  A windowed
          encode writes the picture's samples (v210: its groups) and nothing else; a whole-frame v210 encode writes
          every byte of each row.
"""
import numpy as np

from . import yuv_422_444 as Q
from . import yuv_color as C

COLORS = C.COLORS
LAYOUTS = ('p210', 'i422_10', 'v210')
SHIFT = C.SHIFT[10]                  # 18: the 10-bit row's fraction bits; the chroma of a pair sum takes 19

coefficients = C.coefficients
quantize10 = C.quantize10
samples10 = C.samples10

# field of a v210 group (3 * word + k at bits 10k of that word) holding Y of pixel j, and Cb / Cr of pair p
Y_FIELD = tuple(2 * j + 1 for j in range(6))
U_FIELD = (0, 4, 8)
V_FIELD = (2, 6, 10)


def _check_layout(layout):
    if layout not in LAYOUTS:
        raise ValueError(f'layout must be one of {LAYOUTS}, got {layout!r}')


def word_dtype(layout):
    _check_layout(layout)
    return np.uint8 if layout == 'v210' else np.uint16


def v210_stride(w):
    """Bytes per row of a v210 frame w pixels wide."""
    return 128 * (-(-w // 48))


def check_size(h, w):
    if h <= 0 or w <= 0:
        raise ValueError(f'frame size must be positive, got {h}x{w}')
    if w % 2:
        raise ValueError(f'YUV 4:2:2 needs an even width, got {w}')


def frame_shape(layout, h, w):
    """The [rows, cols] words of one h x w frame: [2h, w] (P210, I422_10) or [h, v210_stride(w)] bytes (v210)."""
    _check_layout(layout)
    check_size(h, w)
    return (h, v210_stride(w)) if layout == 'v210' else (2 * h, w)


# ------------------------------------------------------------------------------------------------- v210 packing
def pack_v210(y, u, v):
    """Samples Y [..., h, w], U, V [..., h, w/2] (0..1023) -> v210 bytes [..., h, v210_stride(w)], unused fields and
    the row padding 0."""
    y, u, v = (np.asarray(a, dtype=np.int64) for a in (y, u, v))
    h, w = y.shape[-2:]
    check_size(h, w)
    lead = y.shape[:-2]
    groups = -(-w // 6)
    f = np.zeros((*lead, h, groups, 12), np.int64)
    yp = np.zeros((*lead, h, 6 * groups), np.int64)
    yp[..., :w] = y
    up, vp = (np.zeros((*lead, h, 3 * groups), np.int64) for _ in range(2))
    up[..., :w // 2], vp[..., :w // 2] = u, v
    f[..., list(Y_FIELD)] = yp.reshape(*lead, h, groups, 6)
    f[..., list(U_FIELD)] = up.reshape(*lead, h, groups, 3)
    f[..., list(V_FIELD)] = vp.reshape(*lead, h, groups, 3)
    words = (f[..., 0::3] | (f[..., 1::3] << 10) | (f[..., 2::3] << 20)).astype('<u4')
    row = words.reshape(*lead, h, 4 * groups).view(np.uint8)            # little-endian bytes
    out = np.zeros((*lead, h, v210_stride(w)), np.uint8)
    out[..., :16 * groups] = row
    return out


def unpack_v210(frame, w):
    """v210 bytes [..., h, v210_stride(w)] -> (Y [..., h, w], U, V [..., h, w/2]) samples (int64)."""
    frame = np.asarray(frame)
    if frame.dtype != np.uint8:
        raise ValueError(f'v210 frames are uint8, got {frame.dtype}')
    h, s = frame.shape[-2:]
    check_size(h, w)
    if s != v210_stride(w):
        raise ValueError(f'a v210 row of {w} pixels is {v210_stride(w)} bytes, got {s}')
    lead = frame.shape[:-2]
    groups = -(-w // 6)
    words = np.ascontiguousarray(frame[..., :16 * groups]).view('<u4').astype(np.int64)
    words = words.reshape(*lead, h, groups, 4)
    f = np.stack([(words >> (10 * k)) & 1023 for k in range(3)], axis=-1).reshape(*lead, h, groups, 12)
    y = f[..., list(Y_FIELD)].reshape(*lead, h, 6 * groups)[..., :w]
    u = f[..., list(U_FIELD)].reshape(*lead, h, 3 * groups)[..., :w // 2]
    v = f[..., list(V_FIELD)].reshape(*lead, h, 3 * groups)[..., :w // 2]
    return y, u, v


# ------------------------------------------------------------------------------------------------- planes
def split_planes(frame, layout, w=None):
    """Frame words -> (Y [..., h, w], U, V [..., h, w/2]) samples (int64).  v210 needs w."""
    _check_layout(layout)
    frame = np.asarray(frame)
    if frame.dtype != word_dtype(layout):
        raise ValueError(f'{layout} frames are {np.dtype(word_dtype(layout)).name}, got {frame.dtype}')
    if layout == 'v210':
        if w is None:
            raise ValueError('v210 frames do not give their width: pass w')
        return unpack_v210(frame, w)
    h2, fw = frame.shape[-2:]
    if h2 % 2 or fw % 2:
        raise ValueError(f'a {layout} frame has 2h rows of w words with w even, got {h2}x{fw}')
    if w is not None and w != fw:
        raise ValueError(f'{layout} frames of {fw} words a row are {fw} wide, not {w}')
    h = h2 // 2
    x = frame.astype(np.int64)
    x = x >> 6 if layout == 'p210' else np.minimum(x, 1023)
    y, c = x[..., :h, :], x[..., h:, :]
    if layout == 'p210':
        return y, c[..., 0::2], c[..., 1::2]
    c = c.reshape(*c.shape[:-2], 2, h, fw // 2)                          # the U plane, then the V plane
    return y, c[..., 0, :, :], c[..., 1, :, :]


def join_planes(y, u, v, layout):
    """Inverse of split_planes for in-range samples: the layout's words."""
    _check_layout(layout)
    y, u, v = (np.asarray(a, dtype=np.int64) for a in (y, u, v))
    h, w = y.shape[-2:]
    check_size(h, w)
    if layout == 'v210':
        return pack_v210(y, u, v)
    lead = y.shape[:-2]
    if layout == 'p210':
        c = np.stack([u, v], axis=-1).reshape(*lead, h, w)
        return np.ascontiguousarray((np.concatenate([y, c], axis=-2) << 6).astype(np.uint16))
    c = np.concatenate([u.reshape(*lead, -1), v.reshape(*lead, -1)], axis=-1).reshape(*lead, h, w)
    return np.ascontiguousarray(np.concatenate([y, c], axis=-2).astype(np.uint16))


# ------------------------------------------------------------------------------------------------- conversions
def yuv_to_rgb(frame, layout, color='bt601', w=None):
    """frame -> RGB10 code values uint16 [..., h, w, 3] (the stream's input is float32(code) / 1023)."""
    cy, cub, cug, cvg, cvr, s, yoff = coefficients(color, 10)[9:]
    half = 1 << (s - 1)
    y, u, v = split_planes(frame, layout, w)
    u, v = np.repeat(u, 2, axis=-1) - 512, np.repeat(v, 2, axis=-1) - 512          # nearest chroma
    ruv, guv, buv = half + cvr * v, half + cvg * v + cug * u, half + cub * u
    yy = (y - yoff) * cy
    sums = [yy + c for c in (ruv, guv, buv)]
    Q._check_int32(yy, ruv, guv, buv, *sums)
    return np.stack([np.clip(a >> s, 0, 1023) for a in sums], axis=-1).astype(np.uint16)


def encode_samples(rgb10, color='bt601'):
    """RGB10 codes [..., h, w, 3] -> (Y [..., h, w], U, V [..., h, w/2]) samples of the 4:2:2 encode."""
    c = coefficients(color, 10)
    s, yoff = c[14], c[15]
    rgb10 = np.asarray(rgb10)
    if rgb10.shape[-1] != 3:
        raise ValueError(f'expected RGB [..., h, w, 3], got {rgb10.shape}')
    check_size(*rgb10.shape[-3:-1])
    if int(np.max(rgb10, initial=0)) > 1023 or int(np.min(rgb10, initial=0)) < 0:
        raise ValueError('RGB10 code values outside [0, 1023]')
    r, g, b = (rgb10[..., k].astype(np.int64) for k in range(3))
    ys = c[0] * r + c[1] * g + c[2] * b + (1 << (s - 1)) + (yoff << s)
    sr, sg, sb = (a[..., 0::2] + a[..., 1::2] for a in (r, g, b))                  # the pair's sum
    sc = s + 1
    us = c[3] * sr + c[4] * sg + c[5] * sb + (1 << (sc - 1)) + (512 << sc)
    vs = c[6] * sr + c[7] * sg + c[8] * sb + (1 << (sc - 1)) + (512 << sc)
    Q._check_int32(ys, us, vs)
    return np.clip(ys >> s, 0, 1023), np.clip(us >> sc, 0, 1023), np.clip(vs >> sc, 0, 1023)


def rgb_to_yuv(rgb10, layout, color='bt601'):
    """RGB10 codes [..., h, w, 3] -> the whole frame's words [..., *frame_shape]."""
    return join_planes(*encode_samples(rgb10, color), layout)


def rgb_f32_to_yuv(rgb_f32, layout, color='bt601'):
    """The encode of an fp32 RGB frame [..., h, w, 3] (tg_rgb_to_yuv from rgb_f32)."""
    return rgb_to_yuv(quantize10(rgb_f32), layout, color)


def black(layout, color, h, w, lead=()):
    """Frames [*lead, *frame_shape] of the colour's black (tg_fill_black)."""
    yoff = coefficients(color, 10)[15]
    return join_planes(np.full((*lead, h, w), yoff), np.full((*lead, h, w // 2), 512),
                       np.full((*lead, h, w // 2), 512), layout)


def luma8(frame, layout, w=None):
    """The 8-bit luma tg_luma_line_sums sums: Y >> 2, [..., h, w]."""
    return split_planes(frame, layout, w)[0] >> 2


# ------------------------------------------------------------------------------------------------- windows
def window_error(layout, fh, fw, top, left, h, w):
    """None if the h x w picture at (top, left) of an fh x fw frame is a valid window of the layout, else why."""
    _check_layout(layout)
    if top < 0 or left < 0 or top + h > fh or left + w > fw:
        return f'a {h}x{w} picture at ({top}, {left}) does not fit a {fh}x{fw} frame'
    if fw % 2 or left % 2 or w % 2:
        return 'YUV 4:2:2 needs an even frame width, picture width and left'
    if layout == 'v210' and (left % 6 or ((left + w) % 6 and left + w != fw)):
        return 'a v210 picture starts on a 6-pixel group and ends on one or at the frame\'s right edge'
    return None


def decode_window(frames, layout, color, top, left, h, w, frame_w=None):
    """RGB10 codes [..., h, w, 3] of the h x w picture at (top, left) of frames [..., *frame_shape(fh, fw)]."""
    fw = frame_w if layout == 'v210' else np.asarray(frames).shape[-1]
    fh = np.asarray(frames).shape[-2] // (1 if layout == 'v210' else 2)
    err = window_error(layout, fh, fw, top, left, h, w)
    if err:
        raise ValueError(err)
    return yuv_to_rgb(frames, layout, color, fw)[..., top:top + h, left:left + w, :]


def encode_window(frames, rgb10, layout, color, top, left, frame_w=None):
    """frames [..., *frame_shape(fh, fw)] with the encode of the picture rgb10 [..., h, w, 3] written at (top, left)
    (tg_rgb_to_yuv_window): the picture's samples, and in v210 its groups -- the fields past its last pixel of a
    partial last group 0 -- and nothing else.  Returns a new array."""
    out = np.array(frames, copy=True)
    h, w = np.asarray(rgb10).shape[-3:-1]
    fw = frame_w if layout == 'v210' else out.shape[-1]
    fh = out.shape[-2] // (1 if layout == 'v210' else 2)
    err = window_error(layout, fh, fw, top, left, h, w)
    if err:
        raise ValueError(err)
    y, u, v = encode_samples(rgb10, color)
    if layout == 'v210':
        pic = pack_v210(y, u, v)                                           # the picture as a frame of its own
        nbytes = 16 * -(-w // 6)
        out[..., top:top + h, 16 * (left // 6):16 * (left // 6) + nbytes] = pic[..., :nbytes]
        return out
    shift = 6 if layout == 'p210' else 0
    out[..., top:top + h, left:left + w] = y << shift
    if layout == 'p210':
        c = np.stack([u, v], axis=-1).reshape(*u.shape[:-1], w)
        out[..., fh + top:fh + top + h, left:left + w] = c << shift
    else:
        flat = out.reshape(*out.shape[:-2], 2 * fh * fw)                  # out is a new array: a view
        for k, c in ((0, u), (1, v)):                                       # the U plane, then the V plane
            p = fh * fw + k * fh * (fw // 2)
            plane = flat[..., p:p + fh * (fw // 2)].reshape(*out.shape[:-2], fh, fw // 2)
            plane[..., top:top + h, left // 2:(left + w) // 2] = c
    return out


# ------------------------------------------------------------------------------------------------- test patterns
def yuv10_pattern(layout, frames=4, seed=10):
    """`frames` 10-bit 4:2:2 frames [frames, *frame_shape] whose pairs hold every (U, V) of samples10()^2 and whose
    pixels cycle Y through samples10() (shifted by one pixel per frame), as words of the layout; returns (frames, h,
    w, (y, u, v)) with the samples.  w = 80 is no multiple of 6 or 48, and h is odd.
    v210 frames carry junk in bits 30-31 and in the row padding (the decode ignores them); 5 % of the I422_10
    words are above 1023 (the decode clamps them)."""
    s = samples10()
    m = s.size
    uu, vv = np.meshgrid(s, s, indexing='ij')
    uu, vv = uu.reshape(-1), vv.reshape(-1)
    per_row = 40                                                     # pairs per row: w = 80, 13 v210 groups
    rows = -(-uu.size // per_row) | 1                                 # an odd height
    ub = np.full(rows * per_row, 512, np.int64)
    vb = ub.copy()
    ub[:uu.size], vb[:vv.size] = uu, vv
    u, v = ub.reshape(rows, per_row), vb.reshape(rows, per_row)
    h, w = rows, 2 * per_row
    y = s[(np.arange(h * w).reshape(h, w) * 7) % m]
    ys = np.stack([np.roll(y.reshape(-1), k).reshape(h, w) for k in range(frames)])
    us, vs = np.broadcast_to(u, (frames, h, w // 2)), np.broadcast_to(v, (frames, h, w // 2))
    f = join_planes(ys, us, vs, layout)
    rng = np.random.default_rng(seed)
    if layout == 'v210':
        words = f.view('<u4').copy()
        words |= (rng.integers(0, 4, size=words.shape).astype('<u4') << 30)
        f = words.view(np.uint8)
        g = 16 * -(-w // 6)
        f[..., g:] = rng.integers(0, 256, size=f[..., g:].shape, dtype=np.uint8)
    elif layout == 'i422_10':
        f = f.astype(np.int64)
        hi = rng.random(f.shape) < 0.05
        f[hi] = rng.integers(1024, 65536, size=int(hi.sum()))
        f = f.astype(np.uint16)
    else:
        f = f | rng.integers(0, 64, size=f.shape).astype(np.uint16)    # P210: junk in the low 6 bits
    return np.ascontiguousarray(f), h, w, (ys, np.array(us), np.array(vs))
