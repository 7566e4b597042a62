"""Specification of picture windows in stored frames (tg_frame_window): crop on the input side, black padding on the
output side, and the letterbox detection rule of tecogan_b200.detect_bars.  Integer / float64 NumPy only.

A window is the h x w picture at (top, left) of a frame of Hf x Wf pixels stored in a layout: 'rgb' (uint8 HWC
[Hf,Wf,c]) or one of the YUV layouts of oracle/yuv_422_444.py (the frame's words, [*frame_shape(layout, Hf, Wf)]).
 - The windowed decode of a frame is the decode of crop_words(frame, ...): the picture's own words, as a frame of
   h x w in the same layout.  On the layout's chroma grid (4:2:0: even top, left, h, w; 4:2:2: even left and w) the
   picture's chroma samples are exactly those of its pixels, so with nearest chroma this also equals the full
   frame's decode cropped (checked by tests/test_stream_window_cpu.py).
 - A padded output frame is place_words(picture, ...): the format's black everywhere (black_words) and the
   picture's words at the window.
 - detect_bars: a row (column) is picture when its mean 8-bit luma exceeds `limit` in any frame; the box spans the
   first to the last picture row and column, rounded inward to the chroma grid; no picture row or column gives the
   whole frame.
"""
import numpy as np

from . import yuv_422_444 as Y

LAYOUTS = ('rgb',) + Y.ALL_LAYOUTS


def grid(layout):
    """(row step, column step) of the layout's chroma grid."""
    if layout in Y.LAYOUTS_422:
        return 1, 2
    return (2, 2) if layout in Y.LAYOUTS_420 else (1, 1)


def _planes(frame, layout, h, w):
    """Views of the planes of one stored h x w frame, each with (row step, column step, words per column step):
    plane pixel (r, q) holds frame rows r*rs.. and columns q*cs.. ."""
    if layout == 'rgb':
        return [(frame, 1, 1, 1)]
    if layout in Y.LAYOUTS_422:
        return [(frame, 1, 2, 4)]                 # one 4-byte group per pixel pair
    if layout in Y.LAYOUTS_444:
        return [(frame[k * h:(k + 1) * h], 1, 1, 1) for k in range(3)]
    yp = frame[:h]
    if layout in ('nv12', 'p010'):
        return [(yp, 1, 1, 1), (frame[h:], 2, 2, 2)]   # interleaved U V: 2 words per 2 columns
    flat = frame[h:].reshape(-1)
    q = (h // 2) * (w // 2)
    return [(yp, 1, 1, 1), (flat[:q].reshape(h // 2, w // 2), 2, 2, 1),
            (flat[q:].reshape(h // 2, w // 2), 2, 2, 1)]


def frame_shape(layout, h, w, c=3):
    return (h, w, c) if layout == 'rgb' else Y.frame_shape(layout, h, w)


def _check_window(layout, Hf, Wf, top, left, h, w):
    if not (0 <= top and 0 <= left and 0 < h and 0 < w and top + h <= Hf and left + w <= Wf):
        raise ValueError(f'a {h}x{w} picture at ({top}, {left}) does not fit a {Hf}x{Wf} frame')
    gy, gx = grid(layout)
    if Hf % gy or Wf % gx or top % gy or h % gy or left % gx or w % gx:
        raise ValueError(f'window off the {layout} chroma grid')


def _slices(rs, cs, wpc, top, left, h, w):
    return slice(top // rs, (top + h) // rs), slice(left // cs * wpc, (left + w) // cs * wpc)


def crop_words(frame, layout, top, left, h, w):
    """The h x w picture at (top, left) of one stored frame, as a stored h x w frame of the same layout."""
    frame = np.ascontiguousarray(frame)
    c = frame.shape[-1] if layout == 'rgb' else 3
    Hf, Wf = (frame.shape[0], frame.shape[1]) if layout == 'rgb' else _frame_size(layout, frame.shape)
    _check_window(layout, Hf, Wf, top, left, h, w)
    out = np.empty(frame_shape(layout, h, w, c), frame.dtype)
    for (src, rs, cs, wpc), (dst, *_) in zip(_planes(frame, layout, Hf, Wf), _planes(out, layout, h, w)):
        r, q = _slices(rs, cs, wpc, top, left, h, w)
        dst[...] = src[r, q]
    return out


def _frame_size(layout, shape):
    a, b = shape[-2:]
    if layout in Y.LAYOUTS_422:
        return a, b // 2
    return (a // 3, b) if layout in Y.LAYOUTS_444 else (2 * a // 3, b)


def black_words(layout, color='bt601'):
    """(Y word, chroma word) of the format's black as stored; RGB: (0, 0).  Y is the colour's black level (16 << (d -
    8) at limited range, 0 at full), chroma the zero point 128 << (d - 8); P010 stores samples << 6."""
    if layout == 'rgb':
        return 0, 0
    d = Y.depth_of(layout)
    yb = 0 if color.endswith('-full') else 16 << (d - 8)
    cb = 128 << (d - 8)
    sh = 6 if layout == 'p010' else 0
    return yb << sh, cb << sh


def black_frame(layout, color, Hf, Wf, c=3):
    """One stored Hf x Wf frame of the format's black."""
    if layout == 'rgb':
        return np.zeros((Hf, Wf, c), np.uint8)
    yb, cb = black_words(layout, color)
    out = np.empty(Y.frame_shape(layout, Hf, Wf), Y.word_dtype(layout))
    if layout in Y.LAYOUTS_422:
        y0, u0 = Y._PACKED[layout]
        g = out.reshape(Hf, Wf // 2, 4)
        g[..., y0] = g[..., y0 + 2] = yb
        g[..., u0] = g[..., u0 + 2] = cb
        return out
    for k, (p, *_) in enumerate(_planes(out, layout, Hf, Wf)):
        p[...] = yb if k == 0 else cb
    return out


def place_words(picture, layout, color, Hf, Wf, top, left):
    """A stored Hf x Wf frame: the format's black with the stored h x w `picture` at (top, left)."""
    picture = np.ascontiguousarray(picture)
    if layout == 'rgb':
        h, w, c = picture.shape
    else:
        (h, w), c = _frame_size(layout, picture.shape), 3
    _check_window(layout, Hf, Wf, top, left, h, w)
    out = black_frame(layout, color, Hf, Wf, c)
    for (dst, rs, cs, wpc), (src, *_) in zip(_planes(out, layout, Hf, Wf), _planes(picture, layout, h, w)):
        r, q = _slices(rs, cs, wpc, top, left, h, w)
        dst[r, q] = src
    return out


def luma8(frames, layout, channel_order='rgb'):
    """8-bit luma [..., h, w] of stored frames: Y (10-bit samples >> 2) or, for uint8 HWC RGB, cv2's gray
    (9798 R + 19235 G + 3735 B + 16384) >> 15 (tg_metrics_frames_in's)."""
    if layout == 'rgb':
        v = np.asarray(frames).astype(np.int64)
        if channel_order == 'bgr':
            v = v[..., ::-1]
        return ((9798 * v[..., 0] + 19235 * v[..., 1] + 3735 * v[..., 2] + 16384) >> 15).astype(np.int64)
    y, _, _ = Y.split_planes(frames, layout)
    return y >> 2 if Y.depth_of(layout) == 10 else y


def line_sums(frames, layout, channel_order='rgb'):
    """(rows [..., h], cols [..., w]): the exact integer sums of luma8 along each row and column."""
    l8 = luma8(frames, layout, channel_order)
    return l8.sum(-1), l8.sum(-2)


def detect_bars(frames, layout, channel_order='rgb', limit=24):
    """(top, left, h, w) of the picture in frames [k, *stored frame] by the rule above."""
    rows, cols = line_sums(frames, layout, channel_order)
    h, w = rows.shape[-1], cols.shape[-1]
    pic_r = (rows.astype(np.float64) > float(limit) * w).any(0)
    pic_c = (cols.astype(np.float64) > float(limit) * h).any(0)
    if not pic_r.any() or not pic_c.any():
        return 0, 0, h, w
    gy, gx = grid(layout)
    r, q = np.flatnonzero(pic_r), np.flatnonzero(pic_c)
    top, bottom = -(-int(r[0]) // gy) * gy, (int(r[-1]) + 1) // gy * gy
    left, right = -(-int(q[0]) // gx) * gx, (int(q[-1]) + 1) // gx * gx
    if bottom <= top or right <= left:
        return 0, 0, h, w
    return top, left, bottom - top, right - left
