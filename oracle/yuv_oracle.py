"""YUV 4:2:0 <-> RGB as cv2.cvtColor does it, restated in integer numpy.

This is the specification of the stream's NV12 / I420 frame I/O (tg_stream_frame_in_yuv420,
tg_rgb_u8_to_yuv420).  It is pinned to cv2 by tests/test_yuv_oracle_cpu.py: exhaustively against a live cv2
when it imports, and always against tests/golden/yuv420_cv2.npz (oracle/gen_yuv_golden.py).

    yuv420_to_rgb(frame, layout)   frame uint8 [..., 3h/2, w] -> RGB uint8 [..., h, w, 3]
                                   == cv2.cvtColor(frame, COLOR_YUV2RGB_NV12 / COLOR_YUV2RGB_I420)
    rgb_to_yuv420(rgb, layout)     RGB uint8 [..., h, w, 3] -> uint8 [..., 3h/2, w]
                                   == cv2.cvtColor(rgb, COLOR_RGB2YUV_I420); 'nv12' interleaves its U and V

BT.601 limited range, 20-bit fixed point.  Decode: nearest chroma (the four pixels of a 2x2 block share its U/V
sample).  Encode: the chroma of a 2x2 block comes from its top-left pixel only.  h and w must be even.
Layouts, per frame: the Y plane h x w, then either the interleaved UV plane (h/2) x w (NV12: U V U V ...) or the
U plane and the V plane of (h/2) x (w/2) each, stored back to back (I420; as cv2 and ffmpeg's yuv420p lay them out,
each plane is (h/4) x w bytes when viewed at width w).
"""
import numpy as np

LAYOUTS = ('nv12', 'i420')
SHIFT = 20
HALF = 1 << (SHIFT - 1)
# RGB -> YUV
CRY, CGY, CBY = 269484, 528482, 102760
CRU, CGU, CBU = -155188, -305135, 460324
CRV, CGV, CBV = 460324, -385875, -74448
# YUV -> RGB
CY, CUB, CUG, CVG, CVR = 1220542, 2116026, -409993, -852492, 1673527


def _check(h, w, layout):
    if layout not in LAYOUTS:
        raise ValueError(f'layout must be one of {LAYOUTS}, got {layout!r}')
    if h % 2 or w % 2 or h <= 0 or w <= 0:
        raise ValueError(f'YUV 4:2:0 needs an even, positive height and width, got {h}x{w}')


def split_planes(frame, layout):
    """uint8 [..., 3h/2, w] -> (Y [..., h, w], U [..., h/2, w/2], V [..., h/2, w/2])."""
    frame = np.asarray(frame)
    h3, w = frame.shape[-2:]
    if h3 % 3:
        raise ValueError(f'a YUV 4:2:0 frame has 3h/2 rows, got {h3}')
    h = h3 // 3 * 2
    _check(h, w, layout)
    lead = frame.shape[:-2]
    y = frame[..., :h, :]
    c = frame[..., h:, :].reshape(*lead, -1)
    if layout == 'nv12':
        uv = c.reshape(*lead, h // 2, w // 2, 2)
        return y, uv[..., 0], uv[..., 1]
    q = (h // 2) * (w // 2)
    return y, c[..., :q].reshape(*lead, h // 2, w // 2), c[..., q:].reshape(*lead, h // 2, w // 2)


def join_planes(y, u, v, layout):
    """Inverse of split_planes."""
    h, w = y.shape[-2:]
    _check(h, w, layout)
    lead = y.shape[:-2]
    if layout == 'nv12':
        c = np.stack([u, v], axis=-1).reshape(*lead, h // 2, w)
    else:
        c = np.concatenate([u.reshape(*lead, -1), v.reshape(*lead, -1)], axis=-1).reshape(*lead, h // 2, w)
    return np.ascontiguousarray(np.concatenate([y, c], axis=-2), dtype=np.uint8)


def yuv420_to_rgb(frame, layout):
    y, u, v = split_planes(frame, layout)
    uu = u.astype(np.int64) - 128
    vv = v.astype(np.int64) - 128
    ruv = HALF + CVR * vv
    guv = HALF + CVG * vv + CUG * uu
    buv = HALF + CUB * uu
    up = lambda a: np.repeat(np.repeat(a, 2, axis=-2), 2, axis=-1)          # nearest chroma
    yy = np.maximum(y.astype(np.int64) - 16, 0) * CY
    rgb = [np.clip((yy + up(c)) >> SHIFT, 0, 255) for c in (ruv, guv, buv)]
    return np.stack(rgb, axis=-1).astype(np.uint8)


def rgb_to_yuv420(rgb, layout):
    rgb = np.asarray(rgb)
    if rgb.shape[-1] != 3:
        raise ValueError(f'expected RGB [..., h, w, 3], got {rgb.shape}')
    h, w = rgb.shape[-3:-1]
    _check(h, w, layout)
    r, g, b = (rgb[..., k].astype(np.int64) for k in range(3))
    y = np.clip((CRY * r + CGY * g + CBY * b + HALF + (16 << SHIFT)) >> SHIFT, 0, 255)
    r, g, b = (a[..., ::2, ::2] for a in (r, g, b))                          # top-left pixel of each 2x2 block
    u = np.clip((CRU * r + CGU * g + CBU * b + HALF + (128 << SHIFT)) >> SHIFT, 0, 255)
    v = np.clip((CRV * r + CGV * g + CBV * b + HALF + (128 << SHIFT)) >> SHIFT, 0, 255)
    return join_planes(y.astype(np.uint8), u.astype(np.uint8), v.astype(np.uint8), layout)


# ------------------------------------------------------------------------------------- exhaustive test patterns
def rgb_triples_pattern(first_row, rows, cols=4096):
    """RGB uint8 [2*rows, 2*cols, 3] whose 2x2 block (r, c) has the top-left pixel i = (first_row + r) * cols + c
    read as the 24-bit triple (i >> 16, i >> 8, i) & 255; the other three pixels hold 255 - that triple, i >> 1 and
    i ^ 0x5a5a5a, so a chroma that read them would differ.  Rows 0..4095 of 4096 columns cover all 2^24 triples."""
    i = (first_row + np.arange(rows, dtype=np.int64))[:, None] * cols + np.arange(cols, dtype=np.int64)
    trip = lambda v: np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], axis=-1).astype(np.uint8)
    out = np.empty((rows, 2, cols, 2, 3), np.uint8)
    out[:, 0, :, 0] = trip(i)
    out[:, 0, :, 1] = 255 - trip(i)
    out[:, 1, :, 0] = trip(i >> 1)
    out[:, 1, :, 1] = trip(i ^ 0x5a5a5a)
    return out.reshape(2 * rows, 2 * cols, 3)


def yuv_triples_pattern(layout):
    """A 4096x4096 YUV 4:2:0 frame ([6144, 4096] uint8) that holds every (Y, U, V) triple exactly once: chroma block
    (by, bx) carries the pair (U, V) = divmod((by % 32) * 2048 + bx, 256), and its four pixels (dy, dx) have
    Y = 4 * (by // 32) + 2 * dy + dx."""
    by = np.arange(2048, dtype=np.int64)[:, None]
    bx = np.arange(2048, dtype=np.int64)[None, :]
    pair = (by % 32) * 2048 + bx
    u, v = (pair >> 8).astype(np.uint8), (pair & 255).astype(np.uint8)
    y = np.empty((2048, 2, 2048, 2), np.uint8)
    for dy in range(2):
        for dx in range(2):
            y[:, dy, :, dx] = np.broadcast_to(4 * (by // 32) + 2 * dy + dx, (2048, 2048))
    return join_planes(y.reshape(4096, 4096), u, v, layout)
