"""Farneback dense optical flow, restated in float64 numpy.

This is the specification of the flow kernels of tg_metrics.cu (tecogan_b200.metrics.farneback): OpenCV's CPU
cv2.calcOpticalFlowFarneback with flags=0 (box-filtered normal equations, flow starting at zero), which is what the
tOF metric of TecoGAN calls (pyr_scale=0.5, levels=3, winsize=15, iterations=3, poly_n=5, poly_sigma=1.2).

  levels   L = the number of times scale *= pyr_scale can be done (at most `levels`) while w*scale and h*scale both
           stay >= 32.
  level k  (k = L .. 0): scale = pyr_scale**k, sigma = (1/scale - 1)/2, ksize = max(rint(5 sigma) | 1, 3), size
           (rint(w scale), rint(h scale)) with rint rounding half to even.  Each image is Gaussian-blurred at full
           size (ksize, sigma; BORDER_REFLECT_101; at k = 0 sigma = 0 selects cv2's fixed [1/4, 1/2, 1/4]), resized
           with INTER_LINEAR to the level size and expanded by poly_exp.  The flow is 0 on the coarsest level and
           the previous level's flow resized with INTER_LINEAR and divided by pyr_scale on the others.
  poly_exp R (5 channels) from separable sums with g, x g, x^2 g over offsets -n .. n (n = poly_n), rows and
           columns clamped, scaled by entries of the inverse of the 6x6 moment matrix G.
  update   M (5 channels) = update_matrices(R0, R1, flow): R1 sampled bilinearly at x + flow, combined with R0, damped
           near the edges.
  iterate  `iterations` times: S = the winsize x winsize box mean of M (borders replicated), solve the 2x2 system
           for the flow, and (except after the last iteration) recompute M from the new flow.

Only tests and the fixture generator import this module.
"""
import numpy as np

MIN_SIZE = 32
BORDER = np.float32([0.14, 0.14, 0.4472, 0.4472, 0.4472])


def rint(v):
    """cvRound: round half to even"""
    return int(np.rint(v))


def check_args(pyr_scale, levels, winsize, iterations, poly_n, poly_sigma, flags):
    """cv2's argument checks plus the variants this specification leaves out (ValueError)."""
    if not (0 < pyr_scale < 1):
        raise ValueError(f'pyr_scale must lie in (0, 1), got {pyr_scale}')
    if int(levels) != levels or levels < 0:
        raise ValueError(f'levels must be a non-negative integer, got {levels}')
    if int(winsize) != winsize or winsize < 1:
        raise ValueError(f'winsize must be a positive integer, got {winsize}')
    if int(iterations) != iterations or iterations < 1:
        raise ValueError(f'iterations must be a positive integer, got {iterations}')
    if poly_n not in (5, 7):
        raise ValueError(f'poly_n must be 5 or 7, got {poly_n}')
    if not (poly_sigma > 0 and np.isfinite(poly_sigma)):
        raise ValueError(f'poly_sigma must be positive, got {poly_sigma}')
    if flags != 0:
        raise ValueError(f'only flags=0 is supported (no OPTFLOW_USE_INITIAL_FLOW / OPTFLOW_FARNEBACK_GAUSSIAN), '
                         f'got {flags}')


def level_count(h, w, pyr_scale, levels):
    scale, k = 1.0, 0
    while k < levels:
        scale *= pyr_scale
        if w * scale < MIN_SIZE or h * scale < MIN_SIZE:
            break
        k += 1
    return k


def level_params(h, w, pyr_scale, k):
    """-> (sigma, ksize, level h, level w) of level k"""
    scale = 1.0
    for _ in range(k):
        scale *= pyr_scale
    sigma = (1.0 / scale - 1.0) * 0.5
    ksize = max(rint(sigma * 5) | 1, 3)
    return sigma, ksize, rint(h * scale), rint(w * scale)


def gaussian_taps(ksize, sigma):
    """cv2.getGaussianKernel(ksize, sigma, CV_32F) as float64 values of the float32 taps"""
    if sigma <= 0 and ksize == 3:
        return np.float64([0.25, 0.5, 0.25])
    if sigma <= 0:
        sigma = 0.3 * ((ksize - 1) * 0.5 - 1) + 0.8
    x = np.arange(ksize) - (ksize - 1) * 0.5
    t = np.exp(-0.5 / (sigma * sigma) * x * x)
    return (t / t.sum()).astype(np.float32).astype(np.float64)


def reflect101(i, n):
    """BORDER_REFLECT_101 index map (n >= 2)"""
    i = np.abs(i)
    period = 2 * (n - 1)
    i = i % period
    return np.where(i >= n, period - i, i)


def gaussian_blur(img, ksize, sigma):
    taps = gaussian_taps(ksize, sigma)
    r = ksize // 2
    h, w = img.shape
    out = np.zeros_like(img)
    ri = reflect101(np.arange(-r, h + r), h)
    tmp = sum(taps[j] * img[ri[j:j + h]] for j in range(ksize))
    ci = reflect101(np.arange(-r, w + r), w)
    out = sum(taps[j] * tmp[:, ci[j:j + w]] for j in range(ksize))
    return out


def _linear_axis(src, dst):
    """cv2 INTER_LINEAR source index and weight along one axis: fx = float32((d + 0.5) * src/dst - 0.5), clamped"""
    scale = 1.0 / (dst / src)
    f = ((np.arange(dst) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    lo = s < 0
    f[lo], s[lo] = 0, 0
    hi = s >= src - 1
    f[hi], s[hi] = 0, src - 1
    s1 = np.minimum(s + 1, src - 1)
    return s, s1, f.astype(np.float64)


def resize_linear(img, h, w):
    """cv2.resize(img, (w, h), interpolation=INTER_LINEAR) for [H, W] or [H, W, C] arrays"""
    H, W = img.shape[:2]
    y0, y1, fy = _linear_axis(H, h)
    x0, x1, fx = _linear_axis(W, w)
    ex = (slice(None),) + (None,) * (img.ndim - 1)
    rows = img[y0] * (1 - fy)[ex] + img[y1] * fy[ex]
    ex = (None, slice(None)) + (None,) * (img.ndim - 2)
    return rows[:, x0] * (1 - fx)[ex] + rows[:, x1] * fx[ex]


def poly_kernels(n, sigma):
    """-> g, xg, xxg (float32 values over offsets -n..n, as float64) and (ig11, ig03, ig33, ig55)"""
    x = np.arange(-n, n + 1)
    g = np.exp(-(x * x) / (2 * sigma * sigma)).astype(np.float32)
    s = 1.0 / g.astype(np.float64).sum()
    g = (g * s).astype(np.float32)
    xg = (x * g).astype(np.float32)
    xxg = (x * x * g).astype(np.float32)
    # the moment sums: float32 products of the taps, accumulated in float64
    gy, gx = g[:, None], g[None, :]
    X = x[None, :].astype(np.float32)
    Y = x[:, None].astype(np.float32)
    gg = gy * gx
    G = np.zeros((6, 6))
    G[0, 0] = gg.astype(np.float64).sum()
    G[1, 1] = (gg * X * X).astype(np.float64).sum()
    G[3, 3] = (gg * X * X * X * X).astype(np.float64).sum()
    G[5, 5] = (gg * X * X * Y * Y).astype(np.float64).sum()
    G[2, 2] = G[0, 3] = G[0, 4] = G[3, 0] = G[4, 0] = G[1, 1]
    G[4, 4] = G[3, 3]
    G[3, 4] = G[4, 3] = G[5, 5]
    iG = np.linalg.inv(G)
    return (g.astype(np.float64), xg.astype(np.float64), xxg.astype(np.float64),
            (iG[1, 1], iG[0, 3], iG[3, 3], iG[5, 5]))


def poly_exp(img, n, sigma):
    """[h, w] -> R [h, w, 5]"""
    g, xg, xxg, (ig11, ig03, ig33, ig55) = poly_kernels(n, sigma)
    h, w = img.shape
    rows = np.arange(h)
    t0 = g[n] * img
    t1 = np.zeros_like(img)
    t2 = xxg[n] * img
    for k in range(1, n + 1):
        a = img[np.maximum(rows - k, 0)]
        b = img[np.minimum(rows + k, h - 1)]
        t0 = t0 + g[n + k] * (a + b)
        t1 = t1 + xg[n + k] * (b - a)
        t2 = t2 + xxg[n + k] * (a + b)
    cols = np.arange(w)
    b1 = g[n] * t0
    b3 = g[n] * t1
    b5 = g[n] * t2
    b2 = np.zeros_like(img)
    b4 = np.zeros_like(img)
    b6 = np.zeros_like(img)
    for k in range(1, n + 1):
        lo, hi = np.maximum(cols - k, 0), np.minimum(cols + k, w - 1)
        b1 = b1 + g[n + k] * (t0[:, hi] + t0[:, lo])
        b4 = b4 + xxg[n + k] * (t0[:, hi] + t0[:, lo])
        b2 = b2 + xg[n + k] * (t0[:, hi] - t0[:, lo])
        b3 = b3 + g[n + k] * (t1[:, hi] + t1[:, lo])
        b6 = b6 + xg[n + k] * (t1[:, hi] - t1[:, lo])
        b5 = b5 + g[n + k] * (t2[:, hi] + t2[:, lo])
    return np.stack([b3 * ig11, b2 * ig11, b1 * ig03 + b5 * ig33, b1 * ig03 + b4 * ig33, b6 * ig55], axis=-1)


def edge_scale(h, w):
    """[h, w] product of BORDER[distance] over every edge closer than 5 px (1 elsewhere)"""
    def axis(n):
        s = np.ones(n)
        i = np.arange(n)
        near = i < 5
        s[near] *= BORDER[i[near]]
        far = i >= n - 5
        s[far] *= BORDER[(n - 1 - i)[far]]
        return s
    return axis(h)[:, None] * axis(w)[None, :]


def update_matrices(R0, R1, flow):
    """-> M [h, w, 5]"""
    h, w = flow.shape[:2]
    dx, dy = flow[..., 0], flow[..., 1]
    fx = np.arange(w)[None, :] + dx
    fy = np.arange(h)[:, None] + dy
    x1 = np.floor(fx).astype(np.int64)
    y1 = np.floor(fy).astype(np.int64)
    ax, ay = fx - x1, fy - y1
    inside = (x1 >= 0) & (x1 < w - 1) & (y1 >= 0) & (y1 < h - 1)
    xc, yc = np.clip(x1, 0, max(w - 2, 0)), np.clip(y1, 0, max(h - 2, 0))
    xc1, yc1 = np.minimum(xc + 1, w - 1), np.minimum(yc + 1, h - 1)
    a00, a01 = ((1 - ax) * (1 - ay))[..., None], (ax * (1 - ay))[..., None]
    a10, a11 = ((1 - ax) * ay)[..., None], (ax * ay)[..., None]
    r = a00 * R1[yc, xc] + a01 * R1[yc, xc1] + a10 * R1[yc1, xc] + a11 * R1[yc1, xc1]
    ins = inside[..., None]
    r = np.where(ins, r, 0.0)
    r4 = np.where(inside, (R0[..., 2] + r[..., 2]) * 0.5, R0[..., 2])
    r5 = np.where(inside, (R0[..., 3] + r[..., 3]) * 0.5, R0[..., 3])
    r6 = np.where(inside, (R0[..., 4] + r[..., 4]) * 0.25, R0[..., 4] * 0.5)
    r2 = (R0[..., 0] - r[..., 0]) * 0.5 + r4 * dy + r6 * dx
    r3 = (R0[..., 1] - r[..., 1]) * 0.5 + r6 * dy + r5 * dx
    s = edge_scale(h, w)
    r2, r3, r4, r5, r6 = r2 * s, r3 * s, r4 * s, r5 * s, r6 * s
    return np.stack([r4 * r4 + r6 * r6, (r4 + r5) * r6, r5 * r5 + r6 * r6, r4 * r2 + r6 * r3, r6 * r2 + r5 * r3],
                    axis=-1)


def box_mean(M, winsize):
    """winsize x winsize mean of M [h, w, c], borders replicated (window rows y - m .. y + m, m = winsize // 2;
    an even winsize has the window of winsize + 1 rows scaled by 1 / winsize**2, as cv2 does)"""
    h, w = M.shape[:2]
    m = winsize // 2
    ri = np.clip(np.arange(-m, h + m), 0, h - 1)
    c = np.concatenate([np.zeros((1,) + M.shape[1:]), np.cumsum(M[ri], axis=0)])
    V = c[2 * m + 1:] - c[:h]
    ci = np.clip(np.arange(-m, w + m), 0, w - 1)
    c = np.concatenate([np.zeros((h, 1) + M.shape[2:]), np.cumsum(V[:, ci], axis=1)], axis=1)
    return (c[:, 2 * m + 1:] - c[:, :w]) / float(winsize * winsize)


def solve(S):
    g11, g12, g22, h1, h2 = (S[..., i] for i in range(5))
    idet = 1.0 / (g11 * g22 - g12 * g12 + 1e-3)
    return np.stack([(g11 * h2 - g12 * h1) * idet, (g22 * h1 - g12 * h2) * idet], axis=-1)


def farneback(prev, nxt, pyr_scale=0.5, levels=3, winsize=15, iterations=3, poly_n=5, poly_sigma=1.2, flags=0):
    """cv2.calcOpticalFlowFarneback(prev, next, None, ...) for single-channel images [h, w] -> float64 [h, w, 2]"""
    check_args(pyr_scale, levels, winsize, iterations, poly_n, poly_sigma, flags)
    prev = np.asarray(prev, np.float64)
    nxt = np.asarray(nxt, np.float64)
    if prev.ndim != 2 or prev.shape != nxt.shape:
        raise ValueError(f'prev / next must be single-channel images of one size, got {prev.shape} {nxt.shape}')
    H, W = prev.shape
    L = level_count(H, W, pyr_scale, levels)
    flow = None
    for k in range(L, -1, -1):
        sigma, ksize, h, w = level_params(H, W, pyr_scale, k)
        if flow is None:
            flow = np.zeros((h, w, 2))
        else:
            flow = resize_linear(flow, h, w) * (1.0 / pyr_scale)
        R = [poly_exp(resize_linear(gaussian_blur(img, ksize, sigma), h, w), poly_n, poly_sigma)
             for img in (prev, nxt)]
        M = update_matrices(R[0], R[1], flow)
        for i in range(iterations):
            flow = solve(box_mean(M, winsize))
            if i < iterations - 1:
                M = update_matrices(R[0], R[1], flow)
    return flow
