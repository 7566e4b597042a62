"""Video quality metrics on the device: PSNR and tOF as TecoGAN's MetricCalculator computes them
(codes/metrics/metric_calculator.py: compute_PSNR, compute_tOF), on the kernels of csrc/tg_metrics.cu.

- PSNR: the per-frame sum of squared differences is an exact integer from the device; the host finishes it with the
  reference's float64 expression, so the values are identical to the reference's, bit for bit.
- tOF: the mean end-point error between the Farneback flows (cv2.calcOpticalFlowFarneback, flags=0) of consecutive
  ground-truth frames and of consecutive predicted frames, computed in fp32 on the device.

LPIPS is not here: it already runs on the GPU in PyTorch (the reference's DistModel).
"""
import math

import numpy as np
import torch

from . import lib as L
from . import ops

DEFAULT_MAX_WORKSPACE_BYTES = 2 << 30


def _check_farneback_args(pyr_scale, levels, winsize, iterations, poly_n, poly_sigma, flags):
    def whole(v):
        return isinstance(v, (int, np.integer)) and not isinstance(v, bool)
    if not (isinstance(pyr_scale, (int, float, np.floating)) and 0 < pyr_scale < 1):
        raise ValueError(f'pyr_scale must lie in (0, 1), got {pyr_scale!r}')
    if not whole(levels) or levels < 0:
        raise ValueError(f'levels must be a non-negative integer, got {levels!r}')
    if not whole(winsize) or not 1 <= winsize <= 63:
        raise ValueError(f'winsize must be an integer in [1, 63], got {winsize!r}')
    if not whole(iterations) or iterations < 1:
        raise ValueError(f'iterations must be a positive integer, got {iterations!r}')
    if not whole(poly_n) or poly_n not in (5, 7):
        raise ValueError(f'poly_n must be 5 or 7, got {poly_n!r}')
    if not (isinstance(poly_sigma, (int, float, np.floating)) and math.isfinite(poly_sigma) and poly_sigma > 0):
        raise ValueError(f'poly_sigma must be a positive number, got {poly_sigma!r}')
    if not whole(flags) or flags != 0:
        raise ValueError(f'only flags=0 is implemented (OPTFLOW_USE_INITIAL_FLOW and OPTFLOW_FARNEBACK_GAUSSIAN are '
                         f'not), got {flags!r}')
    return ops.farneback_params(pyr_scale, levels, winsize, iterations, poly_n, poly_sigma, flags)


def farneback(prev, next, pyr_scale=0.5, levels=3, winsize=15, iterations=3, poly_n=5, poly_sigma=1.2, flags=0):
    """cv2.calcOpticalFlowFarneback(prev[i], next[i], None, pyr_scale, levels, winsize, iterations, poly_n,
    poly_sigma, flags) for every i, in one batch on the device.

    prev, next: uint8 CUDA tensors [N, H, W] (or [H, W]).  Returns float32 [N, H, W, 2] (or [H, W, 2]) on the same
    device: the (dx, dy) flow from prev to next."""
    params = _check_farneback_args(pyr_scale, levels, winsize, iterations, poly_n, poly_sigma, flags)
    for x, nm in ((prev, 'prev'), (next, 'next')):
        if not isinstance(x, torch.Tensor) or not x.is_cuda or x.dtype != torch.uint8:
            raise ValueError(f'{nm} must be a uint8 CUDA tensor')
    if prev.shape != next.shape or prev.dim() not in (2, 3):
        raise ValueError(f'prev / next must be [N, H, W] (or [H, W]) of one shape, got {tuple(prev.shape)} and '
                         f'{tuple(next.shape)}')
    if prev.device != next.device:
        raise ValueError('prev / next on different devices')
    single = prev.dim() == 2
    p, q = (prev[None], next[None]) if single else (prev, next)
    n, h, w = p.shape
    if n == 0:
        return torch.empty(0, h, w, 2, dtype=torch.float32, device=prev.device)
    gray = torch.stack([p, q], 1).reshape(2 * n, h, w)
    with torch.cuda.device(prev.device):
        flow = ops.farneback(gray, n, params)
    return flow[0] if single else flow


def rgb_to_gray(u8):
    """cv2.cvtColor(x, cv2.COLOR_RGB2GRAY) of uint8 RGB frames on the device, bit for bit: [..., H, W, 3] CUDA uint8
    -> [..., H, W] uint8."""
    if not isinstance(u8, torch.Tensor) or not u8.is_cuda or u8.dtype != torch.uint8:
        raise ValueError('rgb_to_gray expects a uint8 CUDA tensor')
    if u8.dim() < 3 or u8.shape[-1] != 3:
        raise ValueError(f'rgb_to_gray expects [..., H, W, 3], got {tuple(u8.shape)}')
    lead, (h, w) = u8.shape[:-3], u8.shape[-3:-1]
    x = u8.reshape(-1, h, w, 3).contiguous()
    gray = torch.empty(x.shape[0], h, w, dtype=torch.uint8, device=u8.device)
    if x.shape[0]:
        with torch.cuda.device(u8.device):
            ops.metrics_frames_in(x, None, L.PSNR_NONE, gray)
    return gray.reshape(*lead, h, w)


def _frames(x, nm):
    if isinstance(x, np.ndarray):
        ok = x.dtype == np.uint8
    elif isinstance(x, torch.Tensor):
        ok = x.dtype == torch.uint8 and x.is_cuda
    else:
        ok = False
    if not ok:
        raise ValueError(f'{nm} must be a uint8 numpy array or a uint8 CUDA tensor')
    if x.ndim != 4 or x.shape[3] != 3:
        raise ValueError(f'{nm} must be RGB frames [T, H, W, 3], got {tuple(x.shape)}')
    return x


def _chunk(x, s, e, device):
    if isinstance(x, np.ndarray):
        return torch.from_numpy(np.ascontiguousarray(x[s:e])).to(device, non_blocking=False)
    return x[s:e].contiguous()


def psnr_from_sse(sse, count):
    """compute_PSNR's float64 expression from the exact per-frame integer SSE: 20 log10(255 / sqrt(sse / count)),
    inf where the frames are equal."""
    out = np.empty(len(sse))
    for i, s in enumerate(sse):
        rmse = np.sqrt(np.float64(int(s)) / count)
        out[i] = np.inf if rmse == 0 else 20 * np.log10(255.0 / rmse)
    return out


def sequence_metrics(true_seq, pred_seq, psnr='y', tof=True, max_workspace_bytes=DEFAULT_MAX_WORKSPACE_BYTES):
    """PSNR and tOF of a predicted sequence against its ground truth, as MetricCalculator.compute_sequence_metrics
    computes them frame by frame.

    true_seq, pred_seq: uint8 RGB frames [T, H, W, 3], host numpy arrays or CUDA tensors (the device is theirs, or
    the current CUDA device for numpy input).  Frames of different sizes are cropped to the smaller height and width
    (their top-left corner), as the reference does.
    psnr: 'y' (the Y of data_utils.rgb_to_ycbcr), 'rgb', or None.  tof: whether to compute tOF (always on gray
    frames, as compute_tOF does).
    max_workspace_bytes: bound on the device memory of the tOF pass; a longer sequence is scored in chunks of
    consecutive frames that overlap by one frame.

    Returns {'PSNR': float64 [T]} and / or {'tOF': float64 [T - 1]} (numpy), in that order."""
    true_seq, pred_seq = _frames(true_seq, 'true_seq'), _frames(pred_seq, 'pred_seq')
    if psnr not in ('y', 'rgb', None):
        raise ValueError(f"psnr must be 'y', 'rgb' or None, got {psnr!r}")
    if not isinstance(tof, bool):
        raise ValueError(f'tof must be a bool, got {tof!r}')
    T = true_seq.shape[0]
    if pred_seq.shape[0] != T:
        raise ValueError(f'true_seq has {T} frames, pred_seq {pred_seq.shape[0]}')
    h, w = min(true_seq.shape[1], pred_seq.shape[1]), min(true_seq.shape[2], pred_seq.shape[2])
    out = {}
    if T == 0 or (psnr is None and not tof):
        if psnr is not None:
            out['PSNR'] = np.zeros(0)
        if tof:
            out['tOF'] = np.zeros(0)
        return out
    device = next((x.device for x in (true_seq, pred_seq) if isinstance(x, torch.Tensor)),
                  torch.device('cuda', torch.cuda.current_device()))
    mode = {'y': L.PSNR_Y, 'rgb': L.PSNR_RGB, None: L.PSNR_NONE}[psnr]
    hw = h * w
    if tof and T >= 2:
        def chunk_bytes(n):
            return (ops.farneback_workspace_bytes(2, n, h, w) + 2 * n * hw + 2 * (n - 1) * hw * 8
                    + 2 * n * hw * 3 * 2)
        n = T
        while n > 2 and chunk_bytes(n) > max_workspace_bytes:
            n -= 1
        if chunk_bytes(n) > max_workspace_bytes:
            raise ValueError(f'max_workspace_bytes={max_workspace_bytes} is below the {chunk_bytes(2)} bytes that '
                             f'one pair of {h}x{w} frames needs')
    else:
        n = T
    sse_parts, epe_parts = [], []
    with torch.cuda.device(device):
        s = 0
        while True:
            e = min(s + n, T)
            tc, pc = _chunk(true_seq, s, e, device), _chunk(pred_seq, s, e, device)
            m = e - s
            gray = torch.empty(2, m, h, w, dtype=torch.uint8, device=device) if tof else None
            sse = ops.metrics_frames_in(tc, pc, mode, gray)
            if sse is not None:
                sse_parts.append(sse if s == 0 else sse[1:])
            if tof and m >= 2:
                flow = ops.farneback(gray.view(2 * m, h, w), 2, _check_farneback_args(0.5, 3, 15, 3, 5, 1.2, 0))
                epe_parts.append(ops.flow_epe_sum(flow[:m - 1], flow[m - 1:]))
            if e == T:
                break
            s = e - 1 if tof else e
    if psnr is not None:
        sse = torch.cat(sse_parts).cpu().numpy().view(np.uint64)
        out['PSNR'] = psnr_from_sse(sse, hw * (3 if psnr == 'rgb' else 1))
    if tof:
        out['tOF'] = (torch.cat(epe_parts).cpu().numpy() / hw) if epe_parts else np.zeros(0)
    return out


# ---- the official metric script (codes/official_metrics/metrics.py) -------------------------------------------------

OFFICIAL_KEYS = ('PSNR', 'SSIM', 'tOF')
OFFICIAL_MIN_SIDE = 48                     # the smallest side whose crop_8x8 is not empty


def crop_8x8(n):
    """(offset, size) of the official script's crop_8x8 along a side of n >= 48 pixels: the largest multiple of 32
    that is <= n - 16, centred at (n - size) // 2"""
    size = (n // 32) * 32
    while size > n - 16:
        size -= 32
    return (n - size) // 2, size


def official_sequence_metrics(true_seq, pred_seq, cutfr=2, keys=OFFICIAL_KEYS,
                              max_workspace_bytes=DEFAULT_MAX_WORKSPACE_BYTES):
    """PSNR, SSIM and tOF of a predicted sequence as TecoGAN's official metric script (the one behind the paper's
    tables) computes them frame by frame, on the device.

    true_seq, pred_seq: uint8 RGB frames [T, H, W, 3], host numpy arrays or CUDA tensors, as sequence_metrics takes
    them.  Both are cropped to their common top-left size (h, w), which must be at least 48 x 48; crop_8x8 of it is
    the scored window.  Frames cutfr .. T - cutfr - 1 are scored:
      PSNR  20 log10(255 / RMSE) of the unrounded float64 Y of _rgb2ycbcr over the window (inf on equal frames)
      SSIM  skimage compare_ssim of those Y (7x7 uniform window), data_range = max - min of the predicted Y
      tOF   from frame cutfr + 1 on: the mean end-point error over the window of the Farneback flows of the full
            common-size gray frames (flow of frame i - 1 -> i, ground truth against prediction)
    keys: the metrics to compute, a subset of OFFICIAL_KEYS.  max_workspace_bytes bounds the device memory of the
    pass; a longer sequence is scored in chunks of consecutive frames that overlap by one frame.

    Returns {key: float64 numpy array} in the order of OFFICIAL_KEYS: PSNR and SSIM of T - 2 cutfr frames, tOF of
    T - 2 cutfr - 1 (empty arrays when there are too few frames)."""
    true_seq, pred_seq = _frames(true_seq, 'true_seq'), _frames(pred_seq, 'pred_seq')
    if isinstance(keys, str) or not all(isinstance(k, str) and k in OFFICIAL_KEYS for k in keys):
        raise ValueError(f'keys must be a subset of {OFFICIAL_KEYS}, got {keys!r}')
    if not isinstance(cutfr, (int, np.integer)) or isinstance(cutfr, bool) or cutfr < 0:
        raise ValueError(f'cutfr must be a non-negative integer, got {cutfr!r}')
    T = true_seq.shape[0]
    if pred_seq.shape[0] != T:
        raise ValueError(f'true_seq has {T} frames, pred_seq {pred_seq.shape[0]}')
    h, w = min(true_seq.shape[1], pred_seq.shape[1]), min(true_seq.shape[2], pred_seq.shape[2])
    if h < OFFICIAL_MIN_SIDE or w < OFFICIAL_MIN_SIDE:
        raise ValueError(f'the common frame size {h}x{w} is below {OFFICIAL_MIN_SIDE}x{OFFICIAL_MIN_SIDE}: its '
                         f'crop_8x8 is empty')
    keys = [k for k in OFFICIAL_KEYS if k in keys]
    tof = 'tOF' in keys
    stats_wanted = 'PSNR' in keys or 'SSIM' in keys
    (y0, hc), (x0, wc) = crop_8x8(h), crop_8x8(w)
    window = (y0, x0, hc, wc)
    n_s = max(T - 2 * cutfr, 0)
    if n_s == 0 or not keys:
        return {k: np.zeros(0) for k in keys}
    true_seq, pred_seq = true_seq[cutfr:T - cutfr], pred_seq[cutfr:T - cutfr]
    device = next((x.device for x in (true_seq, pred_seq) if isinstance(x, torch.Tensor)),
                  torch.device('cuda', torch.cuda.current_device()))
    hw = h * w
    frame_bytes = 3 * (true_seq.shape[1] * true_seq.shape[2] + pred_seq.shape[1] * pred_seq.shape[2])

    def chunk_bytes(n):
        b = n * frame_bytes                                            # the uint8 frames of the chunk, full size
        if stats_wanted:
            b += n * 3 * 8 + ops.official_frames_stats_workspace_bytes(n, hc, wc)
        if 'SSIM' in keys:
            b += n * 8 + ops.ssim_y_workspace_bytes(n, hc, wc)
        if tof and n >= 2:
            b += ops.farneback_workspace_bytes(2, n, h, w) + 2 * n * hw + 2 * (n - 1) * hw * 8
            b += (n - 1) * 8 + int(L.load().tg_flow_epe_sum_window_workspace_bytes(n - 1, hc))
        return b
    n, n_min = n_s, min(n_s, 2 if tof else 1)     # chunks overlap by one frame with tOF, so they need two
    while n > n_min and chunk_bytes(n) > max_workspace_bytes:
        n -= 1
    if chunk_bytes(n) > max_workspace_bytes:
        raise ValueError(f'max_workspace_bytes={max_workspace_bytes} is below the {chunk_bytes(n)} bytes that '
                         f'{n} frames of {h}x{w} need')
    params = _check_farneback_args(0.5, 3, 15, 3, 5, 1.2, 0) if tof else None
    stats_parts, ssim_parts, epe_parts = [], [], []
    with torch.cuda.device(device):
        s = 0
        while True:
            e = min(s + n, n_s)
            tc, pc = _chunk(true_seq, s, e, device), _chunk(pred_seq, s, e, device)
            m = e - s
            # with tOF a chunk's first frame is the last one's last frame, whose PSNR / SSIM are already kept
            new = slice(1 if s > 0 and tof else 0, None)
            if stats_wanted:
                stats = ops.official_frames_stats(tc, pc, window)
                stats_parts.append(stats[new])
                if 'SSIM' in keys:
                    ssim_parts.append(ops.ssim_y(tc, pc, window, stats)[new])
            if tof and m >= 2:
                gray = torch.empty(2, m, h, w, dtype=torch.uint8, device=device)
                ops.metrics_frames_in(tc, pc, L.PSNR_NONE, gray)
                flow = ops.farneback(gray.view(2 * m, h, w), 2, params)
                epe_parts.append(ops.flow_epe_sum(flow[:m - 1], flow[m - 1:], window))
            if e == n_s:
                break
            s = e - 1 if tof else e
    out = {}
    if 'PSNR' in keys:
        sse = torch.cat(stats_parts)[:, 0].cpu().numpy()
        with np.errstate(divide='ignore'):
            out['PSNR'] = 20 * np.log10(255.0 / np.sqrt(sse / (hc * wc)))
    if 'SSIM' in keys:
        out['SSIM'] = torch.cat(ssim_parts).cpu().numpy()
    if tof:
        out['tOF'] = (torch.cat(epe_parts).cpu().numpy() / (hc * wc)) if epe_parts else np.zeros(0)
    return out


def official_averages(per_sequence):
    """The totals the official metric script prints and writes for a list of sequences (its folders), each a dict of
    per-frame arrays as official_sequence_metrics returns them.  Like the script, each sequence's list is cast to
    float32 first.  Returns {'FrameAvg_<key>': the mean over all frames, 'FolderAvg_<key>': the mean of the
    per-sequence means, 'Avg_<key>': float32 [sequences] of the per-sequence means} for every key of the dicts."""
    if not per_sequence:
        raise ValueError('official_averages needs at least one sequence')
    keys = [k for k in per_sequence[0]]
    if any(list(d) != keys for d in per_sequence):
        raise ValueError('every sequence must have the same keys')
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
