"""Video quality metrics on the device: PSNR, LPIPS and tOF as TecoGAN's MetricCalculator computes them
(codes/metrics/metric_calculator.py: compute_PSNR, compute_LPIPS, compute_tOF), on the kernels of csrc/tg_metrics.cu
and csrc/tg_lpips.cu, and the official metric script's PSNR, SSIM, LPIPS, tOF and tLP100.

- PSNR: the per-frame sum of squared differences is an exact integer from the device; the host finishes it with the
  reference's float64 expression, so the values are identical to the reference's, bit for bit.
- LPIPS: net-lin AlexNet v0.1 (LPIPS below) with the caller's weights; its convs run on the fp16 wgmma conv kernel.
- tOF: the mean end-point error between the Farneback flows (cv2.calcOpticalFlowFarneback, flags=0) of consecutive
  ground-truth frames and of consecutive predicted frames, computed in fp32 on the device.
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


# ---- LPIPS (net-lin, AlexNet, v0.1) ----------------------------------------------------------------------------------

_ALEX_CONVS = (0, 3, 6, 8, 10)                 # torchvision alexnet().features indices of the five convs
_ALEX_SHAPES = ((64, 3, 11, 11), (192, 64, 5, 5), (384, 192, 3, 3), (256, 384, 3, 3), (256, 256, 3, 3))
_SLICE_OF = (1, 2, 3, 4, 5)                    # pretrained_networks.alexnet: conv l sits in slice l + 1 ...
_SLICE_IDX = (0, 3, 6, 8, 10)                  # ... under its features index


def _lpips_weights(state_dict):
    """the five conv weights / biases and five heads of an LPIPS state_dict, as float32 CPU tensors"""
    def get(keys, shape):
        for k in keys:
            if k in state_dict:
                v = state_dict[k]
                v = v.detach().cpu() if isinstance(v, torch.Tensor) else torch.from_numpy(np.asarray(v))
                if tuple(v.shape) != tuple(shape):
                    raise ValueError(f'{k} has shape {tuple(v.shape)}, expected {tuple(shape)}')
                return v.to(torch.float32)
        raise ValueError(f'the state_dict has none of {keys}')
    convs, heads = [], []
    for l, (fi, shape) in enumerate(zip(_ALEX_CONVS, _ALEX_SHAPES)):
        names = (f'features.{fi}', f'net.slice{_SLICE_OF[l]}.{_SLICE_IDX[l]}')
        convs.append((get([n + '.weight' for n in names], shape), get([n + '.bias' for n in names], shape[:1])))
        heads.append(get([f'lin{l}.model.1.weight'], (1, shape[0], 1, 1)).reshape(-1))
    return convs, heads


def _lpips_conv1_weight(w):
    """conv1 (11x11, stride 4) as a 3x3 conv over the space-to-depth(4) input: [64, 48, 3, 3], channel (py*4+px)*3+c"""
    w12 = torch.zeros(64, 3, 12, 12, dtype=w.dtype, device=w.device)
    w12[:, :, :11, :11] = w
    return w12.view(64, 3, 3, 4, 3, 4).permute(0, 3, 5, 1, 2, 4).reshape(64, 48, 3, 3).contiguous()


def _lpips_conv2_weight(w):
    """conv2 (5x5) as a 3x3 conv over four shifted copies of its input: [192, 256, 3, 3], block b = by*2+bx"""
    w6 = torch.zeros(192, 64, 6, 6, dtype=w.dtype, device=w.device)
    w6[:, :, :5, :5] = w
    return torch.cat([w6[:, :, 3 * by:3 * by + 3, 3 * bx:3 * bx + 3] for by in (0, 1) for bx in (0, 1)], 1).contiguous()


def lpips_sizes(h, w):
    """per layer (the stored map's height and width, the interior (y0, x0, h, w) that is the feature) for an h x w
    picture: conv1 and conv2 run on grids one pixel larger on every side than their output"""
    oh, ow = (h - 7) // 4 + 1, (w - 7) // 4 + 1
    p1h, p1w = (oh - 3) // 2 + 1, (ow - 3) // 2 + 1
    p2h, p2w = (p1h - 3) // 2 + 1, (p1w - 3) // 2 + 1
    return [((oh + 2, ow + 2), (1, 1, oh, ow)), ((p1h + 2, p1w + 2), (1, 1, p1h, p1w))] + \
        [((p2h, p2w), (0, 0, p2h, p2w))] * 3


class LPIPS:
    """LPIPS (net-lin, AlexNet, v0.1) on the device, as both of TecoGAN's LPIPS copies compute it.

    state_dict: AlexNet's conv weights and biases under torchvision's keys features.{0,3,6,8,10}.* or the LPIPS
    package's net.slice{1..5}.N.*, and the heads lin{0..4}.model.1.weight ([1, C, 1, 1]).  Other keys are ignored;
    a missing or mis-shaped key raises ValueError.  MetricCalculator's DistModel.net.state_dict() has all of them;
    for the official script's copy (its AlexNet is not a registered module) merge torchvision's
    alexnet().state_dict() with the heads of weights/v0.1/alex.pth.  The weights are packed once, on `device`
    (default: the current CUDA device).

    lp(true, pred, max_workspace_bytes=2 GB): uint8 RGB frames [N, H, W, 3] (numpy or CUDA tensors, cropped to their
    common top-left size, at least 31 x 31) -> float64 [N] numpy, with MetricCalculator's input normalisation
    (x * 2 / 255 - 1).  The frames are scored in chunks whose device memory stays within max_workspace_bytes."""

    def __init__(self, state_dict, device=None):
        convs, heads = _lpips_weights(state_dict)
        self.device = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
        if self.device.type != 'cuda':
            raise ValueError(f'LPIPS runs on a CUDA device, got {self.device}')
        dev = self.device
        with torch.cuda.device(dev):
            ws = [_lpips_conv1_weight(convs[0][0]), _lpips_conv2_weight(convs[1][0])] + [c[0] for c in convs[2:]]
            self.convs = [ops.PackedConv(w.to(dev), b.to(dev), L.CONV_3X3, L.ACT_RELU, L.EPI_NHWC_F16)
                          for w, (_, b) in zip(ws, convs)]
            self.heads = [h.to(dev).contiguous() for h in heads]
            torch.cuda.current_stream().synchronize()   # the packers read the staged weights

    @staticmethod
    def image_bytes(h, w):
        """device bytes of one h x w picture's input map and features"""
        sz = lpips_sizes(h, w)
        (g1h, g1w), (g2h, g2w), (p2h, p2w) = sz[0][0], sz[1][0], sz[2][0]
        return 2 * (g1h * g1w * 64 * 2 + g2h * g2w * (256 + 192) + p2h * p2w * (192 + 384 + 256 + 256))

    def features(self, frames, window, norm):
        """frames: uint8 CUDA [n, H, W, 3], window (y0, x0, h, w) of them, norm L.LPIPS_NORM_* -> the five ReLU
        outputs as stored, fp16 NHWC (conv1's and conv2's on their grids: the feature is lpips_sizes' interior)"""
        n, (_, _, h, w) = frames.shape[0], window
        if h < L.LPIPS_MIN_SIDE or w < L.LPIPS_MIN_SIDE:
            raise ValueError(f'LPIPS needs at least {L.LPIPS_MIN_SIDE}x{L.LPIPS_MIN_SIDE} pixels, got {h}x{w}')
        sz = lpips_sizes(h, w)
        x = ops.lpips_frames_in(frames, window, norm,
                                torch.empty(n, *sz[0][0], 64, dtype=torch.float16, device=frames.device))
        f1 = self.convs[0](x)
        f2 = self.convs[1](ops.maxpool3x3s2(f1, sz[0][1], shifts=True))
        f3 = self.convs[2](ops.maxpool3x3s2(f2, sz[1][1], shifts=False))
        f4 = self.convs[3](f3)
        return [f1, f2, f3, f4, self.convs[4](f4)]

    def distances(self, frames, window, norm, pairs):
        """frames: uint8 CUDA [n, H, W, 3] (the batch), window (y0, x0, h, w) of them, norm L.LPIPS_NORM_*, pairs:
        index pairs into the batch -> float64 CUDA [len(pairs)], the LPIPS of each pair"""
        feats = self.features(frames, window, norm)
        sz = lpips_sizes(*window[2:])
        pairs = torch.tensor(pairs, dtype=torch.int32).reshape(-1, 2).to(frames.device)
        out = torch.empty(pairs.shape[0], dtype=torch.float64, device=frames.device)
        for l, f in enumerate(feats):
            ops.lpips_head(f, sz[l][1], pairs, self.heads[l], out, accumulate=l > 0)
        return out

    def __call__(self, true, pred, max_workspace_bytes=DEFAULT_MAX_WORKSPACE_BYTES):
        true, pred = _frames(true, 'true'), _frames(pred, 'pred')
        N = true.shape[0]
        if pred.shape[0] != N:
            raise ValueError(f'true has {N} frames, pred {pred.shape[0]}')
        h, w = min(true.shape[1], pred.shape[1]), min(true.shape[2], pred.shape[2])
        if h < L.LPIPS_MIN_SIDE or w < L.LPIPS_MIN_SIDE:
            raise ValueError(f'LPIPS needs at least {L.LPIPS_MIN_SIDE}x{L.LPIPS_MIN_SIDE} pixels, got {h}x{w}')
        if N == 0:
            return np.zeros(0)
        full = true.shape[1] * true.shape[2] * 3 + pred.shape[1] * pred.shape[2] * 3

        def chunk_bytes(n):      # the uint8 frames as given and cropped, the features, the distances, the heads' work
            return (n * full + 2 * n * h * w * 3 + 2 * n * self.image_bytes(h, w) + n * 8
                    + 5 * ops.lpips_head_workspace_bytes(n, h, w))
        n = N
        while n > 1 and chunk_bytes(n) > max_workspace_bytes:
            n -= 1
        if chunk_bytes(n) > max_workspace_bytes:
            raise ValueError(f'max_workspace_bytes={max_workspace_bytes} is below the {chunk_bytes(1)} bytes that one '
                             f'pair of {h}x{w} frames needs')
        parts = []
        with torch.cuda.device(self.device):
            for s in range(0, N, n):
                e = min(s + n, N)
                batch = _lpips_batch(_chunk(true, s, e, self.device), _chunk(pred, s, e, self.device), h, w)
                parts.append(self.distances(batch, (0, 0, h, w), L.LPIPS_NORM_CALC,
                                            [(i, e - s + i) for i in range(e - s)]))
            return torch.cat(parts).cpu().numpy()


def _check_lpips(lpips, true_seq, pred_seq):
    if not isinstance(lpips, LPIPS):
        raise ValueError(f'lpips must be a tecogan_b200.metrics.LPIPS, got {type(lpips).__name__}')
    for x in (true_seq, pred_seq):
        if isinstance(x, torch.Tensor) and x.device != lpips.device:
            raise ValueError(f'frames on {x.device}, LPIPS weights on {lpips.device}')


def _lpips_batch(tc, pc, h, w):
    """the chunk's true and pred frames cropped to (h, w), as one uint8 CUDA batch [2m, h, w, 3] (true first)"""
    return torch.cat([tc[:, :h, :w], pc[:, :h, :w]]).contiguous()


def psnr_from_sse(sse, count):
    """compute_PSNR's float64 expression from the exact per-frame integer SSE: 20 log10(255 / sqrt(sse / count)),
    inf where the frames are equal."""
    out = np.empty(len(sse))
    for i, s in enumerate(sse):
        rmse = np.sqrt(np.float64(int(s)) / count)
        out[i] = np.inf if rmse == 0 else 20 * np.log10(255.0 / rmse)
    return out


def sequence_metrics(true_seq, pred_seq, psnr='y', tof=True, max_workspace_bytes=DEFAULT_MAX_WORKSPACE_BYTES,
                     lpips=None):
    """PSNR, LPIPS and tOF of a predicted sequence against its ground truth, as
    MetricCalculator.compute_sequence_metrics computes them frame by frame.

    true_seq, pred_seq: uint8 RGB frames [T, H, W, 3], host numpy arrays or CUDA tensors (the device is theirs, or
    the current CUDA device for numpy input).  Frames of different sizes are cropped to the smaller height and width
    (their top-left corner), as the reference does.
    psnr: 'y' (the Y of data_utils.rgb_to_ycbcr), 'rgb', or None.  tof: whether to compute tOF (always on gray
    frames, as compute_tOF does).
    max_workspace_bytes: bound on the device memory of the tOF and LPIPS passes; a longer sequence is scored in chunks
    of consecutive frames (that overlap by one frame with tOF).
    lpips: an LPIPS (its weights' device must be the frames'), or None for no LPIPS.

    Returns {'PSNR': float64 [T]}, {'LPIPS': float64 [T]} and / or {'tOF': float64 [T - 1]} (numpy), in that order."""
    true_seq, pred_seq = _frames(true_seq, 'true_seq'), _frames(pred_seq, 'pred_seq')
    if psnr not in ('y', 'rgb', None):
        raise ValueError(f"psnr must be 'y', 'rgb' or None, got {psnr!r}")
    if not isinstance(tof, bool):
        raise ValueError(f'tof must be a bool, got {tof!r}')
    T = true_seq.shape[0]
    if pred_seq.shape[0] != T:
        raise ValueError(f'true_seq has {T} frames, pred_seq {pred_seq.shape[0]}')
    h, w = min(true_seq.shape[1], pred_seq.shape[1]), min(true_seq.shape[2], pred_seq.shape[2])
    if lpips is not None:
        _check_lpips(lpips, true_seq, pred_seq)
        if h < L.LPIPS_MIN_SIDE or w < L.LPIPS_MIN_SIDE:
            raise ValueError(f'LPIPS needs at least {L.LPIPS_MIN_SIDE}x{L.LPIPS_MIN_SIDE} pixels, got {h}x{w}')
    out = {}
    if T == 0 or (psnr is None and not tof and lpips is None):
        if psnr is not None:
            out['PSNR'] = np.zeros(0)
        if lpips is not None:
            out['LPIPS'] = np.zeros(0)
        if tof:
            out['tOF'] = np.zeros(0)
        return out
    device = next((x.device for x in (true_seq, pred_seq) if isinstance(x, torch.Tensor)),
                  lpips.device if lpips is not None else torch.device('cuda', torch.cuda.current_device()))
    mode = {'y': L.PSNR_Y, 'rgb': L.PSNR_RGB, None: L.PSNR_NONE}[psnr]
    hw = h * w
    if (tof and T >= 2) or lpips is not None:
        def chunk_bytes(n):
            b = 0
            if tof:
                b += (ops.farneback_workspace_bytes(2, n, h, w) + 2 * n * hw + 2 * (n - 1) * hw * 8
                      + 2 * n * hw * 3 * 2)
            if lpips is not None:
                b += 2 * n * hw * 3 * 2 + 2 * n * LPIPS.image_bytes(h, w) + n * 8
                b += 5 * ops.lpips_head_workspace_bytes(n, h, w)
            return b
        n, n_min = T, (2 if tof and T >= 2 else 1)
        while n > n_min and chunk_bytes(n) > max_workspace_bytes:
            n -= 1
        if chunk_bytes(n) > max_workspace_bytes:
            raise ValueError(f'max_workspace_bytes={max_workspace_bytes} is below the {chunk_bytes(n)} bytes that '
                             f'{n} frames of {h}x{w} need')
    else:
        n = T
    sse_parts, epe_parts, lp_parts = [], [], []
    with torch.cuda.device(device):
        s = 0
        while True:
            e = min(s + n, T)
            tc, pc = _chunk(true_seq, s, e, device), _chunk(pred_seq, s, e, device)
            m = e - s
            gray = torch.empty(2, m, h, w, dtype=torch.uint8, device=device) if tof else None
            sse = ops.metrics_frames_in(tc, pc, mode, gray)
            if sse is not None:
                sse_parts.append(sse if s == 0 or not tof else sse[1:])
            if lpips is not None:
                k0 = 1 if s > 0 and tof else 0
                lp_parts.append(lpips.distances(_lpips_batch(tc, pc, h, w), (0, 0, h, w), L.LPIPS_NORM_CALC,
                                                [(i, m + i) for i in range(k0, m)]))
            if tof and m >= 2:
                flow = ops.farneback(gray.view(2 * m, h, w), 2, _check_farneback_args(0.5, 3, 15, 3, 5, 1.2, 0))
                epe_parts.append(ops.flow_epe_sum(flow[:m - 1], flow[m - 1:]))
            if e == T:
                break
            s = e - 1 if tof else e
    if psnr is not None:
        sse = torch.cat(sse_parts).cpu().numpy().view(np.uint64)
        out['PSNR'] = psnr_from_sse(sse, hw * (3 if psnr == 'rgb' else 1))
    if lpips is not None:
        out['LPIPS'] = torch.cat(lp_parts).cpu().numpy()
    if tof:
        out['tOF'] = (torch.cat(epe_parts).cpu().numpy() / hw) if epe_parts else np.zeros(0)
    return out


# ---- the official metric script (codes/official_metrics/metrics.py) -------------------------------------------------

OFFICIAL_KEYS = ('PSNR', 'SSIM', 'tOF')
OFFICIAL_LPIPS_KEYS = ('PSNR', 'SSIM', 'LPIPS', 'tOF', 'tLP100')   # the script's order, with an LPIPS model
OFFICIAL_MIN_SIDE = 48                     # the smallest side whose crop_8x8 is not empty


def crop_8x8(n):
    """(offset, size) of the official script's crop_8x8 along a side of n >= 48 pixels: the largest multiple of 32
    that is <= n - 16, centred at (n - size) // 2"""
    size = (n // 32) * 32
    while size > n - 16:
        size -= 32
    return (n - size) // 2, size


def official_sequence_metrics(true_seq, pred_seq, cutfr=2, keys=OFFICIAL_KEYS,
                              max_workspace_bytes=DEFAULT_MAX_WORKSPACE_BYTES, lpips=None):
    """PSNR, SSIM, LPIPS, tOF and tLP100 of a predicted sequence as TecoGAN's official metric script (the one behind
    the paper's tables) computes them frame by frame, on the device.

    true_seq, pred_seq: uint8 RGB frames [T, H, W, 3], host numpy arrays or CUDA tensors, as sequence_metrics takes
    them.  Both are cropped to their common top-left size (h, w), which must be at least 48 x 48; crop_8x8 of it is
    the scored window.  Frames cutfr .. T - cutfr - 1 are scored:
      PSNR  20 log10(255 / RMSE) of the unrounded float64 Y of _rgb2ycbcr over the window (inf on equal frames)
      SSIM  skimage compare_ssim of those Y (7x7 uniform window), data_range = max - min of the predicted Y
      LPIPS d(true, pred) of the window (LPIPS with the script's input normalisation x / 127.5 - 1)
      tOF   from frame cutfr + 1 on: the mean end-point error over the window of the Farneback flows of the full
            common-size gray frames (flow of frame i - 1 -> i, ground truth against prediction)
      tLP100 from frame cutfr + 1 on: |d(true[i-1], true[i]) - d(pred[i-1], pred[i])| * 100 of the windows, formed in
            float32 as the script does
    keys: the metrics to compute, a subset of OFFICIAL_KEYS, or of OFFICIAL_LPIPS_KEYS when `lpips` (an LPIPS, on
    the frames' device) is given.  max_workspace_bytes bounds the device memory of the pass; a longer sequence is
    scored in chunks of consecutive frames that overlap by one frame.

    Returns {key: float64 numpy array} in the order of OFFICIAL_LPIPS_KEYS: PSNR, SSIM and LPIPS of T - 2 cutfr
    frames, tOF and tLP100 of T - 2 cutfr - 1 (empty arrays when there are too few frames)."""
    true_seq, pred_seq = _frames(true_seq, 'true_seq'), _frames(pred_seq, 'pred_seq')
    allowed = OFFICIAL_KEYS if lpips is None else OFFICIAL_LPIPS_KEYS
    if isinstance(keys, str) or not all(isinstance(k, str) and k in allowed for k in keys):
        raise ValueError(f'keys must be a subset of {allowed}' +
                         ('' if lpips is not None else " ('LPIPS' and 'tLP100' need an LPIPS model: lpips=)") +
                         f', got {keys!r}')
    if lpips is not None:
        _check_lpips(lpips, true_seq, pred_seq)
    if not isinstance(cutfr, (int, np.integer)) or isinstance(cutfr, bool) or cutfr < 0:
        raise ValueError(f'cutfr must be a non-negative integer, got {cutfr!r}')
    T = true_seq.shape[0]
    if pred_seq.shape[0] != T:
        raise ValueError(f'true_seq has {T} frames, pred_seq {pred_seq.shape[0]}')
    h, w = min(true_seq.shape[1], pred_seq.shape[1]), min(true_seq.shape[2], pred_seq.shape[2])
    if h < OFFICIAL_MIN_SIDE or w < OFFICIAL_MIN_SIDE:
        raise ValueError(f'the common frame size {h}x{w} is below {OFFICIAL_MIN_SIDE}x{OFFICIAL_MIN_SIDE}: its '
                         f'crop_8x8 is empty')
    keys = [k for k in OFFICIAL_LPIPS_KEYS if k in keys]
    tof = 'tOF' in keys
    tlp = 'tLP100' in keys
    lp_wanted = 'LPIPS' in keys or tlp
    overlap = tof or tlp                       # the temporal metrics need a chunk's previous frame
    stats_wanted = 'PSNR' in keys or 'SSIM' in keys
    (y0, hc), (x0, wc) = crop_8x8(h), crop_8x8(w)
    window = (y0, x0, hc, wc)
    n_s = max(T - 2 * cutfr, 0)
    if n_s == 0 or not keys:
        return {k: np.zeros(0) for k in keys}
    true_seq, pred_seq = true_seq[cutfr:T - cutfr], pred_seq[cutfr:T - cutfr]
    device = next((x.device for x in (true_seq, pred_seq) if isinstance(x, torch.Tensor)),
                  lpips.device if lpips is not None else torch.device('cuda', torch.cuda.current_device()))
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
        if lp_wanted:
            b += 2 * n * hc * wc * 3 + 2 * n * LPIPS.image_bytes(hc, wc) + 3 * n * (8 + 8)
            b += 5 * ops.lpips_head_workspace_bytes(3 * n, hc, wc)
        return b
    n, n_min = n_s, min(n_s, 2 if overlap else 1)     # overlapping chunks need two frames
    while n > n_min and chunk_bytes(n) > max_workspace_bytes:
        n -= 1
    if chunk_bytes(n) > max_workspace_bytes:
        raise ValueError(f'max_workspace_bytes={max_workspace_bytes} is below the {chunk_bytes(n)} bytes that '
                         f'{n} frames of {h}x{w} need')
    params = _check_farneback_args(0.5, 3, 15, 3, 5, 1.2, 0) if tof else None
    stats_parts, ssim_parts, epe_parts, lp_parts, tlp_parts = [], [], [], [], []
    with torch.cuda.device(device):
        s = 0
        while True:
            e = min(s + n, n_s)
            tc, pc = _chunk(true_seq, s, e, device), _chunk(pred_seq, s, e, device)
            m = e - s
            # with tOF / tLP100 a chunk's first frame is the last one's last frame, whose PSNR / SSIM / LPIPS are kept
            new = slice(1 if s > 0 and overlap else 0, None)
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
            if lp_wanted:
                # true frames 0 .. m-1, pred frames m .. 2m-1 of the batch: (true_i, pred_i) for LPIPS, then the
                # consecutive (true_{i-1}, true_i) and (pred_{i-1}, pred_i) for tLP100; each frame's features once
                first = new.start
                pairs = [(i, m + i) for i in range(first, m)] if 'LPIPS' in keys else []
                if tlp:
                    pairs += [(i - 1, i) for i in range(1, m)] + [(m + i - 1, m + i) for i in range(1, m)]
                if pairs:
                    batch = torch.cat([tc[:, y0:y0 + hc, x0:x0 + wc], pc[:, y0:y0 + hc, x0:x0 + wc]]).contiguous()
                    d = lpips.distances(batch, (0, 0, hc, wc), L.LPIPS_NORM_OFFICIAL, pairs).cpu().numpy()
                    k = m - first if 'LPIPS' in keys else 0
                    if 'LPIPS' in keys:
                        lp_parts.append(d[:k])
                    if tlp:
                        tlp_parts.append((d[k:k + m - 1], d[k + m - 1:]))
            if e == n_s:
                break
            s = e - 1 if overlap else e
    out = {}
    if 'PSNR' in keys:
        sse = torch.cat(stats_parts)[:, 0].cpu().numpy()
        with np.errstate(divide='ignore'):
            out['PSNR'] = 20 * np.log10(255.0 / np.sqrt(sse / (hc * wc)))
    if 'SSIM' in keys:
        out['SSIM'] = torch.cat(ssim_parts).cpu().numpy()
    if 'LPIPS' in keys:
        out['LPIPS'] = np.concatenate(lp_parts)
    if tof:
        out['tOF'] = (torch.cat(epe_parts).cpu().numpy() / (hc * wc)) if epe_parts else np.zeros(0)
    if tlp:
        d0 = np.concatenate([np.float32(a) for a, _ in tlp_parts]) if tlp_parts else np.zeros(0, np.float32)
        d1 = np.concatenate([np.float32(b) for _, b in tlp_parts]) if tlp_parts else np.zeros(0, np.float32)
        out['tLP100'] = (np.absolute(d0 - d1) * np.float32(100.0)).astype(np.float64)   # the script's float32
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
