"""LPIPS (net-lin, AlexNet, v0.1) in float64: the specification of tecogan_b200.metrics.LPIPS and of the layouts of
csrc/tg_lpips.cu (include/tecogan_b200.h).

Both of TecoGAN's copies (codes/metrics/LPIPS and codes/official_metrics/LPIPSmodels) compute
  d(x0, x1) = sum_l mean_hw( sum_c w_lc (f0 / (|f0|_c + 1e-10) - f1 / (|f1|_c + 1e-10))^2 )
over the five ReLU outputs f of torchvision's AlexNet features of the ScalingLayer'd inputs.  The input is
x * 2 / 255 - 1 (MetricCalculator) or x / 127.5 - 1 (the official script's util.im2tensor).

`features` is the direct network; `features_remapped` runs it the way the device does: conv1 as a valid 3x3 conv over
the space-to-depth(4) picture, conv2 as a 3x3 conv over four shifted copies of the pooled map, both on grids one
pixel larger on every side, and the pools on the interiors.  params: a dict of numpy arrays under torchvision's keys
(synthetic.make_lpips_params)."""
import numpy as np
import torch
import torch.nn.functional as F

SHIFT = np.float32([-.030, -.088, -.188]).astype(np.float64)
SCALE = np.float32([.458, .448, .450]).astype(np.float64)
CONVS = (0, 3, 6, 8, 10)
MIN_SIDE = 31


def _t(a, device='cpu'):
    return torch.from_numpy(np.asarray(a, np.float64)).to(device)


def scaled_input(u8, norm='calc'):
    """uint8 [N, H, W, 3] -> float64 [N, 3, H, W], normalised ('calc': x * 2 / 255 - 1, 'official': x / 127.5 - 1)
    and scaled by PNetLin's ScalingLayer"""
    x = np.asarray(u8, np.float64)
    x = x * 2 / 255 - 1 if norm == 'calc' else x / 127.5 - 1
    x = (x - SHIFT) / SCALE
    return _t(x.transpose(0, 3, 1, 2).copy())


def features(params, x):
    """the five ReLU outputs of AlexNet (torchvision's features[0:12] in PNetLin's slices) of x [N, 3, H, W], on
    x's device"""
    w = [(_t(params[f'features.{i}.weight'], x.device), _t(params[f'features.{i}.bias'], x.device)) for i in CONVS]
    f1 = F.relu(F.conv2d(x, *w[0], stride=4, padding=2))
    f2 = F.relu(F.conv2d(F.max_pool2d(f1, 3, 2), *w[1], padding=2))
    f3 = F.relu(F.conv2d(F.max_pool2d(f2, 3, 2), *w[2], padding=1))
    f4 = F.relu(F.conv2d(f3, *w[3], padding=1))
    f5 = F.relu(F.conv2d(f4, *w[4], padding=1))
    return [f1, f2, f3, f4, f5]


# ---- the device's layouts ---------------------------------------------------------------------------------------
def s2d_input(x):
    """conv1's input: space_to_depth(4) of x [N, 3, H, W] zero-padded by 2 at the top and left, on the
    (oh+2) x (ow+2) grid, channel (py*4 + px)*3 + c -> [N, 48, oh+2, ow+2]"""
    N, _, H, W = x.shape
    hs, ws = (H - 7) // 4 + 3, (W - 7) // 4 + 3
    xp = torch.zeros(N, 3, 4 * hs, 4 * ws, dtype=x.dtype)
    hh, ww = min(H, 4 * hs - 2), min(W, 4 * ws - 2)
    xp[:, :, 2:2 + hh, 2:2 + ww] = x[:, :, :hh, :ww]
    return xp.view(N, 3, hs, 4, ws, 4).permute(0, 3, 5, 1, 2, 4).reshape(N, 48, hs, ws)


def conv1_weight(w):
    """[64, 3, 11, 11] -> [64, 48, 3, 3]: zero-padded to 12 x 12 and split like s2d_input"""
    w12 = torch.zeros(64, 3, 12, 12, dtype=w.dtype)
    w12[:, :, :11, :11] = w
    return w12.view(64, 3, 3, 4, 3, 4).permute(0, 3, 5, 1, 2, 4).reshape(64, 48, 3, 3)


def shifted_input(p):
    """conv2's input: four copies of the pooled map p [N, 64, h, w] on the (h+2) x (w+2) grid, copy b = by*2 + bx
    at grid pixel (i, j) = p[i + 3by - 2, j + 3bx - 2] (zero outside) -> [N, 256, h+2, w+2]"""
    N, C, h, w = p.shape
    pp = F.pad(p, (4, 4, 4, 4))
    return torch.cat([pp[:, :, 3 * by + 2:3 * by + 2 + h + 2, 3 * bx + 2:3 * bx + 2 + w + 2]
                      for by in (0, 1) for bx in (0, 1)], 1)


def conv2_weight(w):
    """[192, 64, 5, 5] -> [192, 256, 3, 3]: zero-padded to 6 x 6 and split into four 3x3 blocks"""
    w6 = torch.zeros(192, 64, 6, 6, dtype=w.dtype)
    w6[:, :, :5, :5] = w
    return torch.cat([w6[:, :, 3 * by:3 * by + 3, 3 * bx:3 * bx + 3] for by in (0, 1) for bx in (0, 1)], 1)


def features_remapped(params, x):
    """features() through the device's layouts: returns the five features as the device stores them (conv1's and
    conv2's on their grids, the feature being the interior [1:-1, 1:-1]) and the pooled maps"""
    w = [(_t(params[f'features.{i}.weight']), _t(params[f'features.{i}.bias'])) for i in CONVS]
    g1 = F.relu(F.conv2d(s2d_input(x), conv1_weight(w[0][0]), w[0][1], padding=1))
    p1 = F.max_pool2d(g1[:, :, 1:-1, 1:-1], 3, 2)
    g2 = F.relu(F.conv2d(shifted_input(p1), conv2_weight(w[1][0]), w[1][1], padding=1))
    p2 = F.max_pool2d(g2[:, :, 1:-1, 1:-1], 3, 2)
    f3 = F.relu(F.conv2d(p2, *w[2], padding=1))
    f4 = F.relu(F.conv2d(f3, *w[3], padding=1))
    f5 = F.relu(F.conv2d(f4, *w[4], padding=1))
    return {'grid1': g1, 'pool1': p1, 'grid2': g2, 'pool2': p2, 'f3': f3, 'f4': f4, 'f5': f5}


def layer_distance(f0, f1, w):
    """one layer's term: mean_hw sum_c w_c (f0 / (|f0| + 1e-10) - f1 / (|f1| + 1e-10))^2 -> float64 [N]"""
    n0 = f0 / (torch.sqrt((f0 ** 2).sum(1, keepdim=True)) + 1e-10)
    n1 = f1 / (torch.sqrt((f1 ** 2).sum(1, keepdim=True)) + 1e-10)
    return ((n0 - n1) ** 2 * _t(w, f0.device).reshape(1, -1, 1, 1)).sum(1).mean((1, 2))


def lpips(params, u0, u1, norm='calc', device='cpu'):
    """d(u0[i], u1[i]) for uint8 RGB frames [N, H, W, 3] (one size, at least 31 x 31) -> float64 [N] numpy; the
    float64 arithmetic runs on `device` (a CUDA device makes large pictures fast)"""
    fa = features(params, scaled_input(u0, norm).to(device))
    fb = features(params, scaled_input(u1, norm).to(device))
    d = sum(layer_distance(a, b, params[f'lin{l}.model.1.weight']) for l, (a, b) in enumerate(zip(fa, fb)))
    return d.cpu().numpy()


def crop_8x8(n):
    size = (n // 32) * 32
    while size > n - 16:
        size -= 32
    return (n - size) // 2, size


def official_lpips(params, true, pred, cutfr=2):
    """the official script's LPIPS and tLP100 of two sequences [T, H, W, 3] (cropped to their common size, then
    crop_8x8): LPIPS of frames cutfr .. T-cutfr-1, tLP100 (float32 as the script forms it) from cutfr + 1 on, and
    the two distances tLP100 is made of, d_true = d(true[i-1], true[i]) and d_pred = d(pred[i-1], pred[i])"""
    T = true.shape[0]
    h, w = min(true.shape[1], pred.shape[1]), min(true.shape[2], pred.shape[2])
    (y0, hc), (x0, wc) = crop_8x8(h), crop_8x8(w)
    t = np.asarray(true)[cutfr:T - cutfr, y0:y0 + hc, x0:x0 + wc]
    p = np.asarray(pred)[cutfr:T - cutfr, y0:y0 + hc, x0:x0 + wc]
    lp = lpips(params, t, p, 'official')
    d0 = lpips(params, t[:-1], t[1:], 'official') if len(t) > 1 else np.zeros(0)
    d1 = lpips(params, p[:-1], p[1:], 'official') if len(p) > 1 else np.zeros(0)
    tlp = np.absolute(np.float32(d0) - np.float32(d1)) * np.float32(100.0)
    return {'LPIPS': lp, 'tLP100': tlp.astype(np.float64), 'd_true': d0, 'd_pred': d1}
