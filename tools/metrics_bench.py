"""Throughput of tecogan_b200.metrics.sequence_metrics (PSNR-Y + tOF) on bd4 HR sequences (536x1280, T = 32): scored
frames/s end to end (host uint8 frames in, float64 metrics out), per-phase kernel times from CUDA events, the bytes
each phase must move (from shapes) and their share of the H100 SXM's 3.35 TB/s, and the reference formulas
(cv2 Farneback + numpy PSNR, as MetricCalculator runs them) on the host cores for comparison.

    python tools/metrics_bench.py [--seqs 4] [--ref-frames 4] [--out metrics_bench.json]

--official measures official_sequence_metrics (the official metric script's PSNR, SSIM and tOF on the crop_8x8
window, frames 2 .. T-3) instead: scored frames/s end to end, per-kernel times from CUDA events, the algorithmic
bytes and TB/s of the Y statistics and SSIM kernels, and oracle/official_metrics.py (cv2 + scipy) on the host cores.

--lpips measures all five official keys (PSNR, SSIM, LPIPS, tOF, tLP100) with seeded AlexNet weights
(synthetic.make_lpips_params): scored frames/s end to end, per-kernel times of one LPIPS pass over a chunk's frames
from CUDA events, the AlexNet convs' TFLOP/s (by the reference counter's convention, 2 x MACs of the unpadded convs,
and as executed on the padded layouts) against the 989 TFLOP/s of dense FP16, and the reference's PNetLin (from
oracle/_ref) on the same frames with cuDNN at PyTorch's defaults.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import tecogan_b200 as T      # noqa: E402
import synthetic              # noqa: E402

M, ops, L = T.metrics, T.ops, sys.modules['tecogan-pytorch_b200.lib']
HBM = 3.35e12


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # noqa: BLE001
        q = f'nvidia-smi unavailable: {e}'
    return {'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi': q}


def sequence(seed, T_=32, h=536, w=1280):
    clip = synthetic.make_clip(seed, T_, 3, h, w, shift=2)
    true = np.ascontiguousarray((clip.permute(0, 2, 3, 1) * 255).round().to(torch.uint8).numpy())
    rng = np.random.default_rng(seed + 100)
    pred = np.clip(true.astype(np.int16) + rng.integers(-6, 7, true.shape), 0, 255).astype(np.uint8)
    return true, pred


def level_sizes(h, w, pyr_scale=0.5, levels=3):
    """pyramid level sizes of tOF's Farneback, coarsest first: the level count stops where a side drops below 32"""
    k = 0
    while k < levels and min(h, w) * pyr_scale ** (k + 1) >= 32:
        k += 1
    return [(int(np.rint(h * pyr_scale ** i)), int(np.rint(w * pyr_scale ** i))) for i in range(k, -1, -1)]


def phase_bytes(T_, h, w):
    """algorithmic bytes per phase for one T_-frame sequence (2T_ gray frames, 2(T_-1) flows), each buffer read or
    written once per pass"""
    n, p, hw = 2 * T_, 2 * (T_ - 1), h * w
    b = {'frames_in': 2 * T_ * hw * 3 + n * hw + 8 * T_}
    pyr = flow = 0
    for lh, lw in level_sizes(h, w):
        lhw = lh * lw
        pyr += n * (hw + lh * w * 4) + n * (lh * w * 4 + lhw * 4)        # blur + resize: V and H passes
        pyr += n * (lhw * 4 + 3 * lhw * 4) + n * (3 * lhw * 4 + 5 * lhw * 4)   # poly V and H
        flow += p * (5 * lhw * 4 * 2 + 8 * lhw)                          # init: R0 + R1 reads, M + flow writes
        flow += 3 * p * (5 * lhw * 4 + 8 * lhw) + 2 * p * (5 * lhw * 4 * 3)   # iterations: M in, flow, R0/R1, M out
    b['pyramid+poly'] = pyr
    b['flow'] = flow
    b['epe'] = p * hw * 8
    return b


def timed_phases(true, pred):
    """one chunk-free run of the phases with CUDA events around each"""
    dev = torch.device('cuda:0')
    T_, h, w = true.shape[:3]
    tc, pc = torch.from_numpy(true).to(dev), torch.from_numpy(pred).to(dev)
    gray = torch.empty(2, T_, h, w, dtype=torch.uint8, device=dev)
    params = ops.farneback_params(0.5, 3, 15, 3, 5, 1.2, 0)
    work = torch.empty(ops.farneback_workspace_bytes(2, T_, h, w), dtype=torch.uint8, device=dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    ev[0].record()
    ops.metrics_frames_in(tc, pc, L.PSNR_Y, gray)
    ev[1].record()
    flow = ops.farneback(gray.view(2 * T_, h, w), 2, params, work)
    ev[2].record()
    ops.flow_epe_sum(flow[:T_ - 1], flow[T_ - 1:])
    ev[3].record()
    torch.cuda.synchronize()
    return {'frames_in': ev[0].elapsed_time(ev[1]), 'farneback': ev[1].elapsed_time(ev[2]),
            'epe': ev[2].elapsed_time(ev[3])}


def reference_rate(true, pred, frames):
    import cv2
    from oracle import metrics_oracle as MO
    t0 = time.perf_counter()
    for i in range(1, frames + 1):
        MO.psnr(true[i], pred[i], 'y')
        g = [cv2.cvtColor(x, cv2.COLOR_RGB2GRAY) for x in (true[i - 1], true[i], pred[i - 1], pred[i])]
        a = cv2.calcOpticalFlowFarneback(g[0], g[1], None, 0.5, 3, 15, 3, 5, 1.2, 0)
        b = cv2.calcOpticalFlowFarneback(g[2], g[3], None, 0.5, 3, 15, 3, 5, 1.2, 0)
        np.mean(np.sqrt(np.sum((a - b) ** 2, axis=-1)))
    return frames / (time.perf_counter() - t0), cv2.getNumThreads()


def official_kernel_times(true, pred, cutfr=2, reps=5):
    """CUDA-event times (ms, median of reps) of the kernels of one official_sequence_metrics pass over the T - 2 cutfr
    scored frames of a sequence, and the algorithmic bytes of the Y statistics and SSIM kernels"""
    dev = torch.device('cuda:0')
    tc = torch.from_numpy(true[cutfr:len(true) - cutfr]).to(dev)
    pc = torch.from_numpy(pred[cutfr:len(pred) - cutfr]).to(dev)
    n, h, w = tc.shape[:3]
    (y0, hc), (x0, wc) = M.crop_8x8(h), M.crop_8x8(w)
    win = (y0, x0, hc, wc)
    gray = torch.empty(2, n, h, w, dtype=torch.uint8, device=dev)
    params = ops.farneback_params(0.5, 3, 15, 3, 5, 1.2, 0)
    work = torch.empty(ops.farneback_workspace_bytes(2, n, h, w), dtype=torch.uint8, device=dev)
    times = {k: [] for k in ('stats', 'ssim', 'gray', 'farneback', 'epe')}
    for _ in range(reps + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
        ev[0].record()
        stats = ops.official_frames_stats(tc, pc, win)
        ev[1].record()
        ops.ssim_y(tc, pc, win, stats)
        ev[2].record()
        ops.metrics_frames_in(tc, pc, L.PSNR_NONE, gray)
        ev[3].record()
        flow = ops.farneback(gray.view(2 * n, h, w), 2, params, work)
        ev[4].record()
        ops.flow_epe_sum(flow[:n - 1], flow[n - 1:], win)
        ev[5].record()
        torch.cuda.synchronize()
        for i, k in enumerate(times):
            times[k].append(ev[i].elapsed_time(ev[i + 1]))
    ms = {k: float(np.median(v[1:])) for k, v in times.items()}     # the first pass is a warm-up
    # each kernel reads the window of both uint8 RGB frames once; the outputs are a few doubles per frame
    moved = {'stats': n * 2 * hc * wc * 3 + n * 24, 'ssim': n * 2 * hc * wc * 3 + n * 32}
    return ms, moved, [n, h, w], win


def official_host_rate(true, pred, frames):
    import cv2
    from oracle import official_metrics as OM
    t0 = time.perf_counter()
    OM.sequence_metrics(true[:frames + 1], pred[:frames + 1], cutfr=0)
    return (frames + 1) / (time.perf_counter() - t0), cv2.getNumThreads(), os.cpu_count()


def main_official(a):
    seqs = [sequence(s) for s in range(a.seqs)]
    T_, h, w = seqs[0][0].shape[:3]
    M.official_sequence_metrics(*seqs[0])
    torch.cuda.synchronize()
    rates = []
    for _ in range(3):
        t0 = time.perf_counter()
        for t, p in seqs:
            M.official_sequence_metrics(t, p)
        torch.cuda.synchronize()
        rates.append(len(seqs) * (T_ - 4) / (time.perf_counter() - t0))
    ms, moved, shape, win = official_kernel_times(*seqs[0])
    total = sum(ms.values())
    host = official_host_rate(*seqs[0], a.ref_frames) if a.ref_frames else (None, None, None)
    res = {
        'card': card(),
        'shape': [T_, h, w], 'scored_frames_per_sequence': T_ - 4, 'window': win,
        'scored_frames_per_s_host_to_host': rates,
        'kernel_ms_per_sequence': ms,
        'farneback_share_of_kernel_time': (ms['gray'] + ms['farneback'] + ms['epe']) / total,
        'algorithmic_bytes_per_sequence': moved,
        'TBps': {k: moved[k] / (ms[k] * 1e-3) / 1e12 for k in moved},
        'oracle_host_frames_per_s': host[0], 'oracle_cv2_threads': host[1], 'host_cpus': host[2],
    }
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


def lpips_flops(h, w):
    """(reference-convention, executed) FLOP of one h x w picture's five AlexNet convs: 2 x MACs of the direct convs,
    and 2 x the MACs the device runs on its padded layouts (full grids; conv1 skips its k-steps past 48 channels)"""
    sz = M.lpips_sizes(h, w)
    (g1, i1), (g2, i2), (m3, _) = sz[0], sz[1], sz[2]
    px1, px2, px3 = i1[2] * i1[3], i2[2] * i2[3], m3[0] * m3[1]
    ref = 2 * (px1 * 64 * 3 * 121 + px2 * 192 * 64 * 25 + px3 * 9 * (384 * 192 + 256 * 384 + 256 * 256))
    exe = 2 * 9 * (g1[0] * g1[1] * 48 * 64 + g2[0] * g2[1] * 192 * 256 + px3 * (384 * 192 + 256 * 384 + 256 * 256))
    return ref, exe


def reference_pnetlin(params):
    """the reference's PNetLin (codes/metrics/LPIPS of oracle/_ref, unmodified) with the seeded weights, on cuda:0"""
    from oracle.gen_lpips_golden import install_stubs
    codes = os.path.join(ROOT, 'oracle', '_ref', 'codes')
    if not os.path.isdir(os.path.join(codes, 'metrics', 'LPIPS')):
        return None
    install_stubs(codes)
    from metrics.LPIPS.models import networks_basic as nb
    net = nb.PNetLin(pnet_rand=True, pnet_tune=False, pnet_type='alex', use_dropout=True, spatial=False,
                     version='0.1', lpips=True)
    sd = {}
    for l, fi in enumerate(M._ALEX_CONVS):
        for k in ('weight', 'bias'):
            sd[f'net.slice{l + 1}.{fi}.{k}'] = torch.from_numpy(params[f'features.{fi}.{k}'])
        sd[f'lin{l}.model.1.weight'] = torch.from_numpy(params[f'lin{l}.model.1.weight'])
    net.load_state_dict(sd, strict=False)
    return net.cuda().eval()


def main_lpips(a):
    params = synthetic.make_lpips_params(7)
    lp = M.LPIPS(params, torch.device('cuda', 0))
    seqs = [sequence(s) for s in range(a.seqs)]
    T_, h, w = seqs[0][0].shape[:3]
    keys = ('PSNR', 'SSIM', 'LPIPS', 'tOF', 'tLP100')
    M.official_sequence_metrics(*seqs[0], keys=keys, lpips=lp)
    torch.cuda.synchronize()
    rates = []
    for _ in range(3):
        t0 = time.perf_counter()
        for t, p in seqs:
            M.official_sequence_metrics(t, p, keys=keys, lpips=lp)
        torch.cuda.synchronize()
        rates.append(len(seqs) * (T_ - 4) / (time.perf_counter() - t0))
    # one LPIPS pass over the scored frames of a sequence (true and pred), kernel by kernel
    (y0, hc), (x0, wc) = M.crop_8x8(h), M.crop_8x8(w)
    t, p = seqs[0]
    frames = torch.from_numpy(np.concatenate([t[2:T_ - 2, y0:y0 + hc, x0:x0 + wc],
                                              p[2:T_ - 2, y0:y0 + hc, x0:x0 + wc]])).cuda().contiguous()
    n, m = frames.shape[0], frames.shape[0] // 2
    sz = M.lpips_sizes(hc, wc)
    pairs = torch.tensor([(i, m + i) for i in range(m)] + [(i - 1, i) for i in range(1, m)] +
                         [(m + i - 1, m + i) for i in range(1, m)], dtype=torch.int32).cuda()
    out = torch.empty(pairs.shape[0], dtype=torch.float64, device='cuda')
    x = torch.empty(n, *sz[0][0], 64, dtype=torch.float16, device='cuda')
    steps = {}

    def run():
        def ev(name, fn):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = fn()
            e1.record()
            steps.setdefault(name, []).append((e0, e1))
            return r
        ev('frames_in', lambda: ops.lpips_frames_in(frames, (0, 0, hc, wc), L.LPIPS_NORM_OFFICIAL, x))
        f1 = ev('conv1', lambda: lp.convs[0](x))
        q1 = ev('pool1', lambda: ops.maxpool3x3s2(f1, sz[0][1], True))
        f2 = ev('conv2', lambda: lp.convs[1](q1))
        q2 = ev('pool2', lambda: ops.maxpool3x3s2(f2, sz[1][1], False))
        f3 = ev('conv3', lambda: lp.convs[2](q2))
        f4 = ev('conv4', lambda: lp.convs[3](f3))
        f5 = ev('conv5', lambda: lp.convs[4](f4))
        ev('heads', lambda: [ops.lpips_head(f, sz[l][1], pairs, lp.heads[l], out, l > 0)
                             for l, f in enumerate((f1, f2, f3, f4, f5))])
    for _ in range(3):
        run()
    steps.clear()
    for _ in range(10):
        run()
    torch.cuda.synchronize()
    ms = {k: float(np.median([e0.elapsed_time(e1) for e0, e1 in v])) for k, v in steps.items()}
    conv_ms = sum(ms[f'conv{i}'] for i in range(1, 6))
    ref_f, exe_f = lpips_flops(hc, wc)
    res = {'card': card(), 'shape': [T_, h, w], 'crop': [hc, wc], 'keys': list(keys),
           'scored_frames_per_sequence': T_ - 4,
           'scored_frames_per_s_host_to_host': rates,
           'lpips_pass_images': n, 'lpips_pass_pairs': int(pairs.shape[0]),
           'kernel_ms_per_pass': ms, 'conv_ms_per_pass': conv_ms,
           'gflop_per_image_reference_counter': ref_f / 1e9, 'gflop_per_image_executed': exe_f / 1e9,
           'conv_tflops_reference_counter': n * ref_f / (conv_ms * 1e-3) / 1e12,
           'conv_tflops_executed': n * exe_f / (conv_ms * 1e-3) / 1e12, 'peak_fp16_dense_tflops': 989}
    net = reference_pnetlin(params)
    if net is not None:
        scale = torch.float32
        a0 = (frames[:m].permute(0, 3, 1, 2).to(scale) / 127.5 - 1)
        a1 = (frames[m:].permute(0, 3, 1, 2).to(scale) / 127.5 - 1)
        with torch.no_grad():
            for _ in range(2):
                net.forward(a0, a1)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5):
                d_ref = net.forward(a0, a1)
            e1.record()
            torch.cuda.synchronize()
            ref_ms = e0.elapsed_time(e1) / 5
            # the same pairs through the device kernels, against float64
            mine = lp.distances(frames, (0, 0, hc, wc), L.LPIPS_NORM_OFFICIAL, [(i, m + i) for i in range(m)])
        from oracle import lpips as O
        # float64 reference of all m pairs (on the GPU: cuDNN's float64 convs), 4 pairs at a time
        fr = frames.cpu().numpy()
        want = np.concatenate([O.lpips(params, fr[i:min(i + 4, m)], fr[m + i:m + min(i + 4, m)], 'official', 'cuda')
                               for i in range(0, m, 4)])

        def errs(d):
            r = np.abs(np.asarray(d, np.float64) - want) / want
            return {'max': float(r.max()), 'median': float(np.median(r))}
        res['reference_pnetlin'] = {
            'tf32_matmul': torch.backends.cuda.matmul.allow_tf32, 'tf32_cudnn': torch.backends.cudnn.allow_tf32,
            'ms_per_pass_of_pairs': ref_ms, 'pairs': m,
            'rel_err_vs_float64_all_pairs': errs(d_ref.flatten().double().cpu().numpy()),
        }
        res['device_rel_err_vs_float64_all_pairs'] = errs(mine.cpu().numpy())
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seqs', type=int, default=4)
    ap.add_argument('--ref-frames', type=int, default=4)
    ap.add_argument('--official', action='store_true', help='measure official_sequence_metrics')
    ap.add_argument('--lpips', action='store_true', help='measure official_sequence_metrics with all five keys')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'metrics_bench needs a GPU'
    if a.lpips:
        return main_lpips(a)
    if a.official:
        return main_official(a)
    seqs = [sequence(s) for s in range(a.seqs)]
    T_, h, w = seqs[0][0].shape[:3]
    M.sequence_metrics(*seqs[0])               # warm-up: module load, allocations
    torch.cuda.synchronize()
    rates = []
    for _ in range(2):
        t0 = time.perf_counter()
        for t, p in seqs:
            M.sequence_metrics(t, p, psnr='y', tof=True)
        torch.cuda.synchronize()
        rates.append(len(seqs) * T_ / (time.perf_counter() - t0))
    timed_phases(*seqs[0])
    ph = [timed_phases(*seqs[i % len(seqs)]) for i in range(3)]
    phases = {k: float(np.median([x[k] for x in ph])) for k in ph[0]}
    pb = phase_bytes(T_, h, w)
    moved = {'frames_in': pb['frames_in'], 'farneback': pb['pyramid+poly'] + pb['flow'], 'epe': pb['epe']}
    ref_rate, ref_threads = reference_rate(*seqs[0], a.ref_frames) if a.ref_frames else (None, None)
    res = {
        'card': card(),
        'shape': [T_, h, w],
        'scored_frames_per_s_host_to_host': rates,
        'phase_ms_per_sequence': phases,
        'phase_bytes_per_sequence': moved,
        'phase_share_of_3.35TBps': {k: moved[k] / (phases[k] * 1e-3) / HBM for k in phases},
        'reference_host_frames_per_s': ref_rate,
        'reference_cv2_threads': ref_threads,
    }
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
