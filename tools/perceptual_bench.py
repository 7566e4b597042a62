#!/usr/bin/env python
"""The VGG19 perceptual loss of TecoGAN training, the reference's VGGFeatureExtractor (PyTorch, fp32) against
tecogan_b200.VGGFeatureExtractor, on the training shape.

    python tools/perceptual_bench.py [--batch 32] [--frames 19] [--size 256] [--steps 3] [--warmup 1]
                                     [--no-train-step] [--train-batch 32] [--out-dir DIR]

Per extractor, on --batch clips x --frames frames of --size x --size (608 images of 256 x 256 by default: bench.py's
TecoGAN training batch, the 19-frame ping-pong sequence of HR crops):
  - `vgg_ms`: one hr pass under autograd, one gt pass without it, the four CosineSimilarityLoss terms of
    vsrgan_model.py:229-238 and the backward of the hr pass to its input, CUDA events around --steps repetitions
    after --warmup; the peak memory of those repetitions;
  - per conv layer, forward (conv + ReLU) and, for the layers the backward runs, the input gradient (dgrad + ReLU'),
    each timed alone with CUDA events, as TFLOP/s by 2 * 9 * cin * cout per output pixel (cin = 3 for conv1_1), and
    as a share of the H100 SXM data sheet's 989 dense fp16 TFLOP/s (the reference runs in fp32 with PyTorch's default
    TF32 settings, stated in the output; its share is against the same 989);
  - `train_step_ms`: one full VSRGANModel.train() iteration (bench.py's training setup: --train-batch clips of 10-frame
    3x64x64 LR crops, the library's generator) with each net_F, and its peak memory.
An arm that runs out of device memory reports the error in place of its numbers.
The card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line (also written to
DIR/perceptual_bench.json with --out-dir).  Needs a CUDA device and the reference install (oracle/_ref)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PEAK_TFLOPS = 989.0


def card():
    out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm',
                          '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout
    name, power, clk = [x.strip() for x in out.strip().split(',')]
    return {'name': name, 'power_limit': power, 'sm_max_clock': clk}


def cuda_ms(torch, fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def vgg_step(torch, F, net_F, hr, gt):
    """the feature loss of vsrgan_model.py:229-238 and the input gradient of the hr pass"""
    x = hr.detach().requires_grad_(True)
    hr_feats = net_F(x)
    with torch.no_grad():
        gt_feats = net_F(gt)
    loss = 0
    for a, b in zip(hr_feats, gt_feats):
        loss = loss + (1.0 - F.cosine_similarity(a, b.detach(), dim=1, eps=1e-8).mean())
    g, = torch.autograd.grad(loss, [x])
    return loss.detach(), g


def layer_rates(torch, F, T, ours, ref, n, size, steps):
    """per conv layer: ms and TFLOP/s of the forward and of the input gradient, ours and the reference"""
    ops, L = T.ops, sys.modules['tecogan-pytorch_b200.lib']
    dev = ours.mean.device
    layers = ours.packed_layers()
    rows, h = [], size
    for u, ((fwd, dg), (ci, _, pool)) in enumerate(zip(layers, ours._units)):
        conv = ref.features[ci]
        cin, cout = conv.in_channels, conv.out_channels
        gflop = 2 * 9 * cin * cout * n * h * h * 1e-9
        row = {'layer': f'features.{ci}', 'cin': cin, 'cout': cout, 'hw': h, 'gflop': round(gflop, 1)}
        x16 = torch.randn(n, h, h, fwd.cin, device=dev).half()
        if fwd.cin_real < fwd.cin:
            x16[..., fwd.cin_real:] = 0
        y16 = torch.empty(n, h, h, fwd.cout, device=dev, dtype=torch.float16)
        row['ours_fwd_ms'] = cuda_ms(torch, lambda: fwd(x16, y=y16), steps, 1)
        if u > 0:
            dz = torch.randn(n, h, h, fwd.cout, device=dev).half()
            gx = torch.empty(n, h, h, fwd.cin, device=dev, dtype=torch.float16)
            m = torch.randn(n, h, h, fwd.cin, device=dev).half()
            row['ours_dgrad_ms'] = cuda_ms(torch, lambda: dg(dz, y=gx, mask=m, mask_act=L.ACT_RELU), steps, 1)
            del dz, gx, m
        del x16, y16
        x32 = torch.randn(n, cin, h, h, device=dev)
        row['ref_fwd_ms'] = cuda_ms(torch, lambda: F.relu(conv(x32), inplace=True), steps, 1)
        if u > 0:
            xg = x32.requires_grad_(True)
            y = conv(xg)
            gy = torch.randn_like(y)
            row['ref_dgrad_ms'] = cuda_ms(torch, lambda: torch.autograd.grad(y, [xg], gy, retain_graph=True), steps, 1)
            del y, gy, xg
        del x32
        torch.cuda.empty_cache()
        for k in ('ours_fwd', 'ours_dgrad', 'ref_fwd', 'ref_dgrad'):
            if k + '_ms' in row:
                tf = gflop / row[k + '_ms']               # GFLOP / ms = TFLOP/s
                row[k + '_tflops'] = round(tf, 1)
                row[k + '_of_peak'] = round(tf / PEAK_TFLOPS, 3)
                row[k + '_ms'] = round(row[k + '_ms'], 3)
        rows.append(row)
        if pool:
            h //= 2
    return rows


def train_step(torch, T, bench, refimport, net_f, batch, steps, warmup):
    """ms and peak GB of one VSRGANModel.train() iteration with bench.py's training setup, net_f 'ours' or 'ref'"""
    dev = torch.device('cuda', 0)
    m = bench._train_model('tecogan', dev, 'ours', False, 0, 1)
    if net_f == 'ours':
        donor = m.net_F.state_dict()
        m.net_F = T.VGGFeatureExtractor(m.opt['train']['feature_crit']['feature_layers']).to(dev)
        m.net_F.load_state_dict(donor)
    g = torch.Generator().manual_seed(100)
    data = torch.rand(batch, bench.TRAIN['t'], 3, 264, 264, generator=g).to(dev)

    def step():
        m.prepare_training_data({'gt': data})
        m.train()
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ms = cuda_ms(torch, step, steps, 0)
    out = {'train_step_ms': round(ms, 1), 'train_peak_gb': round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
           'l_feat_G': m.log_dict.get('l_feat_G')}
    del m, data
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--batch', type=int, default=32, help='clips')
    ap.add_argument('--frames', type=int, default=19, help='frames per clip (19: the ping-pong sequence)')
    ap.add_argument('--size', type=int, default=256, help='HR crop side')
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--no-train-step', action='store_true', help='skip the full VSRGANModel.train() timing')
    ap.add_argument('--train-batch', type=int, default=32, help='clips of the full training step (bench.py: 32)')
    ap.add_argument('--out-dir', default=None)
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    import tecogan_b200 as T
    import refimport
    import bench
    if not torch.cuda.is_available():
        raise SystemExit('perceptual_bench: needs a CUDA device')
    dev = torch.device('cuda', 0)
    refimport.stub_pretrained_vgg19()
    refimport._prepare()
    from models.networks.vgg_nets import VGGFeatureExtractor as RefVGG
    ref = RefVGG().to(dev)
    ours = T.VGGFeatureExtractor().to(dev)
    ours.load_state_dict(ref.state_dict())
    n = args.batch * args.frames
    g = torch.Generator().manual_seed(0)
    gt = torch.rand(n, 3, args.size, args.size, generator=g)
    hr = (gt + 0.05 * torch.randn(gt.shape, generator=g)).clamp(0, 1)
    gt, hr = gt.to(dev), hr.to(dev)

    res = {'card': card(), 'shape': f'{n} images (batch {args.batch} x {args.frames} frames) of 3x{args.size}x{args.size}',
           'reference_precision': f'fp32; torch.backends.cuda.matmul.allow_tf32={torch.backends.cuda.matmul.allow_tf32}, '
                                  f'torch.backends.cudnn.allow_tf32={torch.backends.cudnn.allow_tf32} (PyTorch defaults), '
                                  f'cudnn.benchmark={torch.backends.cudnn.benchmark}',
           'peak_tflops_datasheet': PEAK_TFLOPS}
    out = {}
    for name, net in (('ours', ours), ('reference', ref)):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        try:
            ms = cuda_ms(torch, lambda: vgg_step(torch, F, net, hr, gt), args.steps, args.warmup)
            loss, grad = vgg_step(torch, F, net, hr, gt)
        except torch.cuda.OutOfMemoryError as e:         # a shape one of the two cannot hold on this card
            res[name] = {'vgg_ms': None, 'error': f'out of memory: {str(e).splitlines()[0]}'}
            continue
        out[name] = (loss.double().cpu(), grad.double().cpu())
        res[name] = {'vgg_ms': round(ms, 1), 'vgg_peak_gb_above_inputs': round(
            (torch.cuda.max_memory_allocated() - base) / 2 ** 30, 2), 'loss': float(loss)}
        del loss, grad
    if len(out) == 2:
        fl, gl = out['ours'], out['reference']
        res['loss_rel_diff'] = float(abs(fl[0] - gl[0]) / abs(gl[0]))
        res['grad_rel_l2'] = float((fl[1] - gl[1]).norm() / gl[1].norm())
        res['vgg_speedup'] = round(res['reference']['vgg_ms'] / res['ours']['vgg_ms'], 2)
    out = None
    torch.cuda.empty_cache()
    res['layers'] = layer_rates(torch, F, T, ours, ref, n, args.size, args.steps)
    del hr, gt, ref, ours
    torch.cuda.empty_cache()
    if not args.no_train_step:
        for name in ('ours', 'ref'):
            key = 'reference' if name == 'ref' else 'ours'
            try:
                res[key].update(train_step(torch, T, bench, refimport, name, args.train_batch, args.steps, args.warmup))
            except torch.cuda.OutOfMemoryError as e:
                res[key]['train_step_error'] = f'out of memory: {str(e).splitlines()[0]}'
            torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out_dir:
        os.makedirs(args.out_dir, exist_ok=True)
        with open(os.path.join(args.out_dir, 'perceptual_bench.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
