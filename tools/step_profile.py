#!/usr/bin/env python
"""Per-kernel breakdown of one step of the bench.py workload, measured with torch.profiler.

    python tools/step_profile.py --out-dir DIR [--workload bd4] [--steps 6] [--warmup 5]

Builds the same net, weights (bench.make_params) and clips (bench.synthetic_clips) as bench.py, replays
the step's CUDA graph under torch.profiler with CUDA activities and prints
  - per-kernel totals of one step (mean over the profiled steps): launches, device time, share,
  - the ordered launch list of the last profiled step,
and writes both to DIR/step_profile_<workload>.json together with the card name and power limit.
If the graph-replayed kernels do not show up one by one in the trace, the eager step
(ClipEngine(..., use_graph=False)) is profiled instead and the output says so.  Programmatic dependent
launch is off unless --pdl is given: with it on, a kernel starts while its predecessor drains and its
recorded time includes that wait.  Kernel times under the profiler are device times of the kernels
themselves; the step's wall time is bench.py's business.
"""
import argparse
import json
import os
import subprocess
import sys
from collections import OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402


def card():
    """Name and power limit of GPU 0, read from nvidia-smi (None where it is unavailable)."""
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm',
                              '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout
        name, power, clk = [x.strip() for x in out.strip().split(',')]
        return {'name': name, 'power_limit': power, 'sm_max_clock': clk}
    except Exception:
        import torch
        return {'name': torch.cuda.get_device_name(0), 'power_limit': None, 'sm_max_clock': None}


def short_name(name):
    """Kernel name without namespace and argument list; template arguments are kept."""
    name = name.replace('(anonymous namespace)::', '').replace('void ', '')
    depth = 0
    for i, ch in enumerate(name):
        if ch == '<':
            depth += 1
        elif ch == '>':
            depth -= 1
        elif ch == '(' and depth == 0:
            return name[:i]
    return name


def device_events(prof):
    """(name, start_us, duration_us) of every kernel in the trace, in start order; copies and memsets
    are left out."""
    import torch
    evs = []
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        if e.name.startswith(('Memcpy', 'Memset', 'cudaMemcpy', 'cudaMemset')):
            continue
        evs.append((short_name(e.name), e.time_range.start, e.time_range.elapsed_us()))
    evs.sort(key=lambda t: t[1])
    return evs


def profile(eng, step, n_steps, warmup):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    eng.reset()
    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for i in range(n_steps):
            step(warmup + i)
        torch.cuda.synchronize()
    return device_events(prof)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out-dir', required=True, help='directory the JSON result is written to')
    ap.add_argument('--workload', default='bd4', choices=sorted(bench.WORKLOADS))
    ap.add_argument('--steps', type=int, default=6, help='profiled steps')
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--pdl', action='store_true',
                    help='keep programmatic dependent launch on (then a kernel\'s time includes the part of its '
                         'predecessor it overlaps, and the per-kernel times add up to more than the step)')
    args = ap.parse_args()
    if not args.pdl:
        os.environ['TECOGAN_B200_PDL'] = '0'     # read once, at the library's first launch

    import torch
    import tecogan_b200 as T
    assert torch.cuda.is_available(), 'step_profile.py needs a GPU'
    bench.select_workload(args.workload)
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    net = T.FRNet(3, 3, 64, 10, bench.WL['degradation'], bench.SCALE)
    net.load_state_dict(bench.make_params(), strict=True)
    net = net.to(dev).eval()
    n, (c, h, w) = bench.CLIPS_PER_GPU, bench.LR
    frames = bench.synthetic_clips(n, 8, seed=0).to(dev).transpose(0, 1).contiguous()

    mode = 'graph replay'
    eng = T.ClipEngine(net, n, c, h, w, dev, use_graph=True)
    per_step = eng.launches_per_step

    def step(i):
        p = i & 1
        eng.lr[p].copy_(frames[i % frames.shape[0]])
        eng.run_frame(p)

    evs = profile(eng, step, args.steps, args.warmup)
    if len(evs) < per_step * args.steps:
        mode = ('eager step (ClipEngine use_graph=False): the graph replay showed %d kernels for %d steps of %d '
                'launches' % (len(evs), args.steps, per_step))
        eng.close()
        eng = T.ClipEngine(net, n, c, h, w, dev, use_graph=False)
        evs = profile(eng, step, args.steps, args.warmup)
    # the library's launches plus whatever PyTorch kernels the step contains
    assert len(evs) % args.steps == 0, f'{len(evs)} kernels in {args.steps} steps'
    per_step = len(evs) // args.steps

    steps = [evs[k * per_step:(k + 1) * per_step] for k in range(args.steps)]
    agg = OrderedDict()
    for s in steps:
        for name, _, us in s:
            a = agg.setdefault(name, [0, 0.0])
            a[0] += 1
            a[1] += us
    totals = sorted(((name, cnt / args.steps, us / args.steps) for name, (cnt, us) in agg.items()),
                    key=lambda t: -t[2])
    step_us = sum(t[2] for t in totals)
    last = steps[-1]
    spans = [(s[-1][1] + s[-1][2] - s[0][1]) for s in steps]
    info = card()

    print(f'# step profile: {bench.WL["name"]}')
    print(f'card: {info["name"]}, power limit {info["power_limit"]}, max SM clock {info["sm_max_clock"]}')
    print(f'mode: {mode}, programmatic dependent launch {"on" if args.pdl else "off"}; '
          f'{args.steps} profiled steps of {per_step} kernels')
    print(f'kernel time per step: {step_us:.1f} us summed; first-kernel-start to last-kernel-end '
          f'{sum(spans) / len(spans):.1f} us (under the profiler)\n')
    print('| kernel | launches/step | us/step | share |\n|---|---:|---:|---:|')
    for name, cnt, us in totals:
        print(f'| {name} | {cnt:g} | {us:.1f} | {100 * us / step_us:.1f}% |')
    print('\n## launches of the last profiled step, in order\n')
    print('| # | kernel | us |\n|---:|---|---:|')
    for i, (name, _, us) in enumerate(last):
        print(f'| {i} | {name} | {us:.1f} |')

    os.makedirs(args.out_dir, exist_ok=True)
    out = {'workload': bench.WL['name'], 'card': info, 'mode': mode, 'pdl': args.pdl, 'profiled_steps': args.steps,
           'kernels_per_step': per_step, 'kernel_us_per_step': step_us, 'span_us_per_step': sum(spans) / len(spans),
           'totals': [{'kernel': nm, 'launches': cnt, 'us': us, 'share': us / step_us} for nm, cnt, us in totals],
           'launches': [{'kernel': nm, 'us': us} for nm, _, us in last]}
    path = os.path.join(args.out_dir, f'step_profile_{args.workload}.json')
    with open(path, 'w') as f:
        json.dump(out, f, indent=1)
    print(f'\nwritten: {path}')


if __name__ == '__main__':
    main()
