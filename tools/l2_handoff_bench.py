#!/usr/bin/env python
"""How much of each layer's input the step's launches read from L2: the launches that hand a map to the next one,
timed in sequence with every conv walking its tiles forward and with the walk directions the networks assign, and
each kernel timed cold.

    python tools/l2_handoff_bench.py [--n 4] [--h 134] [--w 320] [--reps 20] [--out-dir DIR]

Sequences (bd4 step shapes, n LR frames of h x w, random weights), each captured `--reps` times in one CUDA graph
with programmatic dependent launch on, as in the step; the graph is replayed 3 times untimed and then timed over 5
replays with CUDA events:
  - `srnet`: conv_in, the 10 residual blocks (plain conv, residual conv) and the first transposed conv, 22 launches;
  - `tail`: upsample of the LR frame, the fused SRNet tail accumulating onto it, uint8 output (to_uint8_c3x4), 3 launches;
  - `fnet_front`: pack_pair, encoder1[0], encoder1[2] + pool, 3 launches;
  - `fnet_back`: upsample2x of the h/2 map, flow[0], flow[2], 3 launches.
`forward` sets PackedConv.reverse = False on every conv; `alternate` sets it as networks.SRNet.run_nhwc and
networks.FNet do.  The elementwise kernels' walks are fixed in the kernels, so both arms run the same ones.
`cold`: each launch alone, captured `--reps` times over rotating input / output buffers larger than the 50 MB L2.
Prints a table and one JSON line (also written to DIR/l2_handoff_bench.json with --out-dir)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

L2_BYTES = 50 << 20


def card():
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm',
                              '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout
        name, power, clk = [x.strip() for x in out.strip().split(',')]
        return {'name': name, 'power_limit': power, 'sm_max_clock': clk}
    except Exception:
        import torch
        return {'name': torch.cuda.get_device_name(0), 'power_limit': None, 'sm_max_clock': None}


def time_graph(fn, reps, torch, replays=5):
    """Seconds per call of fn(i), i = 0 .. reps-1, captured in one CUDA graph."""
    fn(0)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(reps):
            fn(i)
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / (reps * replays)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=4)
    ap.add_argument('--h', type=int, default=134)
    ap.add_argument('--w', type=int, default=320)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--out-dir', default=None)
    args = ap.parse_args()
    import torch
    import tecogan_b200  # noqa: F401  (registers the package modules)
    ops = sys.modules['tecogan-pytorch_b200.ops']
    L = sys.modules['tecogan-pytorch_b200.lib']
    assert torch.cuda.is_available(), 'l2_handoff_bench needs a GPU'
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    n, h, w, s = args.n, args.h, args.w, 4

    def conv(cin, cout, act, kind=L.CONV_3X3, epilogue=L.EPI_NHWC_F16):
        shape = (cout, cin, 3, 3) if kind == L.CONV_3X3 else (cin, cout, 3, 3)
        wt = torch.randn(shape, device=dev) * (1.0 / (9 * cin) ** 0.5)
        return ops.PackedConv(wt, torch.randn(cout, device=dev) * 0.05, kind, act, epilogue)

    def act16(*shape):
        return (torch.randn(*shape, device=dev) * 0.5).half()

    # ---- SRNet body + first transposed conv
    body = [conv(64, 64, L.ACT_RELU)]
    for _ in range(10):
        body += [conv(64, 64, L.ACT_RELU), conv(64, 64, L.ACT_NONE)]
    up0 = conv(64, 64, L.ACT_RELU, L.CONVT_3X3_S2)
    x_sr = act16(n, h, w, 64)
    a_bufs = [torch.empty(n, h, w, 64, device=dev, dtype=torch.float16) for _ in range(2)]
    t_buf = torch.empty(n, h, w, 64, device=dev, dtype=torch.float16)
    up_out = torch.empty(n, 2 * h, 2 * w, 64, device=dev, dtype=torch.float16)

    def srnet(_):
        a = body[0](x_sr, y=a_bufs[0])
        for i in range(10):
            t = body[1 + 2 * i](a, y=t_buf)
            a = body[2 + 2 * i](t, y=a_bufs[(i + 1) % 2], residual=a)
        up0(a, y=up_out)

    # ---- fused tail + uint8
    up1 = conv(64, 64, L.ACT_RELU, L.CONVT_3X3_S2)
    outc = conv(64, 3, L.ACT_NONE, epilogue=L.EPI_OUT_NCHW_F32)
    lr = torch.rand(n, 3, h, w, device=dev)
    hr = torch.empty(n, 3, s * h, s * w, device=dev)
    hr_u8 = torch.empty(n, s * h, s * w, 3, device=dev, dtype=torch.uint8)
    tail_in = act16(n, 2 * h, 2 * w, 64)

    def tail(_):
        ops.upsample(lr, s, L.UP_BICUBIC, y=hr)
        ops.fused_tail(up1, outc, tail_in, None, s, L.UP_BICUBIC, y=hr, accumulate=True)
        ops.float_to_uint8_nhwc(hr, hr_u8)

    # ---- FNet full-resolution front and back
    e10, e12 = conv(6, 32, L.ACT_LRELU02), conv(32, 32, L.ACT_LRELU02)
    f0, f2 = conv(64, 32, L.ACT_LRELU02), conv(32, 2, L.ACT_NONE, epilogue=L.EPI_FLOW_NCHW_F32)
    x1, x2 = torch.rand(n, 3, h, w, device=dev), torch.rand(n, 3, h, w, device=dev)
    pair = torch.empty(n, h, w, 64, device=dev, dtype=torch.float16)
    e1a = torch.empty(n, h, w, 64, device=dev, dtype=torch.float16)
    e1p = torch.empty(n, h // 2, w // 2, 64, device=dev, dtype=torch.float16)
    half = act16(n, h // 2, w // 2, 64)
    u3 = torch.empty(n, 2 * (h // 2), 2 * (w // 2), 64, device=dev, dtype=torch.float16)
    f0o = torch.empty(n, 2 * (h // 2), 2 * (w // 2), 64, device=dev, dtype=torch.float16)
    flow = torch.empty(n, 2, 2 * (h // 2), 2 * (w // 2), device=dev)

    def fnet_front(_):
        ops.pack_pair(x1, x2, y=pair)
        e10(pair, y=e1a)
        e12(e1a, y=e1p, pool=True)

    def fnet_back(_):
        ops.upsample2x(half, y=u3)
        f0(u3, y=f0o)
        f2(f0o, y=flow)

    # the directions networks.py assigns: SRNet conv_in reversed, then alternating; FNet convs alternate, forward first
    chains = {'srnet': body + [up0], 'fnet_front': [e10, e12], 'fnet_back': [f0, f2]}
    first_reversed = {'srnet': True, 'fnet_front': False, 'fnet_back': False}
    seqs = [('srnet', srnet, 22), ('tail', tail, 3), ('fnet_front', fnet_front, 3), ('fnet_back', fnet_back, 3)]
    res = {'card': card(), 'n': n, 'h': h, 'w': w, 'reps': args.reps, 'sequences': {}, 'cold_us': {}}
    print(f'card: {res["card"]}')
    print(f'{"sequence":12s} {"launches":>8s} {"forward us":>11s} {"alternate us":>13s} {"us/launch fwd":>14s} '
          f'{"us/launch alt":>14s}')
    for name, fn, nl in seqs:
        t = {}
        for arm in ('forward', 'alternate'):
            for i, pc in enumerate(chains.get(name, [])):
                pc.reverse = arm == 'alternate' and (i % 2 == 0) == first_reversed[name]
            t[arm] = time_graph(fn, args.reps, torch) * 1e6
        for pc in chains.get(name, []):
            pc.reverse = False
        res['sequences'][name] = {'launches': nl, 'forward_us': t['forward'], 'alternate_us': t['alternate']}
        print(f'{name:12s} {nl:8d} {t["forward"]:11.1f} {t["alternate"]:13.1f} {t["forward"] / nl:14.2f} '
              f'{t["alternate"] / nl:14.2f}')

    # ---- cold: each launch alone over rotating buffers larger than L2
    def cold(name, make_io, run):
        io0 = make_io()
        nbytes = sum(x.numel() * x.element_size() for x in io0)
        nbuf = max(3, -(-2 * L2_BYTES // nbytes) + 1)
        ios = [io0] + [make_io() for _ in range(nbuf - 1)]
        us = time_graph(lambda i: run(*ios[i % nbuf]), max(args.reps, 2 * nbuf), torch) * 1e6
        res['cold_us'][name] = us
        print(f'cold {name:28s} {us:8.2f} us  ({nbytes / 1e6:.1f} MB per launch, {nbuf} buffer sets)')
        del ios

    m64 = (n, h, w, 64)
    cold('body plain conv', lambda: [act16(*m64), torch.empty(m64, device=dev, dtype=torch.float16)],
         lambda x, y: body[1](x, y=y))
    cold('body residual conv', lambda: [act16(*m64), act16(*m64), torch.empty(m64, device=dev, dtype=torch.float16)],
         lambda x, r, y: body[2](x, y=y, residual=r))
    cold('first transposed conv', lambda: [act16(*m64), torch.empty(n, 2 * h, 2 * w, 64, device=dev,
                                                                    dtype=torch.float16)],
         lambda x, y: up0(x, y=y))
    cold('to_uint8_c3x4', lambda: [torch.rand(n, 3, s * h, s * w, device=dev),
                                   torch.empty(n, s * h, s * w, 3, device=dev, dtype=torch.uint8)],
         lambda x, y: ops.float_to_uint8_nhwc(x, y))
    cold('pack_pair', lambda: [torch.rand(n, 3, h, w, device=dev), torch.rand(n, 3, h, w, device=dev),
                               torch.empty(m64, device=dev, dtype=torch.float16)],
         lambda a, b, y: ops.pack_pair(a, b, y=y))
    cold('encoder1[0]', lambda: [act16(*m64), torch.empty(m64, device=dev, dtype=torch.float16)],
         lambda x, y: e10(x, y=y))
    cold('encoder1[2] + pool', lambda: [act16(*m64), torch.empty(n, h // 2, w // 2, 64, device=dev,
                                                                 dtype=torch.float16)],
         lambda x, y: e12(x, y=y, pool=True))
    cold('upsample2x', lambda: [act16(n, h // 2, w // 2, 64), torch.empty_like(u3)],
         lambda x, y: ops.upsample2x(x, y=y))
    cold('flow[0]', lambda: [act16(*u3.shape), torch.empty_like(f0o)], lambda x, y: f0(x, y=y))
    cold('flow[2]', lambda: [act16(*u3.shape), torch.empty_like(flow)], lambda x, y: f2(x, y=y))
    line = json.dumps(res)
    print(line)
    if args.out_dir:
        os.makedirs(args.out_dir, exist_ok=True)
        with open(os.path.join(args.out_dir, 'l2_handoff_bench.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
