"""Device time of the FNet convs with 128 / 256 input channels, each layer shape alone, tap kernel
(a_mode=TAP) against the default path (split-K over a thread-block cluster), in one build.

Each measurement captures `--reps` launches over rotating input / output buffers whose total size exceeds
the 50 MB L2 in a CUDA graph, replays it 3 times untimed, then times one replay with CUDA events (the
method of bench.py's kernel timings).  Prints one table row per layer and path, then a JSON line.

    python tools/fnet_conv_bench.py [--n 4] [--reps 60]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# (name, cin, cout, h, w, pooled) of the 4x BD step: the LR frame is 134 x 320, FNet runs on 2 x 67 x 160
LAYERS = [
    ('encoder3[2]+pool', 128, 128, 33, 80, True),
    ('decoder1[0]', 128, 256, 16, 40, False),
    ('decoder1[2]', 256, 256, 16, 40, False),
    ('decoder2[0]', 256, 128, 32, 80, False),
    ('decoder2[2]', 128, 128, 32, 80, False),
    ('decoder3[0]', 128, 64, 64, 160, False),
]


def time_graph(fn, nbuf, reps, torch):
    for i in range(nbuf):
        fn(i)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(reps):
            fn(i % nbuf)
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=4, help='frames per launch (4 = the bd4 step)')
    ap.add_argument('--reps', type=int, default=60)
    args = ap.parse_args()
    import torch
    import tecogan_b200  # noqa: F401  (registers the package modules)
    ops = sys.modules['tecogan-pytorch_b200.ops']
    L = sys.modules['tecogan-pytorch_b200.lib']
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    rows = []
    print(f'{"layer":18s} {"cin->cout":>10s} {"size":>9s} {"GFLOP":>6s} {"tap us":>8s} {"TF/s":>6s} '
          f'{"split-K us":>10s} {"TF/s":>6s} {"speedup":>7s}')
    for name, cin, cout, h, w, pool in LAYERS:
        n = args.n
        wt = torch.randn(cout, cin, 3, 3, device=dev) * (1.5 / (9 * cin) ** 0.5)
        pc = ops.PackedConv(wt, torch.zeros(cout, device=dev), L.CONV_3X3, L.ACT_LRELU02)
        set_mb = n * h * w * (cin + cout) * 2 / 1e6
        nbuf = max(3, int(200 / set_mb) + 1)
        xs = [torch.randn(n, h, w, cin, device=dev).half() for _ in range(nbuf)]
        oshape = (n, h // 2, w // 2, cout) if pool else (n, h, w, cout)
        ys = [torch.empty(oshape, device=dev, dtype=torch.float16) for _ in range(nbuf)]
        gflop = 2.0 * 9 * cin * cout * n * h * w / 1e9
        t = {}
        for path, mode in (('tap', L.AMODE_TAP), ('splitk', L.AMODE_AUTO)):
            t[path] = time_graph(lambda i: pc(xs[i], y=ys[i], a_mode=mode, pool=pool), nbuf, args.reps, torch)
        row = {'layer': name, 'cin': cin, 'cout': cout, 'n': n, 'h': h, 'w': w, 'pool': pool, 'gflop': gflop,
               'tap_us': t['tap'] * 1e6, 'splitk_us': t['splitk'] * 1e6}
        rows.append(row)
        print(f'{name:18s} {f"{cin}->{cout}":>10s} {f"{h}x{w}":>9s} {gflop:6.2f} {row["tap_us"]:8.1f} '
              f'{gflop / t["tap"] / 1e3:6.0f} {row["splitk_us"]:10.1f} {gflop / t["splitk"] / 1e3:6.0f} '
              f'{t["tap"] / t["splitk"]:7.2f}')
        del xs, ys
    tot_tap = sum(r['tap_us'] for r in rows)
    tot_sk = sum(r['splitk_us'] for r in rows)
    print(f'{"total":18s} {"":>10s} {"":>9s} {sum(r["gflop"] for r in rows):6.2f} {tot_tap:8.1f} {"":>6s} '
          f'{tot_sk:10.1f} {"":>6s} {tot_tap / tot_sk:7.2f}')
    print(json.dumps({'device': torch.cuda.get_device_name(0), 'layers': rows,
                      'total_tap_us': tot_tap, 'total_splitk_us': tot_sk}))


if __name__ == '__main__':
    main()
