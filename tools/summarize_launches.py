#!/usr/bin/env python
"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch list into per-kernel totals
for the LAST complete step found in the file (a step = the launches between two pack_pair
kernels, i.e. one FRNet.step + uint8 conversion).

    python tools/summarize_launches.py launches.csv > launches.md
"""
import csv
import sys
from collections import OrderedDict


def main(path):
    rows = []
    with open(path, newline='') as f:
        lines = [l for l in f if not l.startswith('==')]
    rd = csv.DictReader(lines)
    for r in rd:
        if r.get('Metric Name') != 'gpu__time_duration.sum':
            continue
        val = float(r['Metric Value'].replace(',', ''))
        unit = r.get('Metric Unit', 'ns')
        scale = {'ns': 1e-3, 'us': 1.0, 'usecond': 1.0, 'nsecond': 1e-3, 'ms': 1e3, 'msecond': 1e3}.get(unit, 1e-3)
        name = r['Kernel Name'].split('(')[0]
        rows.append((int(r['ID']), name, val * scale, r.get('Grid Size', ''), r.get('Block Size', '')))
    starts = [i for i, r in enumerate(rows) if 'pack_pair' in r[1]]
    if len(starts) >= 2:
        seg = rows[starts[-2]:starts[-1]]
    else:
        seg = rows
    tot = sum(r[2] for r in seg)
    print(f'# launch list summary: {path}\n')
    print(f'launches captured: {len(rows)}; last complete step: {len(seg)} launches, '
          f'{tot:.1f} us summed kernel time (ncu, cold cache, serialised -- compare SHARES)\n')
    agg = OrderedDict()
    for _, name, us, grid, blk in seg:
        a = agg.setdefault(name, [0, 0.0])
        a[0] += 1
        a[1] += us
    print('| kernel | launches | total us | share |\n|---|---:|---:|---:|')
    for name, (cnt, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f'| {name} | {cnt} | {us:.1f} | {100 * us / tot:.1f}% |')
    print('\n## launches of the step, in order\n')
    print('| # | kernel | grid | us |\n|---:|---|---|---:|')
    for i, (_, name, us, grid, blk) in enumerate(seg):
        print(f'| {i} | {name} | {grid} | {us:.1f} |')


if __name__ == '__main__':
    main(sys.argv[1])
