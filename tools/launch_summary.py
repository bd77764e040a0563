"""Aggregate an `ncu --metrics gpu__time_duration.sum --csv` launch list by kernel (markdown table):
    python tools/launch_summary.py launches.csv [top_n]"""
import collections
import csv
import sys

rows = list(csv.reader(open(sys.argv[1])))
top = int(sys.argv[2]) if len(sys.argv) > 2 else 20
hdr = [i for i, r in enumerate(rows) if r and r[0] == 'ID'][0]
h = rows[hdr]
ki, vi = h.index('Kernel Name'), h.index('Metric Value')
agg = collections.defaultdict(lambda: [0, 0.0])
for r in rows[hdr + 1:]:
    if len(r) <= vi:
        continue
    try:
        v = float(r[vi].replace(',', ''))
    except ValueError:
        continue
    name = r[ki].replace('void ', '').replace('g6d::', '').split('(')[0]
    agg[name][0] += 1
    agg[name][1] += v
tot = sum(v[1] for v in agg.values())
print(f'{sum(v[0] for v in agg.values())} launches, {tot / 1e3:.0f} us of kernel time\n')
print('| kernel | launches | us | share |\n|---|---:|---:|---:|')
for n, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:top]:
    print(f'| `{n}` | {c} | {t / 1e3:.0f} | {100 * t / tot:.1f}% |')
