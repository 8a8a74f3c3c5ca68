"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch list into a per-kernel table of ONE step.
    python tools/launch_summary.py launches.csv [launches_per_step] > summary.md
The list holds warm-up steps too: the LAST `launches_per_step` kernel launches are taken (default: everything
after the last prep_clip launch)."""
import csv
import sys
from collections import OrderedDict


def main():
    path = sys.argv[1]
    rows = []
    with open(path) as f:
        lines = [l for l in f if not l.startswith('==')]
    for r in csv.DictReader(lines):
        if r.get('Metric Name') != 'gpu__time_duration.sum':
            continue
        v = float(r['Metric Value'].replace(',', ''))
        unit = r.get('Metric Unit', 'ns')
        us = v / 1000.0 if unit in ('ns', 'nsecond') else (v if unit in ('us', 'usecond') else v * 1000.0)
        rows.append((r['Kernel Name'], us))
    if len(sys.argv) > 2:
        rows = rows[-int(sys.argv[2]):]
    else:
        marks = [i for i, (k, _) in enumerate(rows) if 'prep_clip' in k]
        rows = rows[marks[-1]:] if marks else rows
    agg = OrderedDict()
    for k, us in rows:
        k = k.split('(')[0][:70]
        a = agg.setdefault(k, [0, 0.0])
        a[0] += 1; a[1] += us
    tot = sum(a[1] for a in agg.values())
    print('| kernel | launches | time (us) | share |\n|---|---|---|---|')
    for k, (n, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print('| %s | %d | %.1f | %.1f %% |' % (k, n, us, 100 * us / tot))
    print('| total | %d | %.1f | 100 %% |' % (sum(a[0] for a in agg.values()), tot))


if __name__ == '__main__':
    main()
