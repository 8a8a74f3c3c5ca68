"""Summarise .ncu-rep captures (read with `ncu -i`, no GPU needed) into a small markdown table.
    python tools/ncu_summary.py prof_a.ncu-rep [more.ncu-rep ...] > summary.md"""
import csv
import io
import subprocess
import sys

WANT = [
    'gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum',
    'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active',
    'sm__throughput.avg.pct_of_peak_sustained_elapsed', 'sm__warps_active.avg.pct_of_peak_sustained_active',
    'lts__t_sector_hit_rate.pct', 'launch__registers_per_thread', 'launch__grid_size', 'launch__block_size',
    'launch__shared_mem_per_block_dynamic', 'smsp__cycles_active.avg',
]


def raw(path):
    out = subprocess.run(['ncu', '-i', path, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    h = rows[0]
    res = []
    for r in rows[2:]:
        d = {h[i]: (r[i], rows[1][i]) for i in range(min(len(h), len(r)))}
        res.append(d)
    return res


def main():
    print('| capture | kernel | ' + ' | '.join(w.split('.')[0].replace('__', ' ') for w in WANT) + ' |')
    print('|---|---|' + '---|' * len(WANT))
    for p in sys.argv[1:]:
        for d in raw(p):
            name = d.get('Kernel Name', ('?', ''))[0][:60]
            print('| %s | %s | ' % (p.split('/')[-1], name) + ' | '.join('%s %s' % (d[w][0], d[w][1]) if w in d else '-' for w in WANT) + ' |')


if __name__ == '__main__':
    main()
