#!/usr/bin/env python
"""Condense an `ncu --page raw --csv` export (one row per profiled launch, hundreds of metric columns) into the handful of
metrics the roofline discussion uses, one row per launch, plus a per-kernel summary.

    ncu -i capture.ncu-rep --page raw --csv > raw.csv
    python tools/ncu_select.py raw.csv selected.csv
"""
import csv
import sys

KEEP = [
    'Kernel Name', 'Grid Size', 'Block Size', 'gpu__time_duration.sum', 'dram__bytes_read.sum', 'dram__bytes_write.sum',
    'dram__bytes.sum.per_second',
    'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 'lts__throughput.avg.pct_of_peak_sustained_elapsed',
    'l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed', 'sm__throughput.avg.pct_of_peak_sustained_elapsed',
    'sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active', 'smsp__issue_active.avg.pct_of_peak_sustained_active',
    'sm__warps_active.avg.pct_of_peak_sustained_active', 'launch__registers_per_thread', 'launch__shared_mem_per_block_dynamic',
    'launch__waves_per_multiprocessor', 'launch__occupancy_limit_registers', 'launch__occupancy_limit_shared_mem',
    'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed',
    'sm__inst_executed_pipe_uniform.sum', 'sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active',
]


def main(src, dst):
    rows = list(csv.reader(open(src, newline='')))
    start = next(i for i, r in enumerate(rows) if r and r[0] == 'ID')          # ncu prints ==PROF== lines before the table
    header, units, data = rows[start], rows[start + 1], rows[start + 2:]
    cols = [(name, header.index(name)) for name in KEEP if name in header]
    with open(dst, 'w', newline='') as f:
        w = csv.writer(f)
        w.writerow([n for n, _ in cols])
        w.writerow([units[i] for _, i in cols])
        for r in data:
            if len(r) > max(i for _, i in cols):
                w.writerow([r[i] for _, i in cols])
    # per-kernel summary on stdout
    f = lambda s: float(s.replace(',', '')) if s not in ('', 'n/a') else 0.0
    ki, ti = header.index('Kernel Name'), header.index('gpu__time_duration.sum')
    di = header.index('gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed')
    have_bytes = 'dram__bytes_read.sum' in header
    if have_bytes:
        ri, wi = header.index('dram__bytes_read.sum'), header.index('dram__bytes_write.sum')
    else:
        bi = header.index('dram__bytes.sum.per_second')          # bytes = rate x duration
    agg = {}
    for r in data:
        if len(r) <= max(ki, ti, di):
            continue
        name = r[ki].split('(')[0]
        e = agg.setdefault(name, [0, 0.0, 0.0, 0.0])
        t = f(r[ti])
        e[0] += 1; e[1] += t; e[3] = max(e[3], f(r[di]))
        e[2] += (f(r[ri]) + f(r[wi])) if have_bytes else f(r[bi]) * t
    print(f'time unit: {units[ti]}; dram: ' + (f'bytes in {units[ri]}' if have_bytes else f'rate [{units[bi]}] x duration [{units[ti]}]'))
    print('  total time   launches   total dram      max dram %   kernel')
    for name, (n, t, b, d) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f'{t:12.1f}  n={n:4d}  dram={b:14.1f}  max dram%={d:5.1f}  {name[:90]}')


if __name__ == '__main__':
    main(sys.argv[1], sys.argv[2])
