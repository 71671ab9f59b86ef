"""Summarise an ncu report (ncu -i <rep> --page raw --csv) per kernel: launches, mean duration, DRAM bytes per launch,
achieved HBM GB/s and fraction of the measured copy peak, tensor-pipe %, L2 sectors, warps active/eligible, registers.
CPU-only.   python tools/ncu_summarize.py x.ncu-rep [name-filter-regex] > x_ncu.md"""
import collections
import csv
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNIT = {'nsecond': 1e-9, 'usecond': 1e-6, 'msecond': 1e-3, 'second': 1.0, 'ns': 1e-9, 'us': 1e-6, 'ms': 1e-3,
        'byte': 1.0, 'Kbyte': 1e3, 'Mbyte': 1e6, 'Gbyte': 1e9}
COLS = [('gpu__time_duration.sum', 'dur'), ('dram__bytes_read.sum', 'rd'), ('dram__bytes_write.sum', 'wr'),
        ('sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active', 'tensor_pct'),
        ('sm__inst_executed_pipe_tensor.sum', 'tensor_inst'),
        ('lts__t_sectors.sum', 'l2_sectors'), ('sm__warps_active.avg.pct_of_peak_sustained_active', 'warps_active_pct'),
        ('smsp__warps_eligible.avg.per_cycle_active', 'eligible'), ('launch__registers_per_thread', 'regs'),
        ('launch__grid_size', 'grid'), ('gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 'dram_pct'),
        ('sm__throughput.avg.pct_of_peak_sustained_elapsed', 'sm_pct')]


def main():
    rep = sys.argv[1]
    flt = re.compile(sys.argv[2]) if len(sys.argv) > 2 else None
    peak = json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))['hbm_gbs'] if os.path.exists(os.path.join(ROOT, 'MEASURED_PEAKS.json')) else 3350.0   # H100 SXM data sheet
    # a .csv argument is the already exported raw page (ncu -i x.ncu-rep --page raw --csv > x.csv on the GPU box: the report itself
    # can be very large)
    out = open(rep).read() if rep.endswith('.csv') else subprocess.run(['ncu', '-i', rep, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
    out = out[out.index('"ID"'):] if '"ID"' in out else out
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    idx = {n: i for i, n in enumerate(hdr)}
    agg = collections.OrderedDict()
    for r in rows[2:]:
        name = re.sub(r'\(.*', '', r[idx['Kernel Name']].replace('(anonymous namespace)::', '')).replace('void ', '')
        if flt and not flt.search(name):
            continue
        key = (name, r[idx['launch__grid_size']] if 'launch__grid_size' in idx else '')
        if os.environ.get('NCU_PER_LAUNCH'):
            key = key + (len(agg),)
        a = agg.setdefault(key, collections.defaultdict(list))
        for col, short in COLS:
            if col in idx and r[idx[col]] not in ('', 'n/a'):
                try:
                    v = float(r[idx[col]].replace(',', ''))
                except ValueError:
                    continue
                a[short].append(v * UNIT.get(units[idx[col]], 1.0))
    mean = lambda a, k: (sum(a[k]) / len(a[k])) if a.get(k) else None
    print(f'# ncu summary of `{os.path.basename(rep)}` (per kernel and grid size; means over the captured launches)\n')
    print(f'HBM fraction is against the measured copy peak {peak:.1f} GB/s (MEASURED_PEAKS.json). Durations under ncu are cold-cache, '
          'serialised launches (clock control none).\n')
    print('| kernel | grid | launches | us | DRAM rd MB | DRAM wr MB | GB/s | of HBM peak | tensor pipe % | L2 sectors (MB) | warps active % | eligible/cyc | regs |')
    print('|---|---|---|---|---|---|---|---|---|---|---|---|---|')
    for key, a in agg.items():
        name, grid = key[0], key[1]
        d, rd, wr = mean(a, 'dur'), mean(a, 'rd') or 0.0, mean(a, 'wr') or 0.0
        gbs = (rd + wr) / d / 1e9 if d else 0.0
        f = lambda v, fmt: (fmt % v) if v is not None else '-'
        l2 = mean(a, 'l2_sectors')
        print(f"| `{name}` | {grid} | {len(a['dur'])} | {d * 1e6:.1f} | {rd / 1e6:.2f} | {wr / 1e6:.2f} | {gbs:.0f} | {gbs / peak:.3f} | "
              f"{f(mean(a, 'tensor_pct'), '%.1f')} | {f(l2 * 32 / 1e6 if l2 else None, '%.1f')} | {f(mean(a, 'warps_active_pct'), '%.1f')} | "
              f"{f(mean(a, 'eligible'), '%.2f')} | {f(mean(a, 'regs'), '%.0f')} |")


if __name__ == '__main__':
    main()
