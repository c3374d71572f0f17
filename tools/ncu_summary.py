#!/usr/bin/env python
"""Summarise an `ncu --set full` report into per-kernel roofline rows (run HERE, no GPU needed):

  python tools/ncu_summary.py r2_ops.ncu-rep r2_kernels [--peaks MEASURED_PEAKS.json]

writes <out>.json (one record per profiled launch) and <out>.md (one table row per launch): duration, DRAM bytes read + written,
achieved DRAM GB/s against the measured copy bandwidth, tensor-pipe active %, L2 -> SM bytes, shared-memory bank-conflict share.
"""
import csv
import io
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WANT = {
    'dur_ns': ['gpu__time_duration.sum'],
    'dram_rd': ['dram__bytes_read.sum'],
    'dram_wr': ['dram__bytes_write.sum'],
    'dram_pct': ['gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed'],
    'tensor_pct': ['sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active', 'sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active',
                   'sm__inst_executed_pipe_tensor.avg.pct_of_peak_sustained_active'],
    'sm_pct': ['sm__throughput.avg.pct_of_peak_sustained_elapsed'],
    'l2_to_sm': ['lts__t_bytes_srcunit_tex.sum', 'lts__t_sectors_srcunit_tex.sum'],
    'smem_wavefronts': ['l1tex__data_pipe_lsu_wavefronts_mem_shared.sum'],
    'smem_conflicts': ['l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum'],
    'warps_active_pct': ['sm__warps_active.avg.pct_of_peak_sustained_active'],
    'regs': ['launch__registers_per_thread'],
    'grid': ['launch__grid_size'],
    'block': ['launch__block_size'],
    'smem_dyn': ['launch__shared_mem_per_block_dynamic'],
}
UNIT = {'byte': 1, 'Kbyte': 1e3, 'Mbyte': 1e6, 'Gbyte': 1e9, 'ns': 1, 'us': 1e3, 'ms': 1e6, 'nsecond': 1, 'usecond': 1e3, 'msecond': 1e6,
        'second': 1e9, 'sector': 32}


def num(v):
    try:
        return float(v.replace(',', ''))
    except Exception:
        return None


def main():
    rep, out = sys.argv[1], sys.argv[2]
    peaks = os.path.join(ROOT, 'MEASURED_PEAKS.json')
    hbm = json.load(open(peaks))['hbm_gbs'] if os.path.exists(peaks) else 6650.0
    raw = subprocess.run(['ncu', '-i', rep, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
    lines = [l for l in raw.splitlines() if not l.startswith('==')]
    rd = list(csv.reader(io.StringIO('\n'.join(lines))))
    head, units, rows = rd[0], rd[1], rd[2:]
    col = {n: i for i, n in enumerate(head)}
    recs = []
    for r in rows:
        name = re.sub(r'\(.*', '', r[col['Kernel Name']])
        name = re.sub(r'^void |\(anonymous namespace\)::', '', name)
        rec = {'id': int(r[col['ID']]), 'kernel': name}
        for key, metrics in WANT.items():
            for m in metrics:
                if m in col and num(r[col[m]]) is not None:
                    rec[key] = num(r[col[m]]) * UNIT.get(units[col[m]], 1)
                    break
        if 'dur_ns' not in rec:
            continue
        dram = rec.get('dram_rd', 0) + rec.get('dram_wr', 0)
        rec['dram_bytes'] = dram
        rec['dram_gbs'] = dram / rec['dur_ns'] if rec['dur_ns'] else 0
        rec['hbm_frac_of_measured'] = rec['dram_gbs'] / hbm
        if rec.get('smem_wavefronts'):
            rec['smem_conflict_share'] = rec.get('smem_conflicts', 0) / rec['smem_wavefronts']
        recs.append(rec)
    json.dump({'source': os.path.basename(rep), 'hbm_peak_gbs_measured': hbm, 'launches': recs}, open(out + '.json', 'w'), indent=1)
    with open(out + '.md', 'w') as f:
        f.write(f'# ncu --set full, per launch ({os.path.basename(rep)}); HBM peak = measured copy bandwidth {hbm:.0f} GB/s\n\n')
        f.write('| # | kernel | grid x block | us | DRAM MB (r+w) | DRAM GB/s | of HBM peak | tensor pipe % | SM % | L2->SM MB | smem conflict share | regs |\n')
        f.write('|---:|---|---|---:|---:|---:|---:|---:|---:|---:|---:|---:|\n')
        for r in recs:
            f.write('| {id} | `{k}` | {g:.0f} x {b:.0f} | {us:.1f} | {mb:.2f} | {gbs:.0f} | {fr:.1%} | {tp} | {sm} | {l2} | {cf} | {rg:.0f} |\n'.format(
                id=r['id'], k=r['kernel'][:70], g=r.get('grid', 0), b=r.get('block', 0), us=r['dur_ns'] / 1e3, mb=r['dram_bytes'] / 1e6,
                gbs=r['dram_gbs'], fr=r['hbm_frac_of_measured'], tp=f"{r['tensor_pct']:.1f}" if 'tensor_pct' in r else '-',
                sm=f"{r['sm_pct']:.1f}" if 'sm_pct' in r else '-', l2=f"{r['l2_to_sm'] / 1e6:.1f}" if 'l2_to_sm' in r else '-',
                cf=f"{r['smem_conflict_share']:.2f}" if 'smem_conflict_share' in r else '-', rg=r.get('regs', 0)))
    print(f'{len(recs)} launches -> {out}.md / .json')


if __name__ == '__main__':
    main()
