#!/usr/bin/env python
"""Top stall locations of one profiled kernel (needs a report captured with --import-source on; runs HERE, no GPU):
   python tools/ncu_source_top.py r2_f16s_3x3.ncu-rep f16s_3x3_source.md "title"
"""
import csv
import io
import subprocess
import sys

KEYS = ['gpu__time_duration.sum', 'sm__cycles_elapsed.avg', 'dram__bytes_read.sum', 'dram__bytes_write.sum',
        'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active', 'smsp__issue_active.avg.pct_of_peak_sustained_active',
        'l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed', 'l1tex__data_pipe_lsu_wavefronts_mem_shared.sum',
        'l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum', 'lts__t_sectors_srcunit_tex.sum', 'lts__t_bytes_srcunit_tex.sum',
        'launch__registers_per_thread', 'launch__grid_size', 'launch__block_size', 'launch__shared_mem_per_block_dynamic',
        'sm__warps_active.avg.pct_of_peak_sustained_active']


def page(rep, which):
    raw = subprocess.run(['ncu', '-i', rep, '--page', which, '--csv'], capture_output=True, text=True).stdout
    return list(csv.reader(io.StringIO('\n'.join(l for l in raw.splitlines() if not l.startswith('==')))))


def main():
    rep, out, title = sys.argv[1], sys.argv[2], sys.argv[3]
    raw = page(rep, 'raw')
    h, u, r = raw[0], raw[1], raw[2]
    src = page(rep, 'source')
    kname = src[0][1] if len(src[0]) > 1 else ''
    hdr, data = src[1], src[2:]
    isrc, isamp = hdr.index('Source'), hdr.index('# Samples')
    stall = [i for i, x in enumerate(hdr) if x.startswith('stall_') and 'Not Issued' not in x]
    tot = sum(int(x[isamp] or 0) for x in data)
    agg = {}
    for x in data:
        for i in stall:
            if x[i]:
                agg[hdr[i]] = agg.get(hdr[i], 0) + int(x[i])
    with open(out, 'w') as f:
        f.write(f'# {title}\n\n`{kname[:160]}`\n\nreport: `{rep}` (ncu --set full --import-source on, one launch)\n\n| metric | value |\n|---|---:|\n')
        for k in KEYS:
            if k in h:
                f.write(f'| `{k}` | {r[h.index(k)]} {u[h.index(k)]} |\n')
        f.write(f'\n## warp-stall samples by reason (all {tot} samples)\n\n| reason | share |\n|---|---:|\n')
        for k, v in sorted(agg.items(), key=lambda kv: -kv[1])[:10]:
            f.write(f'| {k} | {100.0 * v / max(tot, 1):.1f} % |\n')
        f.write('\n## hottest SASS instructions\n\n| samples | share | instruction | top reasons |\n|---:|---:|---|---|\n')
        for x in sorted(data, key=lambda x: -int(x[isamp] or 0))[:24]:
            st = sorted(((hdr[i], int(x[i])) for i in stall if x[i] and int(x[i]) > 0), key=lambda kv: -kv[1])[:2]
            f.write(f'| {x[isamp]} | {100.0 * int(x[isamp]) / max(tot, 1):.1f} % | `{x[isrc].strip()[:80]}` | {", ".join(f"{a} {b}" for a, b in st)} |\n')
    print(out)


if __name__ == '__main__':
    main()
