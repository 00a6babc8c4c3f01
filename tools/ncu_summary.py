"""Condense an .ncu-rep (ncu --set full) into the text summary kept under profiles/.
  python tools/ncu_summary.py prof.ncu-rep profiles/<name>.txt ["note"]"""
import csv, io, subprocess, sys

KEYS = ['gpu__time_duration.sum', 'launch__grid_size', 'launch__block_size', 'launch__registers_per_thread',
        'launch__shared_mem_per_block_dynamic', 'launch__shared_mem_per_block_static', 'launch__occupancy_limit_registers',
        'launch__occupancy_limit_shared_mem', 'sm__warps_active.avg.pct_of_peak_sustained_active',
        'smsp__inst_executed.sum', 'smsp__issue_active.avg.pct_of_peak_sustained_active',
        'smsp__thread_inst_executed_per_inst_executed.ratio', 'dram__bytes_read.sum', 'dram__bytes_write.sum',
        'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 'l1tex__t_sector_hit_rate.pct', 'lts__t_sector_hit_rate.pct',
        'l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum', 'sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active',
        'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active', 'sm__throughput.avg.pct_of_peak_sustained_elapsed']


def page(rep, name):
    return subprocess.run(['ncu', '-i', rep, '--page', name, '--csv'], capture_output=True, text=True).stdout


def main():
    rep, out = sys.argv[1], sys.argv[2]
    note = sys.argv[3] if len(sys.argv) > 3 else ''
    rows = list(csv.reader(io.StringIO(page(rep, 'raw'))))
    hdr, units = rows[0], rows[1]
    lines = [f'# ncu summary of {rep}', f'# {note}', '# (ncu --set full --clock-control none; per-launch values; times are cold-cache, serialised replays)', '']
    for r in rows[2:]:
        d = dict(zip(hdr, r))
        lines.append('== ' + d.get('Kernel Name', '?'))
        for k in KEYS:
            if k in d and d[k] != '':
                lines.append(f'   {k:70s} {d[k]:>18s} {units[hdr.index(k)]}')
        st = []
        for k in hdr:
            if 'issue_stalled' in k and k.endswith('per_issue_active.ratio'):
                try:
                    v = float(d[k])
                except ValueError:
                    continue
                if v >= 0.2:
                    st.append((v, k.replace('smsp__average_warps_issue_stalled_', '').replace('_per_issue_active.ratio', '')))
        lines.append('   warp stall reasons (warps per issue slot): ' + ', '.join(f'{n}={v:.2f}' for v, n in sorted(st, reverse=True)))
        lines.append('')
    # hottest SASS of each kernel instance (needs -lineinfo / --import-source)
    src = list(csv.reader(io.StringIO(page(rep, 'source'))))
    starts = [i for i, r in enumerate(src) if r and r[0] == 'Kernel Name'] + [len(src)]
    seen = set()
    for a, b in zip(starts[:-1], starts[1:]):
        name = src[a][1]
        if name in seen:
            continue
        seen.add(name)
        try:
            hi = [i for i in range(a, b) if src[i] and src[i][0] == 'Address'][0]
        except IndexError:
            continue
        h = src[hi]
        ia, isamp, iinst = h.index('Source'), h.index('# Samples'), h.index('Instructions Executed')
        f = lambda x: int(x) if x.strip().isdigit() else 0
        data = [r for r in src[hi + 1:b] if len(r) > max(isamp, iinst)]
        tot_i = sum(f(r[iinst]) for r in data) or 1
        tot_s = sum(f(r[isamp]) for r in data) or 1
        lines.append(f'== hottest SASS by stall samples: {name[:70]}  (total warp-instructions {tot_i}, samples {tot_s})')
        for r in sorted(data, key=lambda r: -f(r[isamp]))[:18]:
            lines.append(f'   {100.0 * f(r[isamp]) / tot_s:5.1f}% samples  {100.0 * f(r[iinst]) / tot_i:5.2f}% inst   {r[ia][:90]}')
        ops = ' '.join(r[ia] for r in data)
        marks = [m for m in ('UBLKCP', 'UTMASTG', 'UTMALDG', 'LDGSTS', 'HMMA', 'UTCHMMA', 'LDTM', 'CCTL.IVALL', 'ATOMS', 'RED.', 'ATOMG') if m in ops]
        lines.append('   SASS markers present: ' + (', '.join(marks) if marks else 'none of UBLKCP/UTMA*/HMMA/UTC*MMA'))
        lines.append('')
    open(out, 'w').write('\n'.join(lines) + '\n')
    print('wrote', out)


if __name__ == '__main__':
    main()
