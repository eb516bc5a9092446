#!/usr/bin/env python
"""Turn gpurun_out/ ncu artefacts into the tracked summaries under profiles/ (run here, no GPU needed).

    python tools/summarize_profiles.py r01a      # tag = round + capture id
"""
import collections
import csv
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, 'gpurun_out')
PROF = os.path.join(ROOT, 'profiles')
KEYS = ['gpu__time_duration.sum', 'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed', 'lts__throughput.avg.pct_of_peak_sustained_elapsed', 'l1tex__data_pipe_tc_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed', 'sm__issue_active.avg.pct_of_peak_sustained_elapsed', 'dram__bytes_read.sum', 'dram__bytes_write.sum', 'lts__t_bytes.sum',
        'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 'sm__throughput.avg.pct_of_peak_sustained_elapsed',
        'sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active', 'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active',
        'sm__warps_active.avg.pct_of_peak_sustained_active', 'launch__registers_per_thread', 'launch__grid_size',
        'launch__block_size', 'launch__shared_mem_per_block_dynamic', 'launch__occupancy_limit_registers',
        'launch__occupancy_limit_shared_mem', 'l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum',
        'l1tex__data_pipe_lsu_wavefronts_mem_shared.sum', 'sm__cycles_elapsed.max']


def launches(tag):
    path = os.path.join(OUT, 'launches.csv')
    if not os.path.exists(path):
        return
    lines = [l for l in open(path) if not l.startswith('==')]
    agg = collections.defaultdict(lambda: [0, 0.0])
    total = 0.0
    n = 0
    for row in csv.DictReader(lines):
        v = float(row['Metric Value'].replace(',', ''))
        u = row['Metric Unit']
        v = v / 1000.0 if u in ('ns', 'nsecond') else (v * 1000.0 if u in ('ms', 'msecond') else v)
        name = re.sub(r'\(.*', '', row['Kernel Name']).replace('<unnamed>::', '').replace('void ', '')[:64]
        agg[name][0] += 1
        agg[name][1] += v
        total += v
        n += 1
    with open(os.path.join(PROF, '%s_launches.md' % tag), 'w') as f:
        f.write('# ncu launch list of ONE bench step (eager launches, `--metrics gpu__time_duration.sum '
                '--clock-control none`)\n\n')
        f.write('Command: `SB200_CUDA_GRAPH=0 ncu ... python bench.py --steps 1 --warmup 3 --lite` '
                '(see tools/profile_gpu.sh).  Per-launch times are cold-cache and serialised: compare SHARES.\n\n')
        f.write('%d launches, %.1f us total\n\n| kernel | launches | total us | avg us | share |\n|---|---:|---:|---:|---:|\n' % (n, total))
        for k, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write('| `%s` | %d | %.1f | %.2f | %.1f%% |\n' % (k, c, t, t / c, 100 * t / total))
    print('wrote launches summary (%d launches)' % n)


def report(name, tag):
    rep = os.path.join(OUT, name + '.ncu-rep')
    if not os.path.exists(rep):
        return
    raw = subprocess.run(['ncu', '-i', rep, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    with open(os.path.join(PROF, '%s_%s.md' % (tag, name)), 'w') as f:
        f.write('# ncu --set full: %s\n\n' % name)
        for vals in rows[2:]:
            kn = vals[hdr.index('Kernel Name')] if 'Kernel Name' in hdr else '?'
            f.write('## %s\n\n| metric | value | unit |\n|---|---:|---|\n' % kn[:120])
            for k in KEYS:
                if k in hdr:
                    i = hdr.index(k)
                    f.write('| %s | %s | %s |\n' % (k, vals[i], units[i]))
            f.write('\n')
    print('wrote', name)


def traffic(pairs):
    """profiles/traffic.json: dram__bytes_read.sum + dram__bytes_write.sum per launch of the captured kernels -- what
    bench.py's roofline objects report as `traffic`."""
    import json
    out = {}
    path = os.path.join(PROF, 'traffic.json')
    if os.path.exists(path):
        out = json.load(open(path))            # keep the entries whose capture is not in gpurun_out/ this time
    for key, name in pairs:
        rep = os.path.join(OUT, name + '.ncu-rep')
        if not os.path.exists(rep):
            continue
        raw = subprocess.run(['ncu', '-i', rep, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
        rows = list(csv.reader(raw.splitlines()))
        hdr, units, vals = rows[0], rows[1], rows[2]

        def val(k):
            i = hdr.index(k)
            v = float(vals[i].replace(',', ''))
            u = units[i].lower()
            return v * {'byte': 1, 'kbyte': 1e3, 'mbyte': 1e6, 'gbyte': 1e9}.get(u, 1)
        out[key] = {'dram_bytes': int(val('dram__bytes_read.sum') + val('dram__bytes_write.sum')),
                    'dram_bytes_read': int(val('dram__bytes_read.sum')), 'dram_bytes_write': int(val('dram__bytes_write.sum')),
                    'gpu_time_us': float(vals[hdr.index('gpu__time_duration.sum')]), 'capture': name + '.ncu-rep',
                    'kernel': vals[hdr.index('Kernel Name')][:80]}
    with open(os.path.join(PROF, 'traffic.json'), 'w') as f:
        json.dump(out, f, indent=1)
    print('wrote traffic.json', out)


def sass_excerpt(tag, obj, out_name, patterns):
    """Counts of the listed SASS mnemonics in one object file, with the lines that carry them."""
    sass = subprocess.run(['cuobjdump', '-sass', obj], capture_output=True, text=True).stdout.splitlines()
    hits = collections.Counter()
    lines = []
    for l in sass:
        m = re.search(r'/\*[0-9a-f]+\*/\s+(@!?U?P\d+\s+)?([A-Z0-9_.]+)', l)
        if not m:
            continue
        op = m.group(2)
        for p_ in patterns:
            if op.startswith(p_):
                hits[op] += 1
                if len(lines) < 40:
                    lines.append(l.strip()[:120])
    with open(os.path.join(PROF, '%s_%s.md' % (tag, out_name)), 'w') as f:
        f.write('# SASS evidence (`cuobjdump -sass %s`)\n\n| opcode | count |\n|---|---:|\n' % os.path.relpath(obj, ROOT))
        for k, v in sorted(hits.items()):
            f.write('| `%s` | %d |\n' % (k, v))
        f.write('\nFirst occurrences:\n\n```\n%s\n```\n' % '\n'.join(lines))
    print('wrote sass excerpt', dict(hits))


if __name__ == '__main__':
    tag = sys.argv[1] if len(sys.argv) > 1 else 'r02'
    os.makedirs(PROF, exist_ok=True)
    launches(tag)
    for n in ('prof_rollout', 'prof_tc5', 'prof_critic', 'prof_gae', 'prof_epochs2', 'prof_gae_large'):
        report(n, tag)
    traffic([('rollout', 'prof_rollout'), ('critic', 'prof_tc5'), ('epochs2', 'prof_epochs2'), ('gae_large', 'prof_gae_large')])
    obj = os.path.join(ROOT, 'surreal_b200', 'build', 'mlp_fwd_tc5.o')
    if os.path.exists(obj):
        sass_excerpt(tag, obj, 'sass_tc5', ['HGMMA', 'UBLKCP', 'SYNCS', 'WARPGROUP'])
