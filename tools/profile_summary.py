#!/usr/bin/env python3
"""Aggregates an ncu --csv launch list (tools/profile_step.sh) into profiles/<tag>_{launches.csv,traffic.json,inst.json}.
The run profiled is `bench.py --profile --steps 1 --warmup 1`: the launches of the SECOND step (the timed one) are kept.
  profile_summary.py RAW.csv TAG OUTDIR        write the summaries to OUTDIR (copy them into profiles/ and commit them
                                               to make them the evidence bench.py's roofline object cites)
  profile_summary.py --count RAW.csv KERNEL    launches of KERNEL in the warm-up step (= ncu -s for the timed step)
"""
import collections
import csv
import json
import os
import re
import sys

STAGE = {'bb_k_build_fragments': 'build_fragments', 'bb_k_mutate': 'error_loop', 'bb_k_mutate_chain': 'error_loop',
         'bb_k_window_lane': 'error_loop', 'bb_k_window_lane_hist': 'error_loop',
         'bb_k_window_warp': 'error_loop', 'bb_k_replay': 'error_loop', 'bb_k_window_tasks': 'error_loop',
         'bb_k_scan': 'scan', 'bb_k_join': 'join',
         'bb_k_push_roots': 'final_align', 'bb_k_node_warp': 'final_align', 'bb_k_node_lane': 'final_align',
         'bb_k_node_pair': 'final_align', 'bb_k_node_quad': 'final_align', 'bb_k_leaf_warp': 'final_align',
         'bb_k_leaf_lane': 'final_align', 'bb_k_leaf_lane_hist': 'final_align',
         'bb_k_qscores': 'qscores', 'bb_k_compact': 'compact'}


def load(path):
    lines = open(path, errors='replace').read().splitlines()
    start = next(i for i, ln in enumerate(lines) if ln.startswith('"ID"'))
    rows = list(csv.DictReader(lines[start:]))
    launches = collections.OrderedDict()
    for r in rows:
        try:
            lid = int(r['ID'])
        except (ValueError, KeyError):
            continue
        name = r['Kernel Name']
        m = re.match(r'(?:void )?(bb_k_\w+)(<[^>]*>)?', name)
        short = (m.group(1) + (m.group(2) or '')) if m else name
        short = re.sub(r'<\(int\)(\d+)>', r'<\1>', short).replace('<0>', '')
        d = launches.setdefault(lid, {'id': lid, 'kernel': short})
        try:
            val = float(r['Metric Value'].replace(',', ''))
        except ValueError:
            continue
        unit = r.get('Metric Unit', '')
        if r['Metric Name'] == 'gpu__time_duration.sum':
            val *= {'ns': 1e-6, 'us': 1e-3, 'usecond': 1e-3, 'ms': 1.0, 'msecond': 1.0, 'second': 1e3, 's': 1e3, 'nsecond': 1e-6}.get(unit, 1e-6)
        if r['Metric Name'].startswith('dram__bytes'):
            val *= {'byte': 1.0, 'Kbyte': 1e3, 'Mbyte': 1e6, 'Gbyte': 1e9, 'Tbyte': 1e12}.get(unit, 1.0)
        d[r['Metric Name']] = val
    return list(launches.values())


def timed_step(launches):
    """The launches of the second (timed) step.  A run is pure enqueueing of the same chain of kernels every step, so the
    profiled run (one warm-up step + one timed step) is two identical halves from the first bb_k_build_fragments on."""
    first = next((i for i, l in enumerate(launches) if l['kernel'].startswith('bb_k_build_fragments')), None)
    if first is None:
        return launches
    rest = launches[first:]
    half = len(rest) // 2
    if len(rest) % 2 == 0 and [l['kernel'] for l in rest[:half]] == [l['kernel'] for l in rest[half:]]:
        return rest[half:]
    # otherwise: everything from the last launch of the first worker's chain head on (best effort)
    idx = [i for i, l in enumerate(launches) if l['kernel'].startswith('bb_k_build_fragments')]
    return launches[idx[len(idx) // 2]:]


def main():
    if sys.argv[1] == '--count':
        launches = load(sys.argv[2])
        step = timed_step(launches)
        first = len(launches) - len(step)
        print(sum(1 for l in launches[:first] if l['kernel'].startswith(sys.argv[3])))
        return
    raw, tag, outdir = sys.argv[1], sys.argv[2], sys.argv[3]
    launches = timed_step(load(raw))
    per = collections.OrderedDict()
    for l in launches:
        k = per.setdefault(l['kernel'], {'launches': 0, 'ms': 0.0, 'dram_read_GB': 0.0, 'dram_write_GB': 0.0,
                                         'warp_inst_G': 0.0, 'thread_inst_G': 0.0, 'active_x_elapsed': 0.0, 'elapsed': 0.0,
                                         'warps_x_ms': 0.0})
        ms = l.get('gpu__time_duration.sum', 0.0)
        k['launches'] += 1
        k['ms'] += ms
        k['dram_read_GB'] += l.get('dram__bytes_read.sum', 0.0) / 1e9
        k['dram_write_GB'] += l.get('dram__bytes_write.sum', 0.0) / 1e9
        k['warp_inst_G'] += l.get('smsp__inst_executed.sum', 0.0) / 1e9
        k['thread_inst_G'] += l.get('smsp__thread_inst_executed.sum', 0.0) / 1e9
        k['active_x_elapsed'] += l.get('smsp__cycles_active.avg', 0.0)
        k['elapsed'] += l.get('sm__cycles_elapsed.max', 0.0)
        k['warps_x_ms'] += l.get('sm__warps_active.avg.per_cycle_active', 0.0) * ms
    total_ms = sum(k['ms'] for k in per.values())
    for name, k in per.items():
        k['share'] = k['ms'] / total_ms if total_ms else 0.0
        k['smsp_active_frac'] = k['active_x_elapsed'] / k['elapsed'] if k['elapsed'] else None
        k['warps_per_sm_when_active'] = k['warps_x_ms'] / k['ms'] if k['ms'] else None
        k['lanes_per_inst'] = k['thread_inst_G'] / k['warp_inst_G'] if k['warp_inst_G'] else None
        for drop in ('active_x_elapsed', 'elapsed', 'warps_x_ms'):
            del k[drop]
        for key, v in list(k.items()):
            if isinstance(v, float):
                k[key] = round(v, 4)
    per_stage = collections.OrderedDict()
    for name, k in per.items():
        st = STAGE.get(name.split('<')[0], 'other')
        s = per_stage.setdefault(st, {'ms': 0.0, 'dram_GB': 0.0, 'warp_inst_G': 0.0})
        s['ms'] += k['ms']
        s['dram_GB'] += k['dram_read_GB'] + k['dram_write_GB']
        s['warp_inst_G'] += k['warp_inst_G']
    src = ('ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum,smsp__inst_executed.sum,... '
           '--clock-control none over `python bench.py --profile --steps 1 --warmup 1` (tools/profile_step.sh; second pass = '
           'the timed step; the sub-batch workers are serialised and cold-cache under ncu, so shares matter, not absolutes)')
    traffic = {'source': src, 'per_kernel': per, 'serialised_total_ms': round(total_ms, 2), 'launches_per_step': len(launches),
               'total_dram_GB': round(sum(k['dram_read_GB'] + k['dram_write_GB'] for k in per.values()), 2),
               'per_stage': {k: {a: round(b, 3) for a, b in v.items()} for k, v in per_stage.items()}}
    inst = {'source': src, 'warp_inst_G_per_step': round(sum(k['warp_inst_G'] for k in per.values()), 3),
            'thread_inst_G_per_step': round(sum(k['thread_inst_G'] for k in per.values()), 3),
            'per_kernel': {n: k['warp_inst_G'] for n, k in per.items()}}
    for d in (outdir,):
        os.makedirs(d, exist_ok=True)
        json.dump(traffic, open(os.path.join(d, f'{tag}_traffic.json'), 'w'), indent=1)
        json.dump(inst, open(os.path.join(d, f'{tag}_inst.json'), 'w'), indent=1)
        with open(os.path.join(d, f'{tag}_launches.csv'), 'w') as f:
            f.write('id,kernel,ms,dram_read_MB,dram_write_MB,warp_inst_M,smsp_active_frac,warps_per_sm\n')
            for l in launches:
                el = l.get('sm__cycles_elapsed.max', 0.0)
                f.write('%d,%s,%.4f,%.2f,%.2f,%.2f,%.3f,%.2f\n' % (
                    l['id'], l['kernel'], l.get('gpu__time_duration.sum', 0.0), l.get('dram__bytes_read.sum', 0.0) / 1e6,
                    l.get('dram__bytes_write.sum', 0.0) / 1e6, l.get('smsp__inst_executed.sum', 0.0) / 1e6,
                    (l.get('smsp__cycles_active.avg', 0.0) / el) if el else 0.0, l.get('sm__warps_active.avg.per_cycle_active', 0.0)))
    for name, k in per.items():
        print('%-26s n=%4d ms=%8.2f dram=%7.2f GB inst=%7.2f G active=%s warps/SM=%s lanes=%s' % (
            name, k['launches'], k['ms'], k['dram_read_GB'] + k['dram_write_GB'], k['warp_inst_G'], k['smsp_active_frac'],
            k['warps_per_sm_when_active'], k['lanes_per_inst']))
    print('total %.1f ms serialised, %.1f GB DRAM, %.1f G warp-inst' % (total_ms, traffic['total_dram_GB'], inst['warp_inst_G_per_step']))


if __name__ == '__main__':
    main()
