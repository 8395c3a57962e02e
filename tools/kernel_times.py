"""Per-kernel times of one workload step on the GPU, with the traceback-history bytes of the lane aligners.

Runs a BASELINE config's workload the way bench.py times it (the batch resident on the device, default knobs): warm-up
steps, then --steps steps under torch.profiler with CUDA activities, in a process of its own.  Writes one JSON file (and
prints it): the card's name, power limit and SM clocks read in the same call; per-kernel device time per step (sum of
the kernel's launches; kernels of the two alignment pipelines and of the two workers overlap, so the sum over kernels is
more than the step); the bb_last_run_ms stages per step; and the history bytes per step of the lane aligners:

  leaves   bb_k_leaf_lane_hist writes one history entry of 8 bytes per column and word, and its traceback stages every
           column the path walks through (about all of them) once.  Counted from the oracle's Hirschberg trees on a seeded
           sample of --sample reads (routing, band and words as the device computes them; a root leaf's band from its
           distance, where the device starts from the read's injected-edit bound), scaled to the step's reads.  Words per
           column: 8 with the full window (the layout before the band slices), bb_band_words(a, b) with the slices.
  windows  bb_k_window_lane_hist<4> / <8>: window counts from bb_last_run_work, 1000 columns a window (the window length;
           the joined window differs by its indels).  The window's band is not known on the host: 4 / 8 words with the
           full window, at most 3 / 7 with the slices (an upper bound).

    python tools/kernel_times.py [--config 1] [--steps 3] [--warmup 2] [--sample 512] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
sys.path.insert(0, ROOT)

HIST_KERNELS = ('bb_k_window_lane_hist', 'bb_k_leaf_lane_hist')
LEAF_LW, LEAF_COLS, WIN_COLS = 8, 2048, 1000


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    out = subprocess.run(['nvidia-smi', '-i', '0', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True,
                         text=True, check=True).stdout.strip()
    return dict(zip(q.split(','), [x.strip() for x in out.split(',')]))


def band(nn, mm, k):
    """bb_task_band: bb_band of the clamped bound, made even."""
    k = max(k, abs(nn - mm))
    k = min(k, max(nn, mm))
    a, b = max(0, (k - (nn - mm)) // 2), max(0, (k + (nn - mm)) // 2)
    if a + b < 1:
        b = 1
    return a + (a & 1), b + (b & 1)


def uses_traceback(n, m):
    return 20 * ((n + 63) // 64) * m + 8 * m < 1048576


def leaf_columns(wl, sample, seed):
    """Columns x words of the lane leaves of `sample` seeded reads, for the full window and for the band slices."""
    import bench
    from oracle import oracle as O
    rs = np.random.RandomState(seed)
    picks = [(b, j) for b, bt in enumerate(wl.batches) for j in range(len(bt))]
    picks = [picks[i] for i in sorted(rs.choice(len(picks), min(sample, len(picks)), replace=False))]
    orc = O.Oracle(*wl.models)
    frs = [wl.batches[b].fragment(j, wl.ref.concat) for b, j in picks]
    ids = [float(wl.batches[b].target_identity[j]) for b, j in picks]
    idx = [int(wl.batches[b].read_index[j]) for b, j in picks]
    outs, _ = orc.sequence_batch(frs, ids, bench.SEED, idx, n_threads=os.cpu_count() or 1, with_stats=True)
    full = slices = leaves = 0
    for o in outs:
        for depth, q0, nn, t0, mm, best, is_leaf, _ in o[4]['tree']:
            if not is_leaf or not uses_traceback(nn, mm):
                continue
            a, b = band(nn, mm, best)
            if ((a + b) >> 5) + 2 > LEAF_LW or mm > LEAF_COLS:
                continue   # bb_k_leaf_warp
            leaves += 1
            full += mm * LEAF_LW
            slices += mm * (((a + b) >> 5) + 1)
    return len(picks), leaves, full, slices


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', type=int, default=1)
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--sample', type=int, default=512, help='reads of the oracle sample for the leaf history bytes')
    ap.add_argument('--out', type=str, default=os.path.join(ROOT, 'profile_out'), help='directory of the JSON file')
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from badread_b200.engine import Engine

    wl = bench.Workload(a.config, 0, 1, 'weak')
    assert len(wl.batches) == 1, 'one resident batch per step'
    eng = Engine(device=0, seed=bench.SEED)
    eng.upload_reference(wl.ref.concat)
    eng.set_error_model(wl.models[0])
    eng.set_qscore_model(wl.models[1])
    eng.upload_batch(wl.batches[0])
    for _ in range(a.warmup):
        eng.run_batch()
        eng.last_run_ms()
    stages, dev_ms = {}, 0.0
    t0 = time.perf_counter()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            eng.run_batch()
            ms, st = eng.last_run_ms()
            dev_ms += ms
            for k, v in st.items():
                stages[k] = stages.get(k, 0.0) + v
        torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    info = card()
    eng.fetch_batch()
    work = eng.last_run_work()

    kernels = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = ev.name
        t = ev.device_time_total if hasattr(ev, 'device_time_total') else ev.cuda_time_total
        k = kernels.setdefault(name, [0.0, 0])
        k[0] += t / 1e3
        k[1] += 1
    per_step = {n: {'ms': round(v[0] / a.steps, 3), 'launches': v[1] // a.steps}
                for n, v in sorted(kernels.items(), key=lambda kv: -kv[1][0])}
    kernel_sum = sum(v['ms'] for v in per_step.values())

    n_reads = wl.n_reads
    n_s, leaves_s, full_s, slices_s = leaf_columns(wl, a.sample, bench.SEED)
    scale = n_reads / n_s
    w4, w8 = int(work['window_lane4']), int(work['window_lane8'])
    hist = {
        'leaf_sample': f'{n_s} reads of {n_reads} (RandomState({bench.SEED})), {leaves_s} lane leaves, scaled x{scale:.1f}',
        'leaf_written_GB_full_window': full_s * 8 * scale / 1e9,
        'leaf_written_GB_band_slices': slices_s * 8 * scale / 1e9,
        'windows_lane4': w4, 'windows_lane8': w8,
        'window_written_GB_full_window': (w4 * 4 + w8 * 8) * WIN_COLS * 8 / 1e9,
        'window_written_GB_band_slices_at_most': (w4 * 3 + w8 * 7) * WIN_COLS * 8 / 1e9,
        'note': 'bytes read by the tracebacks ~ bytes written (every walked column is staged once)',
    }
    hk = {n: v for n, v in per_step.items() if any(h in n for h in HIST_KERNELS)}
    hk_ms = sum(v['ms'] for v in hk.values())
    res = {
        'config': a.config, 'card': info, 'steps': a.steps, 'reads_per_step': n_reads,
        'step_ms_events': dev_ms / a.steps, 'step_ms_wall_profiled': wall * 1e3 / a.steps,
        'stages_ms_per_step': {k: round(v / a.steps, 3) for k, v in stages.items()},
        'kernel_ms_per_step_sum': round(kernel_sum, 3),
        'history_kernels_ms_per_step': round(hk_ms, 3),
        'history_kernels_share_of_kernel_time': round(hk_ms / kernel_sum, 4) if kernel_sum else None,
        'history_bytes_per_step': hist,
        'kernels': per_step,
    }
    os.makedirs(a.out, exist_ok=True)
    path = os.path.join(a.out, f'kernel_times_config{a.config}.json')
    with open(path, 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != 'kernels'}, indent=1))
    for n, v in list(per_step.items())[:25]:
        print(f'{v["ms"]:10.3f} ms {v["launches"]:5d}  {n[:150]}')
    eng.close()


if __name__ == '__main__':
    main()
