"""Throughput of the shared-encoder ablation (single_transformer=1) against the vanilla network, on bench.py's workload:
the 10k-point sphere, res 256, eps 3, the fused reconstruction (tc engine, guard band 0.05, distance-weighted
sub-sample), the same P = 300 and S = 1000.  The two engines are timed in one process, alternating, with CUDA events
around each fused call; a separate profiled pass per engine reads the pass kernel's time, launches and algorithmic FLOPs
from `profile_get`.

    python tools/shared_encoder_bench.py [--res 256] [--steps 5] [--warmup 2]

Prints the card's name and power limit, one line per engine and a JSON summary line."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from points2surf_b200 import ops, synth  # noqa: E402

SEED = 40938661


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = 'unknown'
    return name, power or 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--res', type=int, default=256)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('shared_encoder_bench needs a CUDA device')
    kw = dict(points_per_patch=300, sub_sample_size=1000, precision='tc', guard_band=0.05)
    v = synth.VARIANTS['vanilla']
    engines = {
        'shared encoder': ops.Engine(synth.make_state_dict('shared_encoder', 12, fitted=True), 1, 0, single_transformer=True,
                                     **kw),
        'vanilla': ops.Engine(synth.make_state_dict('vanilla', 6, fitted=True), v['use_point_stn'], v['shared_transformer'],
                              **kw),
    }
    pts = torch.from_numpy(synth.make_cloud('sphere', 10000, seed=0)).cuda()
    times = {k: [] for k in engines}
    Q, guard = {}, {}
    for step in range(a.warmup + a.steps):
        for name, eng in engines.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0.record()
            lin, sdf = eng.reconstruct(pts, a.res, 3, 0, SEED)
            t1.record()
            torch.cuda.synchronize()
            if step >= a.warmup:
                times[name].append(t0.elapsed_time(t1))
            Q[name] = lin.numel()
            guard[name] = eng.last_guard_count()
    prof = {}
    for name, eng in engines.items():          # profiled separately: the events around each pass launch add host work
        eng.profile_enable(True)
        eng.reconstruct(pts, a.res, 3, 0, SEED)
        torch.cuda.synchronize()
        prof[name] = eng.profile_get()
        eng.profile_enable(False)
    gpu, power = card()
    print('card: %s, power limit %s' % (gpu, power))
    result = {'card': gpu, 'power_limit': power, 'res': a.res, 'steps': a.steps, 'engines': {}}
    for name in engines:
        t = np.array(times[name])
        qps = Q[name] / (np.median(t) / 1e3)
        p = prof[name]
        tflops = p['flops'] / (p['ms'] / 1e3) / 1e12 if p['ms'] > 0 else float('nan')
        print('%-15s Q %d  median %.2f ms/shape (min %.2f, max %.2f)  %.0f queries/s  pass kernel %.2f ms in %d launches '
              '(%.2f ms each, %.0f TFLOP/s algorithmic)  guard-band recompute %d'
              % (name, Q[name], np.median(t), t.min(), t.max(), qps, p['ms'], p['launches'], p['ms'] / max(p['launches'], 1),
                 tflops, guard[name]))
        result['engines'][name] = {'queries': Q[name], 'median_ms': float(np.median(t)), 'min_ms': float(t.min()),
                                   'max_ms': float(t.max()), 'queries_per_s': float(qps), 'pass_ms': p['ms'],
                                   'pass_launches': p['launches'], 'pass_tflops': tflops, 'guard_recompute': guard[name]}
    for eng in engines.values():
        eng.close()
    print(json.dumps(result))


if __name__ == '__main__':
    main()
