"""Queries/s of the regression ablation's network (outputs imp_surf: fc4 128 -> 1) against the same network with the
two-output head (imp_surf_magnitude, imp_surf_sign), on bench.py's workload: the 10k-point sphere, res 256, eps 3, the
fused reconstruction (tc engine, default guard band 0.05, distance-weighted sub-sample).  Both engines are timed in one
process, alternating, with CUDA events around each fused call.

    python tools/regression_bench.py [--res 256] [--steps 5] [--warmup 2]

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
        raise SystemExit('regression_bench needs a CUDA device')
    v = synth.VARIANTS['regression']
    sd1 = synth.make_state_dict('regression', 10, fitted=True)
    sd2 = dict(sd1)
    # the same network with the two-output head: both logits are the fitted regression logit
    sd2['fc4.weight'] = sd1['fc4.weight'].repeat(2, 1)
    sd2['fc4.bias'] = sd1['fc4.bias'].repeat(2)
    engines = {
        'regression (output_dim 1)': ops.Engine(sd1, v['use_point_stn'], v['shared_transformer'], precision='tc',
                                                guard_band=0.05, output_dim=1),
        'magnitude + sign (output_dim 2)': ops.Engine(sd2, v['use_point_stn'], v['shared_transformer'], precision='tc',
                                                      guard_band=0.05, output_dim=2),
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
    gpu, power = card()
    print('card: %s, power limit %s' % (gpu, power))
    result = {'card': gpu, 'power_limit': power, 'res': a.res, 'steps': a.steps, 'engines': {}}
    for name in engines:
        t = np.array(times[name])
        qps = Q[name] / (np.median(t) / 1e3)
        print('%-32s Q %d  median %.2f ms (min %.2f, max %.2f)  %.0f queries/s  guard-band recompute %d'
              % (name, Q[name], np.median(t), t.min(), t.max(), qps, guard[name]))
        result['engines'][name] = {'queries': Q[name], 'median_ms': float(np.median(t)), 'min_ms': float(t.min()),
                                   'max_ms': float(t.max()), 'queries_per_s': float(qps), 'guard_recompute': guard[name]}
    for eng in engines.values():
        eng.close()
    print(json.dumps(result))


if __name__ == '__main__':
    main()
