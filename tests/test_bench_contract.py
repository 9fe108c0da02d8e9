"""bench.py contract checks that need no GPU: the reference arm prints one JSON line with the agreed keys, the GPU arm
refuses to run without a CUDA device (no silent CPU fallback)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_json_line():
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--impl', 'reference', '--steps', '1', '--warmup', '0',
                        '--cpu_sample', '16', '--grid_res', '32'], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().split('\n')[-1])
    assert line['impl'] == 'reference' and line['unit'] == 'queries/s' and line['higher_is_better'] is True
    assert line['value'] > 0 and line['n_gpus'] == 1 and line['steps'] == 1
    assert line['metric'].startswith('SDF queries/sec at grid_res=')
    assert 'workload' in line['config']
    cb = line['cpu_baseline']
    assert cb['kind'] == 'port' and cb['cores'] >= 1 and cb['value'] == line['value'] and 'queries' in cb['sample']
    e2e = line['e2e']
    assert e2e['value'] == line['value'] and e2e['h2d_bytes_per_step'] == 0 and e2e['d2h_bytes_per_step'] == 0


def test_b200_arm_fails_loudly_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        return   # on a GPU box the real arm is exercised by the driver
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--steps', '1', '--warmup', '3'], capture_output=True,
                       text=True, timeout=600, cwd=ROOT)
    assert r.returncode != 0 and 'no CPU fallback' in (r.stderr + r.stdout)
