"""Timing of the mesh repair (p2s_mesh_clean_dev), one JSON line:
  - fixture: the three abc_minimal meshes (tests/golden/mesh_sdf.npz), already clean: the common case of the clean stage;
  - large: a >= 1M-face marching-cubes torus as a triangle soup (as read from an STL) with a third of its faces reversed,
    so every step runs at the size of the largest evaluation meshes (cleaned with no face cap).
CUDA-event times after warm-up, median of --reps; each call includes the read-backs of its intermediate counts.
The CPU figure is the float64 NumPy oracle (oracle/mesh_clean_oracle.py) on the same inputs, labelled as such.

    python tools/mesh_clean_bench.py [--reps 10] [--min_faces 1000000]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import mesh_clean_oracle as mco  # noqa: E402
from points2surf_b200 import ops, sdf  # noqa: E402
from mesh_sdf_bench import time_calls  # noqa: E402


def torus_soup(dev, min_faces):
    for res in range(400, 1200, 40):
        x = torch.linspace(-1, 1, res, device=dev)
        X, Y, Z = torch.meshgrid(x, x, x, indexing='ij')
        vol = (0.25 - torch.sqrt((torch.sqrt(X * X + Y * Y) - 0.55) ** 2 + Z * Z)).contiguous()
        del X, Y, Z
        v, f = ops.marching_cubes(vol, 0.0)
        del vol
        if f.shape[0] >= min_faces:
            v, f = v.cpu().numpy(), f.cpu().numpy()
            f = sdf._orient_outward(v, f).copy()
            rows = np.random.RandomState(0).choice(len(f), len(f) // 3, replace=False)
            f[rows] = f[rows][:, ::-1]
            return np.ascontiguousarray(v[f].reshape(-1, 3)), np.arange(3 * len(f), dtype=np.int32).reshape(-1, 3), res
    raise RuntimeError('no torus mesh with %d faces' % min_faces)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--min_faces', type=int, default=1000000)
    a = ap.parse_args()
    dev = torch.device('cuda', 0)
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'mesh_sdf.npz'))
    fixture = [(g['verts_%d' % i].astype(np.float32), g['faces_%d' % i].astype(np.int32)) for i in range(3)]
    fixture_dev = [(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)) for v, f in fixture]
    fix_ms = time_calls([lambda m=m: ops.mesh_clean(*m) for m in fixture_dev], a.reps)

    v, f, res = torus_soup(dev, a.min_faces)
    vt, ft = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)
    big_ms = time_calls([lambda: ops.mesh_clean(vt, ft)], a.reps)
    _, fo, rep = ops.mesh_clean(vt, ft)

    t = time.perf_counter()
    for m in fixture:
        mco.mesh_clean(*m)
    cpu_fix = time.perf_counter() - t
    t = time.perf_counter()
    _, _, rep_cpu = mco.mesh_clean(v, f)
    cpu_big = time.perf_counter() - t
    try:
        smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().split('\n')[0]
    except Exception:
        smi = 'unknown'
    nf = sum(len(m[1]) for m in fixture)
    print(json.dumps({
        'gpu': torch.cuda.get_device_name(dev), 'nvidia_smi_name_power_limit': smi,
        'fixture': {'meshes': 3, 'faces': [int(len(m[1])) for m in fixture], 'ms_all_three': round(fix_ms, 3),
                    'faces_per_s': nf / (fix_ms * 1e-3)},
        'large': {'faces_in': int(len(f)), 'vertices_in': int(len(v)), 'mc_res': res, 'ms': round(big_ms, 3),
                  'faces_per_s': len(f) / (big_ms * 1e-3), 'faces_out': int(fo.shape[0]),
                  'faces_reversed': rep['faces_reversed'], 'watertight': rep['watertight'],
                  'winding_consistent': rep['winding_consistent'], 'report_equals_oracle': rep == rep_cpu},
        'cpu_baseline': {'label': 'float64 NumPy oracle, one process, same inputs',
                         'fixture_s': round(cpu_fix, 3), 'fixture_faces_per_s': nf / cpu_fix,
                         'large_s': round(cpu_big, 3), 'large_faces_per_s': len(f) / cpu_big},
        'reps': a.reps,
    }))


if __name__ == '__main__':
    main()
