"""Timing of the DeepSDF input stage per mesh, one JSON line:
  - repair: p2s_mesh_repair_dev (ops.mesh_repair, hole_filling_mesh_simp.mlx's defaults);
  - far sdf: the far samples' signed distances on the repaired mesh (ops.mesh_signed_distance), int(2 N * 0.2) points
    for an N-point cloud (N = --points, 150 000 by default).
Meshes: the three abc_minimal meshes (tests/golden/mesh_sdf.npz) with 8 deleted patches of 5 faces each, and a
marching-cubes torus of >= --min_faces faces with 200 such patches.  CUDA-event times after warm-up, median of --reps;
each repair includes the read-backs of its intermediate counts.

    python tools/deepsdf_bench.py [--reps 10] [--min_faces 1000000] [--points 150000]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from points2surf_b200 import ops  # noqa: E402
from mesh_sdf_bench import time_calls  # noqa: E402
import mesh_repair_cases as mrc  # noqa: E402


def torus(dev, min_faces):
    for res in range(200, 1200, 40):
        x = torch.linspace(-1, 1, res, device=dev)
        X, Y, Z = torch.meshgrid(x, x, x, indexing='ij')
        vol = (0.25 - torch.sqrt((torch.sqrt(X * X + Y * Y) - 0.55) ** 2 + Z * Z)).contiguous()
        del X, Y, Z
        v, f = ops.marching_cubes(vol, 0.0)
        del vol
        if f.shape[0] >= min_faces:
            return v.cpu().numpy() * 0.5, f.cpu().numpy(), res
    raise RuntimeError('no torus mesh with %d faces' % min_faces)


def measure(dev, v, f, n_far, reps):
    vt, ft = torch.from_numpy(v).to(dev), torch.from_numpy(np.ascontiguousarray(f)).to(dev)
    repair_ms = time_calls([lambda: ops.mesh_repair(vt, ft)], reps)
    vr, fr, st = ops.mesh_repair(vt, ft)
    q = torch.rand((n_far, 3), generator=torch.Generator(device=dev).manual_seed(0), device=dev) - 0.5
    sdf_ms = time_calls([lambda: ops.mesh_signed_distance(vr, fr, q)], reps)
    return {'faces_in': int(len(f)), 'faces_out': int(fr.shape[0]), 'holes_closed': st['holes_closed'],
            'holes_left_open': st['holes_left_open'], 'repair_ms': round(repair_ms, 3), 'far_samples': n_far,
            'far_sdf_ms': round(sdf_ms, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--min_faces', type=int, default=1000000)
    ap.add_argument('--points', type=int, default=150000)
    a = ap.parse_args()
    dev = torch.device('cuda', 0)
    n_far = int(2 * a.points * 0.2)
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'mesh_sdf.npz'))
    out = {'abc_minimal': []}
    for i in range(3):
        f = mrc.delete_random_faces(g['faces_%d' % i], seed=i, n_sets=8, size=5)
        out['abc_minimal'].append(measure(dev, g['verts_%d' % i].astype(np.float32), f, n_far, a.reps))
    v, f, res = torus(dev, a.min_faces)
    out['torus'] = dict(measure(dev, v, mrc.delete_random_faces(f, seed=0, n_sets=200, size=5), n_far, a.reps), mc_res=res)
    try:
        smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().split('\n')[0]
    except Exception:
        smi = 'unknown'
    print(json.dumps(dict(out, gpu=torch.cuda.get_device_name(dev), nvidia_smi_name_power_limit=smi, reps=a.reps)))


if __name__ == '__main__':
    main()
