"""Timing of the training-target signed distance (p2s_mesh_signed_distance_dev), one JSON line:
  - fixture: the three abc_minimal meshes (2.9k-16k faces) x their 2 000 query points each (tests/golden/mesh_sdf.npz),
    the size make_dataset writes per shape;
  - large: ~150k queries (half near the surface, half uniform in the unit cube) against a ~50k-face marching-cubes torus,
    make_dataset's face cap for training meshes (make_dataset.py:796).
CUDA-event times after warm-up (median of --reps; each call includes the face-index check and its read-back).
The CPU figure is the float64 NumPy oracle (oracle/mesh_sdf_oracle.py) on a query sample, labelled as such.

    python tools/mesh_sdf_bench.py [--reps 10] [--cpu_sample 200]
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
from oracle import mesh_sdf_oracle as msdf  # noqa: E402
from points2surf_b200 import ops, sdf  # noqa: E402


def torus_mesh(dev, min_faces=45000):
    for res in range(120, 400, 8):
        x = torch.linspace(-1, 1, res, device=dev)
        X, Y, Z = torch.meshgrid(x, x, x, indexing='ij')
        vol = 0.25 - torch.sqrt((torch.sqrt(X * X + Y * Y) - 0.55) ** 2 + Z * Z)
        v, f = ops.marching_cubes(vol.contiguous(), 0.0)
        if f.shape[0] >= min_faces:
            v, f = v.cpu().numpy(), f.cpu().numpy()
            return v, sdf._orient_outward(v, f), res
    raise RuntimeError('no torus mesh with %d faces' % min_faces)


def torus_queries(v, f, rng, n=150000):
    """n queries, half within the patch radius 6/256 of the surface, half uniform in [-0.5, 0.5)^3"""
    n_near = n // 2
    fi = rng.choice(len(f), n_near)
    r = rng.uniform(0, 1, (n_near, 2))
    r[r.sum(1) > 1] = 1 - r[r.sum(1) > 1]
    va, vb, vc = v[f[fi, 0]], v[f[fi, 1]], v[f[fi, 2]]
    near = va + r[:, :1] * (vb - va) + r[:, 1:] * (vc - va) + rng.uniform(-6 / 256, 6 / 256, (n_near, 1)) * \
        np.cross(vb - va, vc - va) / (np.linalg.norm(np.cross(vb - va, vc - va), axis=1, keepdims=True) + 1e-30)
    return np.concatenate([near, rng.uniform(-0.5, 0.5, (n - n_near, 3))]).astype(np.float32)


def time_calls(calls, reps):
    for c in calls:
        c()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for c in calls:
            c()
        e.record()
        e.synchronize()
        ms.append(s.elapsed_time(e))
    return float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--cpu_sample', type=int, default=200)
    a = ap.parse_args()
    dev = torch.device('cuda', 0)
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'mesh_sdf.npz'))
    fixture = [(torch.from_numpy(g['verts_%d' % i]).to(dev), torch.from_numpy(g['faces_%d' % i]).to(dev),
                torch.from_numpy(g['ref_query_pts_%d' % i]).to(dev)) for i in range(3)]
    fix_ms = time_calls([lambda m=m: ops.mesh_signed_distance(*m) for m in fixture], a.reps)
    fix_q = sum(int(m[2].shape[0]) for m in fixture)
    fix_pairs = sum(int(m[1].shape[0]) * int(m[2].shape[0]) for m in fixture)

    v, f, res = torus_mesh(dev)
    rng = np.random.RandomState(0)
    q = torus_queries(v, f, rng)
    vt, ft, qt = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev), torch.from_numpy(q).to(dev)
    big_ms = time_calls([lambda: ops.mesh_signed_distance(vt, ft, qt)], a.reps)

    cpu = {}
    if a.cpu_sample > 0:
        sel = rng.choice(len(q), a.cpu_sample, replace=False)
        t = time.perf_counter()
        msdf.mesh_signed_distance(v, f, q[sel])
        cpu['large_queries_per_s'] = a.cpu_sample / (time.perf_counter() - t)
        t = time.perf_counter()
        msdf.mesh_signed_distance(g['verts_0'], g['faces_0'], g['ref_query_pts_0'][:a.cpu_sample])
        cpu['fixture0_queries_per_s'] = a.cpu_sample / (time.perf_counter() - t)
    try:
        smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().split('\n')[0]
    except Exception:
        smi = 'unknown'
    print(json.dumps({
        'gpu': torch.cuda.get_device_name(dev), 'nvidia_smi_name_power_limit': smi,
        'fixture': {'meshes': 3, 'faces': [int(m[1].shape[0]) for m in fixture], 'queries': fix_q,
                    'ms_all_three': round(fix_ms, 3), 'face_query_pairs_per_s': fix_pairs / (fix_ms * 1e-3)},
        'large': {'faces': int(len(f)), 'mc_res': res, 'queries': int(len(q)), 'ms': round(big_ms, 3),
                  'queries_per_s': len(q) / (big_ms * 1e-3), 'face_query_pairs_per_s': len(f) * len(q) / (big_ms * 1e-3)},
        'cpu_baseline': dict(label='float64 NumPy oracle, one process, %d-query sample' % a.cpu_sample, **cpu),
        'reps': a.reps,
    }))


if __name__ == '__main__':
    main()
