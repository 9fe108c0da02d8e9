"""Timing of the unsigned closest-point query (p2s_mesh_closest_point_dev) and of the ground-truth normals built on the
device primitives, one JSON line:
  - torus: 150 000 queries (half near the surface, half uniform) against the ~56k-face marching-cubes torus of
    tools/mesh_sdf_bench.py; ops.mesh_closest_point and ops.mesh_signed_distance on the same inputs, alternated in the
    same run, CUDA events, median of --reps (each call includes the face-index check and its read-back);
  - normals: eval_dataset.get_pts_normals on the three abc_minimal meshes (tests/golden/mesh_sdf.npz) at 100 000 samples
    per model, as eval_dataset.py runs it, with --pts points per cloud; wall clock of the whole stage (file reading and
    writing included, outputs removed before every rep) and CUDA-event time of the device part (eval_dataset.pts_normals).

    python tools/closest_point_bench.py [--reps 10] [--pts 20000]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from mesh_sdf_bench import torus_mesh, torus_queries  # noqa: E402
from points2surf_b200 import eval_dataset, make_dataset, mesh_io, ops  # noqa: E402


def event_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--pts', type=int, default=20000)
    a = ap.parse_args()
    dev = torch.device('cuda', 0)

    v, f, res = torus_mesh(dev)
    q = torus_queries(v, f, np.random.RandomState(0))
    vt, ft, qt = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev), torch.from_numpy(q).to(dev)
    closest = lambda: ops.mesh_closest_point(vt, ft, qt)          # noqa: E731
    signed = lambda: ops.mesh_signed_distance(vt, ft, qt)         # noqa: E731
    closest()
    signed()
    torch.cuda.synchronize()
    t_cp, t_sd = [], []
    for _ in range(a.reps):
        t_cp.append(event_ms(closest))
        t_sd.append(event_ms(signed))
    cp_ms, sd_ms = float(np.median(t_cp)), float(np.median(t_sd))

    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'mesh_sdf.npz'))
    tmp = tempfile.mkdtemp()
    try:
        root = os.path.join(tmp, 'ds')
        os.makedirs(os.path.join(root, '03_meshes'))
        os.makedirs(os.path.join(root, '04_pts'))
        clouds = []
        for i in range(3):
            stem = str(g['name_%d' % i])[:-4]
            mesh_file = os.path.join(root, '03_meshes', stem + '.ply')
            mesh_io.write_ply(mesh_file, g['verts_%d' % i], g['faces_%d' % i])
            pts = ops.mesh_sample(torch.from_numpy(g['verts_%d' % i]).to(dev), torch.from_numpy(g['faces_%d' % i]).to(dev),
                                  a.pts, seed=i).cpu().numpy()
            np.save(os.path.join(root, '04_pts', stem + '.xyz.npy'), pts)
            clouds.append((pts, g['verts_%d' % i], g['faces_%d' % i], make_dataset.filename_to_hash(mesh_file)))
        device_part = lambda: [eval_dataset.pts_normals(p, vv, ff, 100000, s) for p, vv, ff, s in clouds]   # noqa: E731
        device_part()
        dev_ms = float(np.median([event_ms(device_part) for _ in range(a.reps)]))
        stage_s = []
        for _ in range(max(1, a.reps // 3)):
            shutil.rmtree(os.path.join(root, '06_normals'), ignore_errors=True)
            torch.cuda.synchronize()
            t = time.perf_counter()
            eval_dataset.get_pts_normals(tmp, 'ds', '04_pts', '03_meshes', '06_normals', samples_per_model=100000)
            torch.cuda.synchronize()
            stage_s.append(time.perf_counter() - t)
    finally:
        shutil.rmtree(tmp)
    try:
        smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().split('\n')[0]
    except Exception:
        smi = 'unknown'
    print(json.dumps({
        'gpu': torch.cuda.get_device_name(dev), 'nvidia_smi_name_power_limit': smi,
        'torus': {'faces': int(len(f)), 'mc_res': res, 'queries': int(len(q)), 'closest_point_ms': round(cp_ms, 3),
                  'signed_distance_ms': round(sd_ms, 3), 'signed_over_closest': round(sd_ms / cp_ms, 3),
                  'closest_point_face_query_pairs_per_s': len(f) * len(q) / (cp_ms * 1e-3)},
        'normals': {'meshes': 3, 'faces': [int(len(g['faces_%d' % i])) for i in range(3)], 'pts_per_cloud': a.pts,
                    'samples_per_model': 100000, 'device_ms_all_three': round(dev_ms, 3),
                    'get_pts_normals_s_all_three': round(float(np.median(stage_s)), 3)},
        'reps': a.reps,
    }))


if __name__ == '__main__':
    main()
