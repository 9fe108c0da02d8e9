"""Timing of the simulated range scans (p2s_range_scan_dev), one JSON line:
  - fixture: the three abc_minimal meshes (2.9k-16k faces) with the reference's scan poses (tests/golden/scan.npz,
    17-28 scans of 176 x 144 rays each), what make_dataset --scan casts per shape;
  - large: a ~50k-face marching-cubes torus (make_dataset's face cap for training meshes, make_dataset.py:796) x 30
    scans with the poses of the first fixture mesh repeated.
CUDA-event times after warm-up (median of --reps; each call includes the face-index check and the two count
read-backs).  Rays cast = the rays that survive the bounding-box cull (counted on the host with the oracle's box test,
which is the kernel's); ray-triangle tests = rays cast x faces.

    python tools/scan_bench.py [--reps 10]
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
from oracle import scan_oracle as so  # noqa: E402
from points2surf_b200 import ops, sdf, trafo  # noqa: E402
from mesh_sdf_bench import time_calls, torus_mesh  # noqa: E402


def rays_cast(v, rot, loc):
    return int(sum(len(so.box_survivors(v, *so.scanner_rays(R, l))) for R, l in zip(rot, loc)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    a = ap.parse_args()
    dev = torch.device('cuda', 0)
    gm = np.load(os.path.join(ROOT, 'tests', 'golden', 'mesh_sdf.npz'))
    gs = np.load(os.path.join(ROOT, 'tests', 'golden', 'scan.npz'))
    fixture = []
    for i in range(3):
        rot = np.stack([trafo.quaternion_matrix(q)[:3, :3] for q in gs['rotations_%d' % i]])
        loc = gs['locations_%d' % i]
        v, f = gm['verts_%d' % i], gm['faces_%d' % i]
        fixture.append(dict(v=torch.from_numpy(v).to(dev), f=torch.from_numpy(f).to(dev), rot=rot, loc=loc,
                            sigma=float(gs['sigma_%d' % i]), faces=len(f), scans=len(loc), rays=rays_cast(v, rot, loc)))
    per = []
    for m in fixture:
        ms = time_calls([lambda m=m: ops.range_scan(m['v'], m['f'], m['rot'], m['loc'], noise_sigma=m['sigma'])], a.reps)
        hits = int(ops.range_scan(m['v'], m['f'], m['rot'], m['loc'])[3].sum())
        per.append({'faces': m['faces'], 'scans': m['scans'], 'rays_cast': m['rays'], 'hits': hits, 'ms': round(ms, 3),
                    'ray_triangle_tests_per_s': m['rays'] * m['faces'] / (ms * 1e-3)})

    v, f, res = torus_mesh(dev)
    rot = np.concatenate([fixture[0]['rot']] * 2)[:30]
    loc = np.concatenate([fixture[0]['loc']] * 2)[:30]
    vt, ft = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)
    big_ms = time_calls([lambda: ops.range_scan(vt, ft, rot, loc, noise_sigma=0.01)], a.reps)
    big_rays = rays_cast(v, rot, loc)
    big_hits = int(ops.range_scan(vt, ft, rot, loc)[3].sum())
    try:
        smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().split('\n')[0]
    except Exception:
        smi = 'unknown'
    print(json.dumps({
        'gpu': torch.cuda.get_device_name(dev), 'nvidia_smi_name_power_limit': smi,
        'fixture': per, 'fixture_ms_all_three': round(sum(p['ms'] for p in per), 3),
        'large': {'faces': int(len(f)), 'mc_res': res, 'scans': len(loc), 'rays_total': len(loc) * 176 * 144,
                  'rays_cast': big_rays, 'hits': big_hits, 'ms': round(big_ms, 3),
                  'ray_triangle_tests_per_s': big_rays * len(f) / (big_ms * 1e-3)},
        'reps': a.reps,
    }))


if __name__ == '__main__':
    main()
