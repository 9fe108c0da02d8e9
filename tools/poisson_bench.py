"""Times the screened Poisson reconstruction (csrc/poisson.cu + marching cubes) stage by stage with CUDA events, and
measures the Chamfer distance of SPSR with ground-truth normals on range scans of the abc_minimal meshes.

    python tools/poisson_bench.py [--out FILE.json]

Workloads: the three abc_minimal meshes scanned with their reference poses at the reference noise, with ground-truth
normals, at depth 8; a ~1M-point torus cloud at depths 8 and 9.  Each is run once to warm up, then 10 times; the median
of each stage is printed.  The Chamfer distance (the reference's definition, evaluation.mesh_comparison) is reported at
pointWeight 0 and 4, and the CPU oracle's time at depth 6 for scale."""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from oracle import poisson_oracle as po  # noqa: E402
from points2surf_b200 import eval_dataset, evaluation, mesh_io, ops, poisson, trafo  # noqa: E402
import poisson_cases as pc  # noqa: E402

STAGES = ('setup', 'rhs', 'solve', 'iso', 'mc')


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        import subprocess
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = 'unknown'
    return name, pl


def abc_scan(i):
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'scan.npz'))
    m = np.load(os.path.join(ROOT, 'tests', 'golden', 'mesh_sdf.npz'))
    name, v, f = str(m['name_%d' % i]), m['verts_%d' % i], m['faces_%d' % i]
    rot = np.stack([trafo.quaternion_matrix(q)[:3, :3] for q in g['rotations_%d' % i]])
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    pts = ops.range_scan(cu(v), cu(f), rot, g['locations_%d' % i], noise_sigma=float(g['sigma_%d' % i]),
                         seed=7)[0].cpu().numpy()
    return name, v, f, pts, eval_dataset.pts_normals(pts, v, f, 100000, i).astype(np.float32)


def time_workload(pts, nrm, depth, reps=10):
    poisson.reconstruct(pts, nrm, depth=depth)   # warm-up
    rows = []
    for _ in range(reps):
        _, _, rep = poisson.reconstruct(pts, nrm, depth=depth)
        rows.append(list(rep['stage_ms']) + [rep['mc_ms']])
    med = np.median(np.array(rows), axis=0)
    out = {s: round(float(x), 3) for s, x in zip(STAGES, med)}
    out['total'] = round(float(np.median(np.array(rows).sum(1))), 3)
    out.update(points=len(pts), depth=depth, iterations=rep['iterations'], residual=rep['residual'])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    name, pl = gpu_info()
    res = {'gpu': name, 'power_limit': pl, 'workloads': [], 'chamfer': []}
    print('GPU: %s, power limit %s; CUDA events, median of 10 after one warm-up' % (name, pl))
    with tempfile.TemporaryDirectory() as tmp:
        for i in range(3):
            mname, v, f, pts, nrm = abc_scan(i)
            r = time_workload(pts, nrm, 8)
            r['name'] = mname
            res['workloads'].append(r)
            print(json.dumps(r))
            ref = os.path.join(tmp, 'ref.ply')
            mesh_io.write_ply(ref, v, f)
            for pw in (0.0, 4.0):
                rv, rf, rep = poisson.reconstruct(pts, nrm, depth=8, point_weight=pw)
                rec = os.path.join(tmp, 'rec.ply')
                mesh_io.write_ply(rec, rv, rf)
                c = evaluation._chamfer_distance_single_file(rec, ref, 10000)[2]
                row = dict(name=mname, point_weight=pw, chamfer=c, iterations=rep['iterations'],
                           residual=rep['residual'])
                res['chamfer'].append(row)
                print(json.dumps(row))
    tp, tn = pc.torus(1000000, seed=5)
    for depth in (8, 9):
        r = time_workload(tp, tn, depth)
        r['name'] = 'torus_1M'
        res['workloads'].append(r)
        print(json.dumps(r))
    sp, sn = pc.sphere(20000, seed=1)
    t0 = time.perf_counter()
    po.solve(sp, sn, 6)
    res['oracle_cpu_s_depth6'] = round(time.perf_counter() - t0, 2)
    print('CPU oracle, 20k-point sphere at depth 6: %.2f s' % res['oracle_cpu_s_depth6'])
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as fp:
            json.dump(res, fp, indent=1)


if __name__ == '__main__':
    main()
