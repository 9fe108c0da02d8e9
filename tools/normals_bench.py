"""Times the oriented point normals (csrc/normals.cu) stage by stage with CUDA events and measures what they are worth to
the Screened Poisson baseline.

    python tools/normals_bench.py [--out FILE.json] [--big 1000000]

Workloads: range scans of the three abc_minimal meshes (reference poses and noise), a 150 000-point and a `--big`-point
noisy torus (synth.make_cloud).  Per workload one warm-up, then 10 runs with a 256 MB buffer overwritten before each (the
L2 cache starts cold): the median of a (cell index + neighbours), b (plane fit), c (orientation), their sum, and of c
alone through ops.orient_normals; Boruvka rounds and sweeps; the fraction of normals that agree in sign with the
ground-truth / analytic normal.  For the scans also the Chamfer distance (evaluation.mesh_comparison's definition) of the
Poisson surface from the estimated normals next to the one from ground-truth normals, and for scale the device time of the
exhaustive neighbour search (ops.knn_patch, the cloud as its own query set) on the first scan.  Fails without a GPU."""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from points2surf_b200 import evaluation, mesh_io, ops, poisson, synth  # noqa: E402
from poisson_bench import abc_scan, gpu_info  # noqa: E402

K = 10


def torus_normals(pts):
    """outward normal of synth's torus (ring radius 0.45 around z) at the points' projections"""
    ring = pts[:, :2] / np.linalg.norm(pts[:, :2], axis=1, keepdims=True) * 0.45
    d = pts - np.concatenate([ring, np.zeros((len(pts), 1))], 1)
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def time_workload(pts, ref, reps=10):
    p = torch.from_numpy(np.ascontiguousarray(pts, np.float32)).cuda()
    flush = torch.empty(64 << 20, dtype=torch.float32, device='cuda')
    rows, alone = [], []
    for rep in range(reps + 1):
        flush.zero_()
        n, ids, st = ops.point_normals(p, k=K, return_neighbours=True, return_stats=True)
        flush.zero_()
        _, st_c = ops.orient_normals(p, n, ids, return_stats=True)      # oriented normals are valid input of c as well
        if rep:
            rows.append(st['stage_ms'])
            alone.append(st_c['stage_ms'][2])
    med = np.median(np.array(rows), axis=0)
    agree = float((np.einsum('ij,ij->i', n.cpu().numpy().astype(np.float64), ref) > 0).mean())
    return dict(points=len(pts), k=K, neighbours_ms=round(float(med[0]), 3), fit_ms=round(float(med[1]), 3),
                orient_ms=round(float(med[2]), 3), total_ms=round(float(np.median(np.array(rows).sum(1))), 3),
                orient_alone_ms=round(float(np.median(alone)), 3), rounds=st['rounds'], sweeps=st['sweeps'],
                components=st['components'], degenerate=st['degenerate'], sign_agreement=round(agree, 5)), n.cpu().numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--big', type=int, default=1000000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('normals_bench needs a CUDA device')
    name, pl = gpu_info()
    res = {'gpu': name, 'power_limit': pl, 'workloads': [], 'chamfer': []}
    print('GPU: %s, power limit %s; CUDA events, cold L2, median of 10 after one warm-up, K = %d' % (name, pl, K))
    with tempfile.TemporaryDirectory() as tmp:
        for i in range(3):
            mname, v, f, pts, gt = abc_scan(i)
            r, est = time_workload(pts, gt.astype(np.float64))
            r['name'] = mname
            res['workloads'].append(r)
            print(json.dumps(r))
            ref = os.path.join(tmp, 'ref.ply')
            mesh_io.write_ply(ref, v, f)
            row = dict(name=mname)
            for label, nrm in (('estimated', est), ('ground_truth', gt)):
                rv, rf, _ = poisson.reconstruct(pts, nrm, depth=8)
                rec = os.path.join(tmp, 'rec.ply')
                mesh_io.write_ply(rec, rv, rf)
                row['chamfer_' + label] = evaluation._chamfer_distance_single_file(rec, ref, 10000)[2]
            res['chamfer'].append(row)
            print(json.dumps(row))
            if i == 0:
                p = torch.from_numpy(pts).cuda()
                ops.knn_patch(p, p, K)
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                ev[0].record()
                ops.knn_patch(p, p, K)
                ev[1].record()
                torch.cuda.synchronize()
                res['exhaustive_knn_ms'] = dict(name=mname, points=len(pts), ms=round(ev[0].elapsed_time(ev[1]), 3))
                print(json.dumps(res['exhaustive_knn_ms']))
    for n in (150000, args.big):
        pts = synth.make_cloud('torus', n, seed=4)
        r, _ = time_workload(pts, torus_normals(pts.astype(np.float64)))
        r['name'] = 'torus_%d' % n
        res['workloads'].append(r)
        print(json.dumps(r))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as fp:
            json.dump(res, fp, indent=1)


if __name__ == '__main__':
    main()
