"""Times the stages of make_dataset --gt_recon with CUDA events and measures where the reconstruction error of the
volume stage comes from, on range scans of the abc_minimal meshes.

    python tools/gt_recon_bench.py [--res 256] [--out FILE.json]

Workload: the three abc_minimal meshes (tests/golden/mesh_sdf.npz) scanned at their reference poses and noise
(tests/golden/scan.npz, as in tools/poisson_bench.py), the reconstruction grid of the scan at res 256, eps 3.  Stages:
the ground-truth signed distances at the grid queries (ops.mesh_signed_distance), the inside kernel
(ops.mesh_inside_grid), sign propagation (ops.sdf_to_volume, sigma 5, certainty threshold 13) and marching cubes on the
propagated and on the exact-sign volume.  Each is run once to warm up, then 10 times; the median is printed.  Chamfer
distances (the reference's definition, evaluation._chamfer_distance_single_file, 10 000 samples) of both meshes against
the ground-truth mesh, and the number of voxels whose propagated sign differs from the exact sign."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from points2surf_b200 import evaluation, make_dataset, mesh_io, ops, sdf, trafo  # noqa: E402


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = 'unknown'
    return name, pl


def timed(fn, reps=10):
    """-> (result of the last call, median ms over reps after one warm-up)"""
    out = fn()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return out, round(float(np.median(ms)), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--res', type=int, default=256)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    res, eps, sigma, thr = args.res, 3, 5, 13.0
    name, pl = gpu_info()
    result = {'gpu': name, 'power_limit': pl, 'res': res, 'eps': eps, 'sigma': sigma, 'certainty_threshold': thr,
              'shapes': []}
    print('GPU: %s, power limit %s; CUDA events, median of 10 after one warm-up' % (name, pl))
    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'scan.npz'))
    m = np.load(os.path.join(ROOT, 'tests', 'golden', 'mesh_sdf.npz'))
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    with tempfile.TemporaryDirectory() as tmp:
        for i in range(3):
            mname, v, f = str(m['name_%d' % i]), m['verts_%d' % i], m['faces_%d' % i]
            rot = np.stack([trafo.quaternion_matrix(q)[:3, :3] for q in g['rotations_%d' % i]])
            vc, fc = cu(v), cu(sdf._orient_outward(v, f))
            pts = ops.range_scan(vc, fc, rot, g['locations_%d' % i], noise_sigma=float(g['sigma_%d' % i]), seed=7)[0]
            lin = ops.query_grid(pts, res, eps)
            q = ops.query_points(lin, res)
            dist, t_sdf = timed(lambda: ops.mesh_signed_distance(vc, fc, q))
            d = dist.double()
            d[torch.isnan(d)] = 0.0
            d[torch.isinf(d)] = 1.0
            dist = d.clamp(-1.0, 1.0).float()
            inside, t_inside = timed(lambda: ops.mesh_inside_grid(vc, fc, res))
            (prop, iters), t_prop = timed(lambda: ops.sdf_to_volume(lin, dist, res, sigma, thr))
            exact = make_dataset.exact_sign_volume(inside, lin, dist)
            (pv, pf), t_mc = timed(lambda: ops.marching_cubes(prop, 0.0))
            (ev, ef), t_mc_exact = timed(lambda: ops.marching_cubes(exact, 0.0))
            ref = os.path.join(tmp, 'ref.ply')
            mesh_io.write_ply(ref, v, f)
            chamfer = {}
            for key, (mv, mf) in (('mc_gt_recon', (pv, pf)), ('mc_gt_exact_sign', (ev, ef))):
                rec = os.path.join(tmp, key + '.ply')
                mesh_io.write_ply(rec, mv.cpu().numpy(), mf.cpu().numpy())
                chamfer[key] = evaluation._chamfer_distance_single_file(rec, ref, 10000)[2]
            row = dict(name=mname, faces=len(f), points=len(pts), queries=len(lin), propagation_iterations=iters,
                       sign_mismatches=int(((prop > 0) != (exact > 0)).sum()), ms_signed_distance=t_sdf,
                       ms_inside=t_inside, ms_sign_propagation=t_prop, ms_marching_cubes=t_mc,
                       ms_marching_cubes_exact=t_mc_exact, chamfer=chamfer)
            result['shapes'].append(row)
            print(json.dumps(row))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as fp:
            json.dump(result, fp, indent=1)


if __name__ == '__main__':
    main()
