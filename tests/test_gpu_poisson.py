"""GPU tests of the screened Poisson reconstruction (p2s_poisson_solve_dev through ops.poisson_solve): against the
float64 oracle (oracle/poisson_oracle.py), mesh shape at depth 8, determinism, input errors, range scans of the
abc_minimal meshes with ground-truth normals, and eval_dataset's --spsr stage."""
import os

import numpy as np
import pytest
import torch

from oracle import poisson_oracle as po
from points2surf_b200 import eval_dataset, evaluation, mesh_io, ops, poisson, trafo
from points2surf_b200._lib import P2SError
from helpers import load_golden
import poisson_cases as pc
from test_gpu_eval_dataset import _dataset

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _mesh(i):
    g = load_golden('mesh_sdf.npz')
    return str(g['name_%d' % i]), g['verts_%d' % i], g['faces_%d' % i]


def _abc_samples(n, seed=0):
    """noisy samples of an abc_minimal mesh with eval_dataset's ground-truth normals"""
    _, v, f = _mesh(0)
    p = ops.mesh_sample(cu(v), cu(f), n, seed=seed).cpu().numpy()
    p += np.random.RandomState(seed).normal(0, 0.002, p.shape).astype(np.float32)
    return p, eval_dataset.pts_normals(p, v, f, 100000, seed).astype(np.float32)


def _cloud(kind, n=20000):
    if kind == 'sphere':
        return pc.sphere(n, seed=1)
    if kind == 'torus':
        return pc.torus(n, seed=2)
    return _abc_samples(n)


@pytest.mark.parametrize('depth', [5, 6])
@pytest.mark.parametrize('kind', ['sphere', 'torus', 'abc'])
def test_against_oracle(kind, depth):
    pts, nrm = _cloud(kind)
    vals, rep = ops.poisson_solve(cu(pts), cu(nrm), depth=depth)
    ref = po.solve(pts, nrm, depth)
    chi = rep['iso'] - vals.double().cpu().numpy().reshape(-1)
    rng = ref['chi'].max() - ref['chi'].min()
    err = np.abs(chi - ref['chi']).max() / rng
    print('%s d=%d: max|dchi|/range %.2e  |diso|/range %.2e  residual %.2e  iterations %d'
          % (kind, depth, err, abs(rep['iso'] - ref['iso']) / rng, rep['residual'], rep['iterations']))
    assert rep['residual'] <= 1e-5
    assert err <= 1e-4
    assert abs(rep['iso'] - ref['iso']) <= 1e-4 * rng
    assert np.allclose(rep['origin'], ref['origin'], rtol=0, atol=1e-12) and rep['edge'] == pytest.approx(ref['edge'], 1e-15)
    assert rep['occupied_cells'] == ref['occupied_cells'] and rep['dropped_points'] == 0
    assert rep['grid_res'] == 2 ** depth + 1 and rep['points_used'] == len(pts)


@pytest.mark.parametrize('kind', ['sphere', 'torus'])
def test_mesh_shape_depth8(kind):
    pts, nrm = _cloud(kind, 200000)
    v, f, rep = poisson.reconstruct(pts, nrm, depth=8)
    h = rep['edge'] / 256
    assert rep['residual'] <= 1e-5
    assert pc.closed_manifold(f)
    assert pc.euler_characteristic(v, f) == (2 if kind == 'sphere' else 0)
    assert pc.signed_volume(v, f) > 0
    if kind == 'sphere':
        err = np.abs(np.linalg.norm(v - pc.SPHERE_CENTER, axis=1) - pc.SPHERE_RADIUS)
    else:
        err = pc.torus_distance(v)
    print('%s d=8: mean error %.3f h, max %.3f h, %d iterations, residual %.2e'
          % (kind, err.mean() / h, err.max() / h, rep['iterations'], rep['residual']))
    if kind == 'sphere':
        assert err.mean() <= 0.25 * h and err.max() <= h


def test_deterministic_and_permutation_invariant():
    pts, nrm = _cloud('torus', 50000)
    a, ra = ops.poisson_solve(cu(pts), cu(nrm), depth=7)
    b, rb = ops.poisson_solve(cu(pts), cu(nrm), depth=7)
    assert torch.equal(a, b) and ra['iso'] == rb['iso'] and ra['iterations'] == rb['iterations']
    va, fa, _ = poisson.reconstruct(pts, nrm, depth=7)
    vb, fb, _ = poisson.reconstruct(pts, nrm, depth=7)
    assert np.array_equal(va, vb) and np.array_equal(fa, fb)
    perm = np.random.RandomState(0).permutation(len(pts))
    c, rc = ops.poisson_solve(cu(pts[perm]), cu(nrm[perm]), depth=7)
    chi_a = ra['iso'] - a.double()
    chi_c = rc['iso'] - c.double()
    assert float((chi_a - chi_c).abs().max()) <= 1e-5 * float(chi_a.max() - chi_a.min())


def test_bad_inputs_and_dropped_points():
    pts, nrm = pc.sphere(5000, seed=4)
    with pytest.raises(P2SError):
        ops.poisson_solve(cu(pts[:0]), cu(nrm[:0]), depth=5)
    for bad in (np.nan, np.inf):
        p = pts.copy()
        p[10, 1] = bad
        with pytest.raises(P2SError):
            ops.poisson_solve(cu(p), cu(nrm), depth=5)
        n = nrm.copy()
        n[20, 2] = bad
        with pytest.raises(P2SError):
            ops.poisson_solve(cu(pts), cu(n), depth=5)
    with pytest.raises(P2SError):
        ops.poisson_solve(cu(np.repeat(pts[:1], 100, 0)), cu(nrm[:100]), depth=5)
    for depth in (1, 10):
        with pytest.raises(P2SError):
            ops.poisson_solve(cu(pts), cu(nrm), depth=depth)
    with pytest.raises(P2SError):
        ops.poisson_solve(cu(pts), cu(np.zeros_like(nrm)), depth=5)
    n = nrm.copy()
    n[::7] = 0
    vals, rep = ops.poisson_solve(cu(pts), cu(n), depth=5)
    assert rep['dropped_points'] == len(pts[::7]) and rep['points_used'] == len(pts) - len(pts[::7])
    ref = po.solve(pts, n, 5)
    assert ref['dropped'] == rep['dropped_points']
    chi = rep['iso'] - vals.double().cpu().numpy().reshape(-1)
    assert np.abs(chi - ref['chi']).max() <= 1e-4 * (ref['chi'].max() - ref['chi'].min())


def _scan(i, noise):
    g = load_golden('scan.npz')
    name, v, f = _mesh(i)
    rot = np.stack([trafo.quaternion_matrix(q)[:3, :3] for q in g['rotations_%d' % i]])
    sigma = float(g['sigma_%d' % i]) if noise else 0.0
    noisy, _, _, _ = ops.range_scan(cu(v), cu(f), rot, g['locations_%d' % i], noise_sigma=sigma, seed=7)
    return name, v, f, noisy.cpu().numpy()


@pytest.mark.parametrize('noise', [False, True])
def test_scans_with_ground_truth_normals(tmp_path, noise):
    for i in range(3):
        name, v, f, pts = _scan(i, noise)
        nrm = eval_dataset.pts_normals(pts, v, f, 100000, i)
        rv, rf, rep = poisson.reconstruct(pts, nrm, depth=8)
        h = rep['edge'] / 256
        s = ops.mesh_sample(cu(rv), cu(rf), 20000, seed=1)
        _, d, _ = ops.mesh_closest_point(cu(v), cu(f), s)
        med = float(d.median())
        rec = str(tmp_path / ('rec_%d.ply' % i))
        ref = str(tmp_path / ('ref_%d.ply' % i))
        mesh_io.write_ply(rec, rv, rf)
        mesh_io.write_ply(ref, v, f)
        chamfer = evaluation._chamfer_distance_single_file(rec, ref, 10000)[2]
        print('%s noise=%s: %d points, median mesh->GT %.3f h, Chamfer %.5f, %d iterations'
              % (name, noise, len(pts), med / h, chamfer, rep['iterations']))
        assert rep['residual'] <= 1e-5
        if not noise:
            assert med <= 0.5 * h


def test_spsr_stage_of_eval_dataset(tmp_path, capsys):
    root = tmp_path / 'ds'
    names = _dataset(root)
    (root / 'valset.txt').write_text('\n'.join(names[:2]) + '\n')
    eval_dataset.main([str(root), '--spsr'])
    assert 'meshlabserver' not in capsys.readouterr().out
    plys = [root / '06_poisson_rec_gt_normals' / (s + '.ply') for s in names]
    for p in plys:
        v, f = mesh_io.read_ply(str(p))
        assert len(f) > 100 and pc.signed_volume(v, f) > 0
    lines = (root / 'comp_poisson_rec_gt_normals.csv').read_text().split('\n')
    assert lines[0].startswith('in mesh,ref mesh,Hausdorff dist new-ref')
    assert len(lines) == 3 and all(len(l.split(',')) == 6 and float(l.split(',')[-1]) > 0 for l in lines[1:])
    mtimes = [os.path.getmtime(str(p)) for p in plys]
    eval_dataset.main([str(root), '--spsr'])
    assert [os.path.getmtime(str(p)) for p in plys] == mtimes
