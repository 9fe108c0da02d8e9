"""GPU tests of the oriented point normals (ops.point_normals / ops.orient_normals) against oracle/normals_oracle.py, and
of the mesh-less path make_pc_dataset -> eval_dataset --spsr_estimated_normals."""
import os

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from oracle import normals_oracle as no
from points2surf_b200 import eval_dataset, make_pc_dataset, mesh_io, ops
import poisson_cases as pc
from test_gpu_mesh_sdf import _fixture, _mc_mesh, cu

pytestmark = pytest.mark.gpu


def _abc_cloud(i, n_pts=4000):
    """the noisy cloud test_gpu_eval_dataset._dataset samples from the i-th abc_minimal mesh"""
    fx = _fixture(i)
    pts = ops.mesh_sample(cu(fx['verts']), cu(fx['faces']), n_pts, seed=100 + i).cpu().numpy()
    return pts + np.random.RandomState(i).normal(0, 0.002, pts.shape).astype(np.float32)


def _two_spheres():
    a, _ = pc.sphere(3000, seed=2)
    return np.concatenate([a, a * np.float32(0.5) + np.float32([3, 0, 0])]).astype(np.float32)


def _box(n=6000, seed=0):
    """points on the faces of an axis-aligned cube: almost every plane fit is an axis, so edge costs are 0 or 1 and tie"""
    rs = np.random.RandomState(seed)
    uv = rs.uniform(-0.5, 0.5, (n, 2)).astype(np.float32)
    face = rs.randint(0, 6, n)
    pts = np.empty((n, 3), np.float32)
    for f in range(6):
        m = face == f
        axis, side = f // 2, np.float32(0.5 if f % 2 else -0.5)
        pts[m, axis] = side
        pts[np.ix_(m, [a for a in range(3) if a != axis])] = uv[m]
    return pts


def _cloud(name):
    if name == 'sphere':
        return pc.sphere(5000, seed=1)[0]
    if name == 'torus':
        return pc.torus(5000, seed=1)[0]
    if name == 'two':
        return _two_spheres()
    if name == 'box':
        return _box()
    return _abc_cloud(int(name[3:]))


def _fit(pts, k=10):
    """the kernel's unoriented plane fit and neighbour ids: the pre-sign rule applied to a viewpoint-oriented result"""
    n, ids = ops.point_normals(cu(pts), k=k, mode='viewpoint', viewpoint=(0, 0, 9), return_neighbours=True)
    return no.presign(n.cpu().numpy()), ids.cpu().numpy()


@pytest.mark.parametrize('n,k', [(2000, 3), (20000, 10), (100000, 16), (5000, 64)])
def test_neighbours_are_ckdtrees(n, k):
    pts = pc.torus(n, seed=k)[0]
    pts[-50:] = pts[:50]                                   # exact duplicates: ties resolved by id
    _, ids = ops.point_normals(cu(pts), k=k, return_neighbours=True)
    ids = ids.cpu().numpy()
    assert np.array_equal(ids, no.neighbours(pts, k))
    d, _ = cKDTree(pts.astype(np.float64)).query(pts.astype(np.float64), k=k)
    assert np.array_equal(np.sqrt(no.dist2(pts[ids], pts[:, None, :])), d)


@pytest.mark.parametrize('name', ['sphere', 'box', 'abc0'])
def test_plane_fit_matches_eigh(name):
    pts = _cloud(name)
    if name == 'sphere':                                   # a duplicate cluster and a collinear run: degenerate fits
        pts = np.concatenate([pts, np.repeat(np.float32([[5, 5, 5]]), 12, 0),
                              np.stack([np.linspace(8, 9, 40), np.zeros(40), np.zeros(40)], 1).astype(np.float32)])
    fit, ids = _fit(pts)
    ref, gap = no.plane_fit(pts, ids)
    assert np.array_equal(np.any(fit != 0, 1), np.any(ref != 0, 1))
    if name == 'sphere':
        assert (fit[5000:] == 0).all()
    ok = np.any(ref != 0, 1) & (gap > 1e-6)
    assert ok.mean() > 0.9
    sin = np.linalg.norm(np.cross(fit[ok].astype(np.float64), ref[ok].astype(np.float64)), axis=1)
    assert sin.max() <= 1e-5
    assert np.abs(np.linalg.norm(fit[ok], axis=1) - 1).max() <= 1e-6
    # the pre-sign rule holds on the kernel's own output, and picks the oracle's sign wherever the leading axis is clear
    assert np.array_equal(no.presign(fit), fit)
    mag = np.sort(np.abs(ref[ok]), axis=1)
    clear = mag[:, 2] - mag[:, 1] > 1e-5
    assert (np.einsum('ij,ij->i', fit[ok][clear], ref[ok][clear]) > 0).all()


@pytest.mark.parametrize('name', ['sphere', 'torus', 'two', 'box', 'abc0', 'abc1', 'abc2'])
def test_orientation_is_the_oracles_bit_for_bit(name):
    pts = _cloud(name)
    fit, ids = _fit(pts)
    out, parents, stats = ops.orient_normals(cu(pts), cu(fit), cu(ids), return_parents=True, return_stats=True)
    ref, ref_parents, ref_stats = no.orient(pts, fit, ids)
    assert np.array_equal(out.cpu().numpy(), ref)
    assert np.array_equal(parents.cpu().numpy(), ref_parents)
    for key in ('components', 'degenerate', 'flipped'):
        assert stats[key] == ref_stats[key], key
    assert 1 <= stats['rounds'] <= int(np.ceil(np.log2(len(pts)))) + 1 and stats['sweeps'] % 64 == 0
    print('%s: %d points, %d components, %d Boruvka rounds, %d sweeps' % (name, len(pts), stats['components'],
                                                                          stats['rounds'], stats['sweeps']))
    if name == 'two':
        assert stats['components'] == 2
    # the fused entry point gives the same, again, and on another stream
    full = ops.point_normals(cu(pts)).cpu().numpy()
    assert np.array_equal(full, ref)
    with torch.cuda.stream(torch.cuda.Stream()):
        again = ops.point_normals(cu(pts))
        out2 = ops.orient_normals(cu(pts), cu(fit), cu(ids))
    torch.cuda.synchronize()
    assert np.array_equal(again.cpu().numpy(), ref) and np.array_equal(out2.cpu().numpy(), ref)


def test_analytic_surfaces_point_outward():
    for kind in ('sphere', 'torus'):
        pts, ref = getattr(pc, kind)(20000, seed=3)
        n = ops.point_normals(cu(pts)).cpu().numpy()
        assert (np.einsum('ij,ij->i', n, ref) > 0).all()


@pytest.mark.parametrize('i', [0, 1, 2])
def test_orientation_quality_on_scan_like_clouds(i):
    fx = _fixture(i)
    pts = _abc_cloud(i)
    gt = eval_dataset.pts_normals(pts, fx['verts'], fx['faces'], 100000, seed=i)
    n = ops.point_normals(cu(pts)).cpu().numpy().astype(np.float64)
    frac = float((np.einsum('ij,ij->i', n, gt) > 0).mean())
    print('abc_minimal %d: %.4f of the estimated normals agree in sign with the ground truth' % (i, frac))
    assert frac > QUALITY_FLOOR[i]


# measured 0.5948, 0.9650, 0.7035 (NVIDIA H100 80GB HBM3; the result is a function of the input, so the margin is for the
# sampler only).  Hoppe's propagation crosses sharp edges and thin walls of these CAD parts with the wrong sign.
QUALITY_FLOOR = [0.55, 0.93, 0.65]


def test_viewpoint_mode():
    pts = _cloud('abc1')
    view = (0.3, -2.0, 1.5)
    n, stats = ops.point_normals(cu(pts), mode='viewpoint', viewpoint=view, return_stats=True)
    n = n.cpu().numpy()
    ref, _ = no.point_normals(pts, 10, mode='viewpoint', viewpoint=view)
    d = np.einsum('ij,ij->i', n.astype(np.float64), np.asarray(view)[None] - pts.astype(np.float64))
    assert (d >= 0).all() and stats['rounds'] == 0
    fit, _ = _fit(pts)
    assert np.array_equal(np.abs(n), np.abs(fit))
    same = np.abs(n - ref).max(1) < 1e-5
    assert same.mean() > 0.999


def test_errors_write_nothing_and_leave_the_device_usable():
    pts = cu(pc.sphere(500, seed=0)[0])
    bad = pts.clone()
    bad[7, 1] = float('nan')
    with pytest.raises(ops.P2SError, match='K must be'):
        ops.point_normals(pts, k=2)
    with pytest.raises(ops.P2SError, match='K must be'):
        ops.point_normals(pts, k=65)
    with pytest.raises(ops.P2SError, match='N > K'):
        ops.point_normals(pts[:10], k=10)
    with pytest.raises(ops.P2SError, match='non-finite'):
        ops.point_normals(bad)
    with pytest.raises(ValueError):
        ops.point_normals(pts, mode='outward')
    with pytest.raises(ValueError):
        ops.point_normals(pts, mode='viewpoint')
    with pytest.raises(ops.P2SError):
        ops.point_normals(pts.cpu())
    lib = ops._lib.load()
    out = torch.full((500, 3), 7.0, device=pts.device)
    stream = ops._stream()
    assert lib.p2s_point_normals_dev(ops._ptr(pts), 500, 10, 5, None, ops._ptr(out), None, None, stream) != 0
    assert b'mode' in lib.p2s_last_error()
    assert lib.p2s_point_normals_dev(ops._ptr(pts), 500, 10, 1, None, ops._ptr(out), None, None, stream) != 0
    assert lib.p2s_point_normals_dev(None, 500, 10, 0, None, ops._ptr(out), None, None, stream) != 0
    assert lib.p2s_point_normals_dev(ops._ptr(bad), 500, 10, 0, None, ops._ptr(out), None, None, stream) != 0
    fit, ids = _fit(pts.cpu().numpy())
    wrong = cu(ids).clone()
    wrong[3, 2] = 500
    assert lib.p2s_orient_normals_dev(ops._ptr(pts), ops._ptr(cu(fit)), ops._ptr(wrong), 500, 10, ops._ptr(out), None, None,
                                      stream) != 0
    assert b'neighbour id' in lib.p2s_last_error()
    wrong[3, 2] = -1
    with pytest.raises(ops.P2SError, match='neighbour id'):
        ops.orient_normals(pts, cu(fit), wrong)
    torch.cuda.synchronize()
    assert (out == 7.0).all()
    ref, _ = no.point_normals(pts.cpu().numpy(), 10)
    assert np.array_equal(ops.point_normals(pts).cpu().numpy(), ref)


def test_mesh_less_dataset_end_to_end(tmp_path, capsys):
    root = tmp_path / 'real'
    os.makedirs(str(root / '00_base_pc'))
    v, f = _mc_mesh('sphere', 96)
    sphere = ops.mesh_sample(cu(v), cu(f), 20000, seed=1).cpu().numpy() * np.float32(3) + np.float32(1)   # not unit size
    mesh_io.write_ply(str(root / '00_base_pc' / 'ball.ply'), sphere)
    np.savetxt(str(root / '00_base_pc' / 'ring.xyz'), pc.torus(20000, seed=2)[0])
    make_pc_dataset.main([str(root)])
    eval_dataset.main([str(root), '--spsr_estimated_normals'])
    out = capsys.readouterr().out
    assert '### normal estimation for point cloud' in out and 'ground truth' not in out
    for name in ('ball', 'ring'):
        pts = np.load(str(root / '04_pts' / (name + '.xyz.npy')))
        n = np.load(str(root / '06_normals_est' / (name + '.xyz.npy')))
        assert n.shape == pts.shape and n.dtype == np.float64
        assert np.loadtxt(str(root / '06_normals_est' / 'pts' / (name + '.xyz'))).shape == (len(pts), 6)
        rv, rf = mesh_io.read_ply(str(root / '06_poisson_rec' / (name + '.ply')))
        assert len(rf) > 100 and pc.closed_manifold(rf) and pc.signed_volume(rv, rf) > 0
    assert not (root / 'comp_poisson_rec_ml_normals.csv').exists() and not (root / '06_normals').exists()
    # with ground-truth meshes: both baselines side by side
    os.remove(str(root / '04_pts' / 'ring.xyz.npy'))
    (root / 'valset.txt').write_text('ball')
    (root / 'testset.txt').write_text('ball')
    lo, hi = sphere.astype(np.float64).min(0), sphere.astype(np.float64).max(0)      # the cloud's move into the unit cube
    gv = ((v.astype(np.float64) * 3.0 + 1.0) - (lo + hi) * 0.5) / (hi - lo).max()
    mesh_io.write_ply(str(root / '03_meshes' / 'ball.ply'), gv, f)
    eval_dataset.main([str(root), '--spsr', '--spsr_estimated_normals'])

    def chamfer(csv):
        lines = (root / csv).read_text().split('\n')
        assert lines[0].startswith('in mesh,ref mesh,Hausdorff dist new-ref') and len(lines) == 2
        assert len(lines[1].split(',')) == 6
        return float(lines[1].split(',')[-1])
    est, gt = chamfer('comp_poisson_rec_ml_normals.csv'), chamfer('comp_poisson_rec_gt_normals.csv')
    print('sphere Chamfer: estimated normals %.6f, ground-truth normals %.6f, ratio %.3f' % (est, gt, est / gt))
    assert est <= 1.1 * gt          # measured ratio 0.996
