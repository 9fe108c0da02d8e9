"""The solid voxelisation kernel (csrc/inside.cu, ops.mesh_inside_grid) and make_dataset --gt_recon on the GPU.

- The kernel equals oracle/inside_oracle.py bit for bit at res 32, 64, 128 and 100 on an icosphere, a torus, the three
  abc_minimal meshes and the two lattice meshes (and on an open mesh, where the flags are the rule's parity).
- At res 64 it agrees with the sign of ops.mesh_signed_distance (winding number) at every voxel with |d| > 1e-5.
- --gt_recon end to end on a temporary dataset: the abc_minimal meshes scanned at the poses of tests/golden/scan.npz plus
  a copy of one with a deleted face, at res 64.
- On a sphere, the exact-sign mesh's Chamfer distance to the analytic surface is within 0.25 voxel."""
import os

import numpy as np
import pytest
import torch

import inside_cases as ic
from oracle import inside_oracle as io
from points2surf_b200 import make_dataset, mesh_io, ops, sdf, trafo

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _open_sphere():
    v, f = ic.icosphere(level=3)
    return v, f[1:]


def _cases():
    out = dict(ic.closed_cases())
    out['open_sphere'] = _open_sphere()
    return out


@pytest.mark.parametrize('res', [32, 64, 128, 100, 16])
@pytest.mark.parametrize('name', ['sphere', 'torus', 'abc0', 'abc1', 'abc2', 'box', 'octahedron', 'open_sphere'])
def test_kernel_equals_oracle_bit_for_bit(name, res):
    v, f = _cases()[name]
    got = ops.mesh_inside_grid(_cu(v), _cu(f), res).cpu().numpy().astype(np.uint8)
    want, cross = io.inside_grid(v, f, res)
    assert np.array_equal(got, want), int((got != want).sum())
    if name != 'open_sphere':
        assert (cross % 2 == 0).all()
    print('%s res %d: %d inside' % (name, res, int(got.sum())))


def test_lattice_meshes_give_the_geometric_inside_set():
    for kind in ('box', 'octahedron'):
        v, f = getattr(ic, kind)()
        got = ops.mesh_inside_grid(_cu(v), _cu(f), ic.LATTICE_RES).cpu().numpy().astype(np.uint8)
        assert np.array_equal(got, getattr(ic, kind + '_inside')()), kind


@pytest.mark.parametrize('name', ['sphere', 'torus', 'abc0', 'abc1', 'abc2'])
def test_kernel_agrees_with_winding_number_sign_at_res64(name):
    res = 64
    v, f = ic.closed_cases()[name]
    inside = ops.mesh_inside_grid(_cu(v), _cu(f), res).reshape(-1)
    q = ops.query_points(torch.arange(res ** 3, dtype=torch.int32, device=DEV), res)
    d, w = ops.mesh_signed_distance(_cu(v), _cu(f), q, return_winding=True)
    far = d.abs() > 1e-5
    # the crossing parity is the winding number mod 2; where the winding number is 0 or 1 that is the distance's sign.
    # abc0 is two closed components that overlap in a sliver: there w = 2, the distance is positive and the parity even.
    wr = torch.round(w)
    assert float((w - wr).abs()[far].max()) < 1e-2
    assert int(((wr.remainder(2) == 1) != inside)[far].sum()) == 0
    simple = far & ((wr == 0) | (wr == 1))
    bad = int(((d > 0) != inside)[simple].sum())
    print('%s: %d of %d voxels far from the surface, %d inside, %d with a winding number other than 0 or 1' % (
        name, int(far.sum()), res ** 3, int(inside.sum()), int((far & ~simple).sum())))
    assert bad == 0
    assert int(simple.sum()) > 0.99 * res ** 3


def test_wrapper_rejects_bad_input_and_recovers():
    v, f = ic.box()
    with pytest.raises(ops.P2SError, match='resolution'):
        ops.mesh_inside_grid(_cu(v), _cu(f), 1025)
    with pytest.raises(ops.P2SError, match='face index'):
        ops.mesh_inside_grid(_cu(v), _cu(f + 8), 16)
    far = v.copy()
    far[0, 1] = -16.0
    with pytest.raises(ops.P2SError, match='16'):
        ops.mesh_inside_grid(_cu(far), _cu(f), 16)
    empty = ops.mesh_inside_grid(_cu(v), torch.zeros((0, 3), dtype=torch.int32, device=DEV), 16)
    assert not empty.any()
    got = ops.mesh_inside_grid(_cu(v), _cu(f), 16).cpu().numpy().astype(np.uint8)
    assert np.array_equal(got, ic.box_inside())


# ------------------------------------------------------------------ make_dataset --gt_recon
def _scan(v, f, i):
    g = np.load(os.path.join(ic.GOLDEN, 'scan.npz'))
    rot = np.stack([trafo.quaternion_matrix(q)[:3, :3] for q in g['rotations_%d' % i]])
    return ops.range_scan(_cu(v), _cu(f), rot, g['locations_%d' % i], noise_sigma=float(g['sigma_%d' % i]),
                          seed=7)[0].cpu().numpy()


def _tree_mtimes(root):
    out = {}
    for d in ('05_query_pts_grid', '05_query_dist_grid', '06_mc_gt_recon', '06_mc_gt_recon/vol', '06_mc_gt_exact_sign'):
        for f in os.listdir(os.path.join(root, d)):
            p = os.path.join(root, d, f)
            if os.path.isfile(p):
                out[p] = os.stat(p).st_mtime_ns
    return out


def test_gt_recon_end_to_end(tmp_path, capsys):
    res = 64
    root = str(tmp_path / 'ds')
    os.makedirs(os.path.join(root, '03_meshes'))
    os.makedirs(os.path.join(root, '04_pts'))
    names = []
    for i in range(3):
        v, f = ic.abc(i)
        pts = _scan(v, f, i)
        for name, faces in (('abc%d' % i, f),) + ((('open', f[1:]),) if i == 2 else ()):
            mesh_io.write_ply(os.path.join(root, '03_meshes', name + '.ply'), v, faces)
            np.save(os.path.join(root, '04_pts', name + '.xyz.npy'), pts)
            names.append(name)
    with open(os.path.join(root, 'testset.txt'), 'w') as fp:
        fp.write('\n'.join(names))
    make_dataset.main([root, '--gt_recon', '--grid_resolution', str(res)])
    out = capsys.readouterr().out
    assert 'open: mesh is not closed' in out
    for name in names:
        v, f = mesh_io.read_ply(os.path.join(root, '03_meshes', name + '.ply'))
        pts = np.load(os.path.join(root, '04_pts', name + '.xyz.npy'))
        file_q = os.path.join(root, '05_query_pts_grid', name + '.xyz.npy')
        file_d = os.path.join(root, '05_query_dist_grid', name + '.xyz.npy')
        q, d = np.load(file_q), np.load(file_d)
        assert q.dtype == np.float32 and d.dtype == np.float32
        want_q = ops.query_points(ops.query_grid(_cu(pts.astype(np.float32)), res, 3), res).cpu().numpy()
        assert np.array_equal(q, want_q)
        fo = sdf._orient_outward(v.astype(np.float32), f.astype(np.int32))
        want_d = ops.mesh_signed_distance(_cu(v.astype(np.float32)), _cu(fo), _cu(q)).cpu().numpy().astype(np.float64)
        want_d[np.isnan(want_d)] = 0.0
        want_d[np.isinf(want_d)] = 1.0
        assert np.array_equal(d, np.clip(want_d, -1.0, 1.0).astype(np.float32))
        # 06_mc_gt_recon is implicit_surface_to_mesh on those files
        mine_vol, mine = str(tmp_path / (name + '.xyz.off')), str(tmp_path / (name + '.ply'))
        sdf.implicit_surface_to_mesh_file(file_d, file_q, mine_vol, mine, res, 5, 13)
        rv, rf = mesh_io.read_ply(os.path.join(root, '06_mc_gt_recon', name + '.ply'))
        mv, mf = mesh_io.read_ply(mine)
        assert np.array_equal(rv, mv) and np.array_equal(rf, mf) and len(rf) > 1000
        assert os.path.isfile(os.path.join(root, '06_mc_gt_recon', 'vol', name + '.xyz.off'))
        exact = os.path.join(root, '06_mc_gt_exact_sign', name + '.ply')
        assert os.path.isfile(exact) == (name != 'open')
        if name != 'open':
            assert '%s: %d grid queries, ' % (name, len(q)) in out
            ev, ef = mesh_io.read_ply(exact)
            assert len(ef) > 1000
    for report in ('comp_mc_gt_recon.csv', 'comp_mc_gt_exact_sign.csv'):
        with open(os.path.join(root, report)) as fp:
            lines = fp.read().splitlines()
        print(report, *lines, sep='\n')
        assert len(lines) == 1 + len(names)
    before = _tree_mtimes(root)
    assert len(before) == 5 * len(names) - 1
    make_dataset.main([root, '--gt_recon', '--grid_resolution', str(res)])
    assert _tree_mtimes(root) == before


def test_exact_sign_mesh_of_a_sphere_is_within_a_quarter_voxel_of_the_analytic_surface():
    res, r = 64, 0.45
    v, f = ic.icosphere(radius=r, level=5)
    vc, fc = _cu(v), _cu(f)
    pts = ops.mesh_sample(vc, fc, 50000, seed=3)
    lin = ops.query_grid(pts, res, 3)
    dist = ops.mesh_signed_distance(vc, fc, ops.query_points(lin, res))
    vol = make_dataset.exact_sign_volume(ops.mesh_inside_grid(vc, fc, res), lin, dist)
    mv, mf = ops.marching_cubes(vol, 0.0)
    rec = ops.mesh_sample(mv, mf, 200000, seed=4)
    g = torch.Generator().manual_seed(5)
    sph = torch.randn((200000, 3), generator=g).to(DEV)
    sph = (sph / sph.norm(dim=1, keepdim=True) * r).float().contiguous()
    to_sphere = (rec.norm(dim=1) - r).abs()
    to_rec, _ = ops.nn_distance(sph, rec)
    voxel = 2.0 / res
    chamfer = float(to_sphere.mean() + to_rec.mean()) / voxel
    print('sphere r %.2f at res %d: Chamfer %.4f voxel (mesh->sphere %.4f, sphere->mesh samples %.4f), max |d| %.4f '
          'voxel' % (r, res, chamfer, float(to_sphere.mean()) / voxel, float(to_rec.mean()) / voxel,
                     float(to_sphere.max()) / voxel))
    assert chamfer < 0.25
    assert float(to_sphere.max()) < 0.5 * voxel
