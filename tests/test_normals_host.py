"""CPU: the point-normal oracle on analytic clouds, its spanning forest against SciPy's, the normals_poisson.mlx reader,
make_pc_dataset end to end, and the binding's prototypes of the two normal entry points."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import scipy.sparse as sparse
from scipy.sparse.csgraph import connected_components, minimum_spanning_tree

from oracle import normals_oracle as no
from points2surf_b200 import _lib, eval_dataset, make_pc_dataset, mesh_io, synth
import poisson_cases as pc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

NORMALS_POISSON_MLX = """<!DOCTYPE FilterScript>
<FilterScript>
 <filter name="Compute normals for point sets">
  <Param type="RichInt" name="K" value="%d"/>
  <Param type="RichInt" name="smoothIter" value="%d"/>
  <Param type="RichBool" name="flipFlag" value="%s"/>
  <Param type="RichPoint3f" x="0.5" y="0" name="viewPos" z="-2"/>
 </filter>
 <xmlfilter name="Screened Poisson Surface Reconstruction">
  <xmlparam name="depth" value="7"/>
  <xmlparam name="iters" value="8"/>
  <xmlparam name="pointWeight" value="2"/>
  <xmlparam name="scale" value="1.1"/>
 </xmlfilter>
 <filter name="Delete Current Mesh"/>
</FilterScript>
"""
POISSON_MLX = """<!DOCTYPE FilterScript>
<FilterScript>
 <xmlfilter name="Screened Poisson Surface Reconstruction">
  <xmlparam name="depth" value="8"/>
 </xmlfilter>
</FilterScript>
"""


def _agree(n, ref):
    """fraction of the non-zero normals with a positive dot against ref"""
    ok = np.any(n != 0, axis=1)
    return float((np.einsum('ij,ij->i', n[ok].astype(np.float64), ref[ok].astype(np.float64)) > 0).mean())


def test_noisy_plane_faces_up():
    rs = np.random.RandomState(0)
    pts = np.concatenate([rs.uniform(-1, 1, (3000, 2)), rs.normal(0, 0.002, (3000, 1))], 1).astype(np.float32)
    n, _ = no.point_normals(pts, 10)
    assert np.any(n != 0, axis=1).all() and (n[:, 2] > 0.9).all()


@pytest.mark.parametrize('shape', ['sphere', 'torus'])
def test_noise_free_surfaces_point_outward(shape):
    pts, ref = getattr(pc, shape)(5000, seed=1)
    n, ids = no.point_normals(pts, 10)
    assert np.abs(np.linalg.norm(n, axis=1) - 1).max() < 1e-6
    assert _agree(n, ref) == 1.0
    assert (ids[:, 0] == np.arange(len(pts))).all()


def test_noisy_cloud_floor():
    pts = synth.make_cloud('sphere', 5000, seed=3)
    ref = pts / np.linalg.norm(pts, axis=1, keepdims=True)
    frac = _agree(no.point_normals(pts, 10)[0], ref)
    print('oracle, noisy synth sphere: %.4f of the normals outward' % frac)
    assert frac > 0.97


def test_two_components_are_oriented_independently():
    a, ra = pc.sphere(1500, seed=2)
    b = a * np.float32(0.5) + np.float32([3, 0, 0])
    pts = np.concatenate([a, b]).astype(np.float32)
    ids = no.neighbours(pts, 10)
    fit, _ = no.plane_fit(pts, ids)
    n, parents, stats = no.orient(pts, fit, ids)
    assert stats['components'] == 2 and (parents == np.arange(len(pts))).sum() == 2
    assert _agree(n, np.concatenate([ra, ra])) == 1.0


def test_duplicates_and_collinear_points_are_degenerate():
    pts, _ = pc.sphere(2000, seed=4)
    dup = np.repeat(np.float32([[5, 5, 5]]), 12, 0)
    line = np.stack([np.linspace(8, 9, 40), np.zeros(40), np.zeros(40)], 1).astype(np.float32)
    allp = np.concatenate([pts, dup, line])
    ids = no.neighbours(allp, 10)
    fit, _ = no.plane_fit(allp, ids)
    assert (fit[2000:] == 0).all() and np.any(fit[:2000] != 0, axis=1).all()
    n, parents, stats = no.orient(allp, fit, ids)
    assert (n[2000:] == 0).all() and (parents[2000:] == -1).all() and stats['degenerate'] == 52


def test_kruskal_forest_is_the_minimum_spanning_forest():
    pts, _ = pc.torus(3000, seed=5)
    ids = no.neighbours(pts, 8)
    fit, _ = no.plane_fit(pts, ids)
    lo, hi, cost = no.edges(fit, ids)
    assert (np.diff(cost) >= 0).all()
    take = no.spanning_forest(len(pts), lo, hi)
    # SciPy drops zero weights: shift every cost by 1 and take the shift out again
    g = sparse.coo_matrix((cost + 1.0, (lo, hi)), shape=(len(pts), len(pts))).tocsr()
    mst = minimum_spanning_tree(g)
    ncomp = connected_components(g, directed=False)[0]
    assert take.sum() == mst.nnz == len(pts) - ncomp
    assert abs((mst.sum() - mst.nnz) - cost[take].sum()) <= 1e-9 * max(1.0, cost[take].sum())


def test_read_normals_poisson_filter(tmp_path):
    f = tmp_path / 'normals_poisson.mlx'
    f.write_text(NORMALS_POISSON_MLX % (12, 0, 'true'))
    normals, params = eval_dataset.read_normals_poisson_filter(str(f))
    assert normals == dict(k=12, smooth_iter=0, flip_flag=True, view_pos=(0.5, 0.0, -2.0))
    assert params == dict(depth=7, point_weight=2.0, scale=1.1, iters=8)
    f.write_text(NORMALS_POISSON_MLX % (10, 2, 'false'))
    with pytest.raises(ValueError, match='smoothIter'):
        eval_dataset.read_normals_poisson_filter(str(f))
    f.write_text(POISSON_MLX)
    with pytest.raises(ValueError):
        eval_dataset.read_normals_poisson_filter(str(f))
    assert eval_dataset.read_poisson_filter(str(f))['depth'] == 8


def test_make_pc_dataset(tmp_path, capsys):
    root = tmp_path / 'real'
    base = root / '00_base_pc'
    os.makedirs(str(base))
    rs = np.random.RandomState(0)
    clouds = {n: (rs.uniform(-3, 5, (700, 3)) * [1, 2, 0.5]).astype(np.float32) for n in ('a', 'b', 'c', 'd')}
    mesh_io.write_ply(str(base / 'a.ply'), clouds['a'])
    with open(str(base / 'b.obj'), 'w') as fp:
        fp.write(''.join('v %r %r %r\n' % tuple(float(x) for x in p) for p in clouds['b']))
    mesh_io.write_off(str(base / 'c.off'), clouds['c'], np.array([]))
    np.savetxt(str(base / 'd.xyz'), clouds['d'])
    np.savetxt(str(base / 'flat.xyz'), np.concatenate([clouds['d'][:, :2], np.zeros((700, 1))], 1))
    make_pc_dataset.main([str(root), '--target_num_points', '500'])
    assert 'flat.xyz' in capsys.readouterr().out
    names = ['a', 'b', 'c', 'd']
    assert (root / 'testset.txt').read_text() == (root / 'valset.txt').read_text() == '\n'.join(names)
    assert not (root / 'trainset.txt').exists() and not (root / '04_pts' / 'flat.xyz.npy').exists()
    outs = []
    for n in names:
        p = np.load(str(root / '04_pts' / (n + '.xyz.npy')))
        outs += [root / '04_pts' / (n + '.xyz.npy'), root / '04_pts_vis' / (n + '.xyz')]
        assert p.shape == (500, 3) and p.dtype == np.float32
        full = make_pc_dataset._to_unit_cube(clouds[n]).astype(np.float32)
        assert np.abs(full.max(0) + full.min(0)).max() < 1e-6 and abs((full.max(0) - full.min(0)).max() - 1) < 1e-6
        assert np.abs(p).max() <= 0.5 + 1e-6
        # the seeded sub-sample: rows of the full cloud, the same ones on every run
        assert len(np.unique(p, axis=0)) == 500 and (p[:, None, :] == full[None, :, :]).all(2).any(1).all()
        assert len(np.loadtxt(str(root / '04_pts_vis' / (n + '.xyz')))) == 500
    first = [np.load(str(o)) for o in outs[::2]]
    mtimes = [os.path.getmtime(str(o)) for o in outs]
    make_pc_dataset.main([str(root), '--target_num_points', '500'])
    assert [os.path.getmtime(str(o)) for o in outs] == mtimes          # up to date: skipped
    for o in outs:
        os.remove(str(o))
    make_pc_dataset.main([str(root), '--target_num_points', '500'])
    assert all(np.array_equal(a, np.load(str(o))) for a, o in zip(first, outs[::2]))


def test_binding_declares_the_normal_entry_points():
    txt = re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'p2s_b200.h')).read(), flags=re.S)
    for name in ('p2s_point_normals_dev', 'p2s_orient_normals_dev'):
        args = re.search(name + r'\s*\((.*?)\)\s*;', txt, re.S).group(1).split(',')
        res, argtypes = _lib.SIGNATURES[name]
        assert res is C.c_int and len(argtypes) == len(args)
        for decl, ct in zip(args, argtypes):
            if 'p2s_normals_stats' in decl:
                assert ct is C.POINTER(_lib.NormalsStats)
            elif 'double*' in decl:
                assert ct is C.POINTER(C.c_double)
            elif '*' in decl:
                assert ct is C.c_void_p
            else:
                assert ct is (C.c_int64 if 'int64_t' in decl else C.c_int)
    assert C.sizeof(_lib.NormalsStats) == 48
