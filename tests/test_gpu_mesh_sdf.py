"""GPU tests of the training-target stage: p2s_mesh_signed_distance_dev against the reference's own 05_query_dist and the
float64 oracle (oracle/mesh_sdf_oracle.py), and the make_dataset / sdf mirrors built on it (tests/golden/mesh_sdf.npz)."""
import os

import numpy as np
import pytest
import torch

from oracle import mesh_sdf_oracle as msdf
from points2surf_b200 import ops, sdf, mesh_io, make_dataset
from helpers import load_golden

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _fixture(i):
    g = load_golden('mesh_sdf.npz')
    return {k: g[k + '_%d' % i] for k in ('name', 'verts', 'faces', 'ref_query_pts', 'ref_query_dist', 'hash', 'oracle_dist',
                                          'oracle_face', 'oracle_wind')}


def _check_faces(verts, faces, query, face, face_o, d_o, tol):
    """closest faces equal the oracle's except where the two faces are equally close within tol"""
    bad = np.nonzero(face != face_o)[0]
    if len(bad):
        v = verts.astype(np.float64)
        for k in bad:
            a, b, c = (v[faces[face[k]][j]][None, None] for j in range(3))
            d = np.sqrt(msdf._closest_dist2(query[k].astype(np.float64)[None, None], a, b, c)[0, 0])
            assert abs(d - abs(d_o[k])) <= tol, (k, face[k], face_o[k], d, d_o[k])


def _mc_mesh(kind, res):
    """closed, outward-oriented marching-cubes mesh of an analytic sphere or torus (positive inside)"""
    x = torch.linspace(-1, 1, res, device=DEV)
    X, Y, Z = torch.meshgrid(x, x, x, indexing='ij')
    if kind == 'sphere':
        vol = 0.6 - torch.sqrt(X * X + Y * Y + Z * Z)
    else:
        vol = 0.25 - torch.sqrt((torch.sqrt(X * X + Y * Y) - 0.55) ** 2 + Z * Z)
    v, f = ops.marching_cubes(vol.contiguous(), 0.0)
    v, f = v.cpu().numpy(), f.cpu().numpy()
    return v, sdf._orient_outward(v, f)


def _torus_50k():
    for res in range(120, 400, 8):
        v, f = _mc_mesh('torus', res)
        if len(f) >= 45000:
            return v, f
    raise AssertionError('no torus mesh with 45k faces')


@pytest.mark.parametrize('i', [0, 1, 2])
def test_fixture_matches_reference_and_oracle(i):
    fx = _fixture(i)
    q = fx['ref_query_pts']
    d, face, w = ops.mesh_signed_distance(cu(fx['verts']), cu(fx['faces']), cu(q), return_face_ids=True, return_winding=True)
    d, face, w = d.cpu().numpy(), face.cpu().numpy(), w.cpu().numpy()
    assert np.array_equal(np.sign(d), np.sign(fx['ref_query_dist']))
    assert np.abs(np.abs(d) - np.abs(fx['ref_query_dist'])).max() <= 1e-5
    assert np.abs(d - fx['oracle_dist']).max() <= 1e-6
    off = np.abs(fx['oracle_dist']) > 1e-6
    np.testing.assert_allclose(w[off], fx['oracle_wind'][off], atol=1e-5)
    _check_faces(fx['verts'], fx['faces'], q, face, fx['oracle_face'], fx['oracle_dist'], 1e-12)


def _stress_points(v, f, rng):
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    fi = rng.choice(len(f), 300, replace=False)
    n = np.cross(b - a, c - a)
    n /= np.linalg.norm(n, axis=1, keepdims=True) + 1e-30
    return np.concatenate([
        v[rng.choice(len(v), 200, replace=False)],                                  # exactly on vertices
        (0.5 * (a[fi] + b[fi])),                                                    # on edges
        (a[fi] + b[fi] + c[fi]) / 3.0,                                              # on faces
        (a[fi] + b[fi] + c[fi]) / 3.0 + n[fi] * rng.uniform(-0.02, 0.02, (300, 1)),   # near faces, both sides
        rng.uniform(-1, 1, (400, 3)),                                               # in the cube
        rng.normal(size=(100, 3)) * np.array([[3.0], [50.0]]).repeat(50, 0),        # far outside
    ]).astype(np.float32)


@pytest.mark.parametrize('kind,res,degenerate', [('sphere', 32, False), ('torus', 40, False), ('sphere', 24, True)])
def test_stress_against_oracle(kind, res, degenerate):
    v, f = _mc_mesh(kind, res)
    rng = np.random.RandomState(res)
    q = _stress_points(v, f, rng)
    if degenerate:   # zero-area faces (a point, a segment) and duplicated faces
        extra = np.stack([f[:20, 0], f[:20, 0], f[:20, 0]], 1)
        seg = np.stack([f[20:40, 0], f[20:40, 1], f[20:40, 0]], 1)
        f = np.concatenate([f, extra, seg, f[40:60]]).astype(np.int32)
    d, face, w = ops.mesh_signed_distance(cu(v), cu(f), cu(q), return_face_ids=True, return_winding=True)
    d, face, w = d.cpu().numpy(), face.cpu().numpy(), w.cpu().numpy()
    d_o, face_o, w_o = msdf.mesh_signed_distance(v, f, q)
    # 1e-6, relative beyond |d| = 1: the far points (|d| up to ~150) are stored in fp32 (half an ulp at 128 is 3.8e-6)
    assert (np.abs(np.abs(d) - np.abs(d_o)) <= 1e-6 * np.maximum(1.0, np.abs(d_o))).all()
    decided = np.abs(w_o - 0.5) > 1e-3
    assert np.array_equal(np.signbit(d[decided]), np.signbit(d_o[decided]))   # on the surface: +0 in both
    off = np.abs(d_o) > 1e-6
    np.testing.assert_allclose(w[off], w_o[off], atol=1e-4)
    _check_faces(v, f, q, face, face_o, d_o, 1e-12)
    if not degenerate:   # closed outward mesh: inside is exactly w ~ 1
        assert ((w_o > 0.5) == (np.abs(w_o - 1.0) < 1e-6))[off].all()


def test_deterministic_and_independent_of_the_query_split():
    fx = _fixture(0)
    v, f = cu(fx['verts']), cu(fx['faces'])
    rng = np.random.RandomState(0)
    q = np.concatenate([fx['ref_query_pts'], rng.uniform(-1, 1, (3001, 3)).astype(np.float32)])
    r1 = [t.cpu().numpy() for t in ops.mesh_signed_distance(v, f, cu(q), True, True)]
    r2 = [t.cpu().numpy() for t in ops.mesh_signed_distance(v, f, cu(q), True, True)]
    parts = [[t.cpu().numpy() for t in ops.mesh_signed_distance(v, f, cu(q[a:b]), True, True)]
             for a, b in ((0, 777), (777, 778), (778, len(q)))]
    for k in range(3):
        assert r1[k].tobytes() == r2[k].tobytes()
        assert r1[k].tobytes() == np.concatenate([p[k] for p in parts]).tobytes()


def test_errors():
    v = cu(np.eye(3, dtype=np.float32))
    q = cu(np.zeros((4, 3), np.float32))
    for bad in ([[0, 1, 3]], [[0, -1, 2]]):
        with pytest.raises(ops.P2SError):
            ops.mesh_signed_distance(v, cu(np.array(bad, np.int32)), q)
    with pytest.raises(ops.P2SError):
        ops.mesh_signed_distance(v, cu(np.zeros((0, 3), np.int32)), q)
    with pytest.raises(ops.P2SError):
        ops.mesh_signed_distance(v.cpu(), cu(np.array([[0, 1, 2]], np.int32)), q)
    with pytest.raises(ops.P2SError):
        ops.mesh_signed_distance(v, cu(np.array([[0, 1, 2]], np.int32)), q.cpu())
    # a valid call still works after the errors, and Q = 0 is fine
    d = ops.mesh_signed_distance(v, cu(np.array([[0, 1, 2]], np.int32)), q)
    assert torch.isfinite(d).all()
    assert ops.mesh_signed_distance(v, cu(np.array([[0, 1, 2]], np.int32)), q[:0]).numel() == 0


def test_large_case_against_oracle_sample():
    v, f = _torus_50k()
    assert 45000 <= len(f) <= 60000
    rng = np.random.RandomState(7)
    fi = rng.choice(len(f), 75000)
    a, b, c = v[f[fi, 0]], v[f[fi, 1]], v[f[fi, 2]]
    r = rng.uniform(0, 1, (75000, 2))
    r[r.sum(1) > 1] = 1 - r[r.sum(1) > 1]
    near = a + r[:, :1] * (b - a) + r[:, 1:] * (c - a) + rng.normal(0, 0.01, (75000, 3))
    q = np.concatenate([near, rng.uniform(-1, 1, (75000, 3))]).astype(np.float32)
    d, face = ops.mesh_signed_distance(cu(v), cu(f), cu(q), return_face_ids=True)
    d, face = d.cpu().numpy(), face.cpu().numpy()
    sel = rng.choice(len(q), 500, replace=False)
    d_o, face_o, w_o = msdf.mesh_signed_distance(v, f, q[sel])
    assert np.abs(d[sel] - d_o).max() <= 1e-6
    _check_faces(v, f, q[sel], face[sel], face_o, d_o, 1e-12)


def test_query_pts_for_mesh_far_half_and_close_points():
    fx = _fixture(0)
    pr = 6.0 / 256
    rng = np.random.RandomState(int(fx['hash']))
    q = sdf.get_query_pts_for_mesh((fx['verts'], fx['faces']), 2000, pr, 0.5, rng)
    assert q.shape == (2000, 3) and q.dtype == np.float64
    assert np.array_equal(q[:1000].astype(np.float32), fx['ref_query_pts'][:1000])
    d = ops.mesh_signed_distance(cu(fx['verts']), cu(fx['faces']), cu(q[1000:].astype(np.float32))).cpu().numpy()
    assert np.abs(d).max() <= pr + 1e-6
    # the same stream gives the same points; source.sdf re-exports the mirror
    from source import sdf as src_sdf
    q2 = src_sdf.get_query_pts_for_mesh((fx['verts'], fx['faces']), 2000, pr, 0.5, np.random.RandomState(int(fx['hash'])))
    assert np.array_equal(q, q2)
    dd = src_sdf.get_signed_distance((fx['verts'], fx['faces']), fx['ref_query_pts'])
    assert dd.dtype == np.float64 and np.array_equal(np.sign(dd), np.sign(fx['ref_query_dist']))


def test_close_samples_are_area_weighted():
    # faces with areas 1 : 4 : 9 (+ a zero-area face that is never sampled)
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [2, 0, 1], [0, 2, 1], [0, 0, 2], [3, 0, 2], [0, 3, 2]], np.float32)
    f = np.array([[0, 1, 2], [3, 4, 5], [0, 0, 0], [6, 7, 8]], np.int32)
    n = 200000
    _, fid = sdf._query_pts_and_faces((v, f), n, 0.01, 0.0, np.random.RandomState(3))
    p = np.array([1, 4, 0, 9]) / 14.0
    cnt = np.bincount(fid, minlength=4)
    assert cnt[2] == 0
    assert (np.abs(cnt / n - p) <= 4 * np.sqrt(p * (1 - p) / n)).all()


def _write_fixture_meshes(mesh_dir):
    os.makedirs(mesh_dir, exist_ok=True)
    for i in range(3):
        fx = _fixture(i)
        mesh_io.write_ply(os.path.join(mesh_dir, str(fx['name'])), fx['verts'], fx['faces'])


def test_get_query_pts_dist_ms_on_the_fixture_meshes(tmp_path):
    root = tmp_path / 'abc'
    _write_fixture_meshes(str(root / '03_meshes'))
    make_dataset.get_query_pts_dist_ms(str(tmp_path), 'abc', '03_meshes', '05_query_pts', '05_query_dist', '05_query_vis',
                                       6.0 / 256, num_query_pts=2000, far_query_pts_ratio=0.5, debug=True)
    outs = []
    for i in range(3):
        fx = _fixture(i)
        name = str(fx['name'])
        q = np.load(str(root / '05_query_pts' / (name + '.npy')))
        d = np.load(str(root / '05_query_dist' / (name + '.npy')))
        assert q.dtype == np.float32 and q.shape == (2000, 3) and d.dtype == np.float32 and d.shape == (2000,)
        assert np.array_equal(q[:1000], fx['ref_query_pts'][:1000])
        assert np.array_equal(np.sign(d[:1000]), np.sign(fx['ref_query_dist'][:1000]))
        assert np.abs(d[:1000] - fx['ref_query_dist'][:1000]).max() <= 1e-5
        assert np.abs(d).max() <= 1.0 and (root / '05_query_vis' / (name + '.ply')).exists()
        outs += [root / '05_query_pts' / (name + '.npy'), root / '05_query_dist' / (name + '.npy')]
    mtimes = [os.path.getmtime(str(p)) for p in outs]
    # up-to-date outputs are skipped, also through the command line (patch radius from settings.ini)
    (root / 'settings.ini').write_text('[general]\ngrid_resolution = 256\nepsilon = 5\n')
    make_dataset.main([str(root)])
    assert [os.path.getmtime(str(p)) for p in outs] == mtimes


def test_chain_mesh_to_training_epoch(tmp_path):
    from points2surf_b200 import points_to_surf_train as p2s_train
    root = tmp_path / 'data'
    _write_fixture_meshes(str(root / '03_meshes'))
    os.makedirs(str(root / '04_pts'))
    names = []
    for i in range(3):
        fx = _fixture(i)
        stem = str(fx['name'])[:-4]
        names.append(stem)
        pts = ops.mesh_sample(cu(fx['verts']), cu(fx['faces']), 5000, seed=i).cpu().numpy()
        np.save(str(root / '04_pts' / (stem + '.xyz.npy')), pts)
    make_dataset.get_query_pts_dist_ms(str(tmp_path), 'data', '03_meshes', '05_query_pts', '05_query_dist', '05_query_vis',
                                       6.0 / 256, num_query_pts=256, far_query_pts_ratio=0.5)
    (root / 'trainset.txt').write_text('\n'.join(names[:2]) + '\n')
    (root / 'testset.txt').write_text(names[2] + '\n')
    opt = p2s_train.parse_arguments([
        '--name', 'chain', '--indir', str(root), '--outdir', str(tmp_path / 'models'), '--logdir', str(tmp_path / 'logs'),
        '--nepoch', '1', '--batchSize', '16', '--patches_per_shape', '32', '--points_per_patch', '300',
        '--sub_sample_size', '1000', '--patch_radius', '0.0', '--lr', '0.001', '--shared_transformer', '1',
        '--outputs', 'imp_surf_magnitude', 'imp_surf_sign', 'patch_pts_ids', 'p_index'])
    hist = p2s_train.points_to_surf_train(opt)
    assert len([h for h in hist if h[0] == 'train']) == 4 and all(np.isfinite(h[3]).all() for h in hist)
