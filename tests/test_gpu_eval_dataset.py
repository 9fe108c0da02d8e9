"""GPU tests of the evaluation outputs built on point-to-mesh queries: the ground-truth point normals of
eval_dataset.get_pts_normals (06_normals) and the distance maps of figure.distance_vis."""
import os

import numpy as np
import pytest
import scipy.spatial as spatial

from points2surf_b200 import eval_dataset, make_dataset, mesh_io, ops, point_cloud, sdf
from points2surf_b200.figure import distance_vis
from test_gpu_mesh_sdf import _fixture, _mc_mesh, cu

pytestmark = pytest.mark.gpu


def _dataset(root, n_pts=4000):
    """03_meshes with the three abc_minimal meshes; 04_pts: [N,3] clouds for two, an [N,6] one (points + normals) for the
    third"""
    os.makedirs(str(root / '03_meshes'))
    os.makedirs(str(root / '04_pts'))
    names = []
    for i in range(3):
        fx = _fixture(i)
        stem = str(fx['name'])[:-4]
        names.append(stem)
        mesh_io.write_ply(str(root / '03_meshes' / (stem + '.ply')), fx['verts'], fx['faces'])
        pts = ops.mesh_sample(cu(fx['verts']), cu(fx['faces']), n_pts, seed=100 + i).cpu().numpy()
        pts += np.random.RandomState(i).normal(0, 0.002, pts.shape).astype(np.float32)
        if i == 2:
            pts = np.concatenate([pts, np.ones_like(pts)], 1)
        np.save(str(root / '04_pts' / (stem + '.xyz.npy')), pts)
    return names


def _expected_normals(pts, verts, faces, samples_per_model, mesh_file):
    """-> (oriented face normal of the nearest sample by cKDTree [N,3], samples, their faces, oriented face normals)"""
    s, fid = ops.mesh_sample(cu(verts), cu(faces), samples_per_model, make_dataset.filename_to_hash(mesh_file),
                             return_face_ids=True)
    s, fid = s.cpu().numpy(), fid.cpu().numpy()
    _, sid = spatial.cKDTree(s).query(pts.astype(np.float32), k=1)
    fn = make_dataset.face_normals(verts, sdf._orient_outward(verts, faces))
    return fn[fid[sid]], s, fid, fn


def test_get_pts_normals_files_and_values(tmp_path, capsys):
    root = tmp_path / 'ds'
    names = _dataset(root)
    eval_dataset.main([str(root)])
    assert 'meshlabserver' in capsys.readouterr().out
    outs = []
    for i, stem in enumerate(names):
        fx = _fixture(i)
        npy = root / '06_normals' / (stem + '.xyz.npy')
        xyz = root / '06_normals' / 'pts' / (stem + '.xyz')
        outs += [npy, xyz]
        pts = np.load(str(root / '04_pts' / (stem + '.xyz.npy')))[:, :3]
        n = np.load(str(npy))
        assert n.shape == (len(pts), 3) and n.dtype == np.float64
        assert np.abs(np.linalg.norm(n, axis=1) - 1.0).max() <= 1e-6
        exp, s, fid, fn = _expected_normals(pts, fx['verts'], fx['faces'], 100000,
                                               str(root / '03_meshes' / (stem + '.ply')))
        diff = np.abs(n - exp).max(1) > 1e-12
        # every difference is a distance tie: the normal is that of an equally near sample
        for k in np.nonzero(diff)[0]:
            d = np.linalg.norm(s.astype(np.float64) - pts[k], axis=1)
            cand = np.nonzero(d <= d.min() + 1e-6)[0]
            assert any(np.abs(fn[fid[c]] - n[k]).max() <= 1e-12 for c in cand), k
        assert diff.mean() < 1e-3
        # the reference's text layout: 'x y z nx ny nz ' per point, values as str() of their NumPy scalars
        ref_txt = tmp_path / 'ref.xyz'
        point_cloud.write_xyz(str(ref_txt), pts, normals=n)
        assert xyz.read_text() == ref_txt.read_text()
        first = xyz.read_text().split('\n')[0]
        assert first == ' '.join(str(x) for x in list(pts[0]) + list(n[0])) + ' '
    # up-to-date outputs are skipped
    mtimes = [os.path.getmtime(str(p)) for p in outs]
    eval_dataset.get_pts_normals(str(tmp_path), 'ds', '04_pts', '03_meshes', '06_normals', samples_per_model=100000)
    assert [os.path.getmtime(str(p)) for p in outs] == mtimes


def test_pts_normals_of_an_inverted_mesh_point_outward():
    fx = _fixture(0)
    inverted = np.ascontiguousarray(fx['faces'][:, ::-1])
    pts = ops.mesh_sample(cu(fx['verts']), cu(fx['faces']), 2000, seed=9).cpu().numpy()
    n = eval_dataset.pts_normals(pts, fx['verts'], inverted, 20000, seed=3)
    s, fid = ops.mesh_sample(cu(fx['verts']), cu(inverted), 20000, 3, return_face_ids=True)
    _, sid = spatial.cKDTree(s.cpu().numpy()).query(pts, k=1)
    outward = make_dataset.face_normals(fx['verts'], fx['faces'])     # the fixture mesh is oriented outward
    assert (np.abs(n - outward[fid.cpu().numpy()[sid]]).max(1) <= 1e-12).mean() > 0.999


# fraction of the noise-free scan points of abc_minimal mesh 0 whose ground-truth normal has dot > 0.9 with the normal of
# the face the ray hit: 0.9666 of 60 013 points, measured on one H100 80GB HBM3 at a 400 W power limit (seeded, so it
# only moves when the sampler, the scan or the nearest-neighbour rule changes)
SCAN_NORMAL_AGREEMENT_MIN = 0.96


def test_gt_normals_on_a_noise_free_scan(tmp_path):
    fx = _fixture(0)
    mesh_file = str(tmp_path / str(fx['name']))
    mesh_io.write_ply(mesh_file, fx['verts'], fx['faces'])
    _, locations, rotations = make_dataset.get_scan_poses(mesh_file, 5, 30)
    from points2surf_b200 import trafo
    rot = np.stack([trafo.quaternion_matrix(q)[:3, :3] for q in rotations])
    _, clean, face_ids, _ = ops.range_scan(cu(fx['verts']), cu(fx['faces']), rot, locations, noise_sigma=0.0, seed=1)
    clean, face_ids = clean.cpu().numpy(), face_ids.cpu().numpy()
    assert len(clean) > 1000
    n = eval_dataset.pts_normals(clean, fx['verts'], fx['faces'], 100000, make_dataset.filename_to_hash(mesh_file))
    hit = make_dataset.face_normals(fx['verts'], sdf._orient_outward(fx['verts'], fx['faces']))[face_ids]
    frac = float((np.einsum('ij,ij->i', n, hit) > 0.9).mean())
    print('scan points: %d, fraction of GT normals with dot > 0.9 with the hit face normal: %.4f' % (len(clean), frac))
    assert frac >= SCAN_NORMAL_AGREEMENT_MIN


def _icosphere(r, level):
    t = (1 + 5 ** 0.5) / 2
    v = np.array([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                  [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], np.float64)
    f = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2],
                  [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11],
                  [6, 2, 10], [8, 6, 7], [9, 8, 1]])
    v = list(v / np.linalg.norm(v, axis=1, keepdims=True))
    for _ in range(level):
        mid, nf = {}, []
        for a, b, c in f:
            m = []
            for x, y in ((a, b), (b, c), (c, a)):
                key = (min(x, y), max(x, y))
                if key not in mid:
                    p = v[x] + v[y]
                    v.append(p / np.linalg.norm(p))
                    mid[key] = len(v) - 1
                m.append(mid[key])
            nf += [[a, m[0], m[2]], [b, m[1], m[0]], [c, m[2], m[1]], m]
        f = np.array(nf)
    return (np.array(v) * r).astype(np.float32), f.astype(np.int32)


def test_distance_maps_on_a_sphere_reconstruction(tmp_path):
    vg, fg = _icosphere(0.6, 5)
    gt = str(tmp_path / 'gt.ply')
    mesh_io.write_ply(gt, vg, fg)
    recs = []
    for res in (24, 40):
        v, f = _mc_mesh('sphere', res)
        recs.append(str(tmp_path / ('rec%d.ply' % res)))
        mesh_io.write_ply(recs[-1], v, f)
    distance_vis.make_distance_comparison(recs, gt, cut_percentil=0.9)
    from source.figure import distance_vis as src_dv
    assert src_dv.make_distance_comparison is distance_vis.make_distance_comparison
    dists = []
    for r in recs:
        v, f = mesh_io.read_ply(r)
        d = np.load(r + '_dist.npy')
        _, d_ref, _ = point_cloud.get_closest_distance_batched(v, (vg, fg))
        assert d.dtype == np.float64 and np.array_equal(d, d_ref)
        # the marching-cubes vertices lie near the sphere of radius 0.6; the icosphere lies within 1.6e-4 of it
        assert np.abs(d - np.abs(np.linalg.norm(v.astype(np.float64), axis=1) - 0.6)).max() <= 2.5e-4
        dists.append(d)
        vo, fo = mesh_io.read_ply(r + '_vis.ply')
        assert np.array_equal(vo, v) and np.array_equal(fo, f)
    cat = np.sort(np.concatenate(dists))
    target = cat[int(len(cat) * 0.9)]
    for r, d in zip(recs, dists):
        assert open(r + '_stats.txt').read() == (
            'Distance from reconstructed mesh vertex to nearest sample on GT mesh, Min={}, Max={}, Mean={}, normalized to '
            '{}, cut percentil 0.9'.format(np.min(d), np.max(d), np.mean(d), target))
    # one ground-truth mesh per reconstruction gives the same result
    distance_vis.make_distance_comparison(recs, [gt, gt], cut_percentil=0.9)
    for r, d in zip(recs, dists):
        assert np.array_equal(np.load(r + '_dist.npy'), d)
