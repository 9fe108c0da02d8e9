"""CPU tests of the scan stage: the restated scan-pose stream against the reference's own sample_blensor
(tests/golden/scan.npz), the quaternion helpers, the float64 scan oracle (oracle/scan_oracle.py) on hand-built cases, and
the file layout of make_dataset.sample_blensor with ops.range_scan stubbed."""
import os

import numpy as np
import pytest
import torch

from oracle import scan_oracle as so
from points2surf_b200 import make_dataset, mesh_io, ops, trafo
from helpers import load_golden


def _golden(i):
    g = load_golden('scan.npz')
    return {k: g[k + '_%d' % i] for k in ('name', 'num_scans', 'sigma', 'locations', 'rotations', 'ref_num_pts')}


@pytest.mark.parametrize('i', [0, 1, 2])
def test_scan_pose_stream_matches_the_reference(i, tmp_path):
    g = _golden(i)
    mesh = tmp_path / (str(g['name']) + '.ply')
    mesh.write_text('')   # the stream depends on the file name only
    sigma, loc, rot = make_dataset.get_scan_poses(str(mesh), 5, 30, 0.0, 0.05)
    assert len(loc) == len(rot) == int(g['num_scans'])
    assert sigma == g['sigma']
    assert np.array_equal(loc, g['locations']) and np.array_equal(rot, g['rotations'])


def test_quaternion_helpers():
    rng = np.random.RandomState(0)
    for _ in range(200):
        q = trafo.random_quaternion(rng.rand(3))
        assert abs(np.dot(q, q) - 1.0) < 1e-12
        M = trafo.quaternion_matrix(q)
        R = M[:3, :3]
        assert np.allclose(R @ R.T, np.eye(3), atol=1e-12) and abs(np.linalg.det(R) - 1.0) < 1e-12
        assert np.array_equal(M[3], [0, 0, 0, 1]) and np.array_equal(M[:3, 3], [0, 0, 0])
        Ri = trafo.quaternion_matrix(trafo.quaternion_conjugate(q))[:3, :3]
        assert np.allclose(Ri @ R, np.eye(3), atol=1e-12)
        assert np.allclose(trafo.quaternion_matrix(-q), M, atol=1e-12)   # q and -q are the same rotation
        assert np.array_equal(trafo.quaternion_conjugate(trafo.quaternion_conjugate(q)), q)
    # 90 degrees about z: x -> y
    q = np.array([np.cos(np.pi / 4), 0.0, 0.0, np.sin(np.pi / 4)])
    assert np.allclose(trafo.quaternion_matrix(q)[:3, :3] @ [1, 0, 0], [0, 1, 0], atol=1e-15)
    assert np.array_equal(trafo.quaternion_matrix([0.0, 0.0, 0.0, 0.0]), np.eye(4))


def _cube():
    v = np.array([[x, y, z] for x in (-0.5, 0.5) for y in (-0.5, 0.5) for z in (-0.5, 0.5)], np.float32)
    f = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1],
                  [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]], np.int32)
    return v, f


def test_oracle_rays_through_shared_edges_and_vertices_hit_once():
    # a square fan of four triangles around a centre vertex, facing the scanner
    v = np.array([[0.0, -0.5, 0.0], [-0.5, -0.5, -0.5], [0.5, -0.5, -0.5], [0.5, -0.5, 0.5], [-0.5, -0.5, 0.5]], np.float32)
    f = np.array([[0, 2, 1], [0, 3, 2], [0, 4, 3], [0, 1, 4]], np.int32)
    o = np.array([0.0, -4.0, 0.0])
    # the centre vertex (shared by all four faces), the middle of two shared edges, and an interior point
    targets = np.array([[0.0, -0.5, 0.0], [0.25, -0.5, 0.25], [-0.25, -0.5, -0.25], [0.1, -0.5, -0.2]])
    d = targets - o
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    t, face, margin = so.cast(v, f, o, d)
    assert np.all(face >= 0)
    np.testing.assert_allclose(o + d * t[:, None], targets, atol=1e-12)
    assert (margin[:3] < 1e-12).all() and margin[3] > 1e-3
    # ties go to the lowest face index among the faces that contain the point
    for k in range(4):
        on = [j for j in range(len(f)) if _contains(v[f[j]], targets[k])]
        assert face[k] == min(on), (k, face[k], on)
    assert face[3] == 0 and face[0] == 0 and face[1] == 1 and face[2] == 0


def _contains(tri, p):
    a, b, c = tri.astype(np.float64)
    n = np.cross(b - a, c - a)
    if abs(np.dot(p - a, n)) > 1e-12:
        return False
    return all(np.dot(np.cross(y - x, p - x), n) >= -1e-15 for x, y in ((a, b), (b, c), (c, a)))


def test_oracle_watertight_on_a_grid_through_a_closed_mesh():
    # every ray of a dense grid through a closed mesh hits it exactly once on the way in: no ray leaks through the
    # shared edges, whose edge functions are exact negatives of each other
    v, f = _cube()
    s = np.linspace(-0.5, 0.5, 41)
    X, Z = np.meshgrid(s, s)
    d = np.stack([X.ravel(), np.full(X.size, 4.0), Z.ravel()], 1) * 0.25
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    assert np.sum(np.abs(X - Z) < 1e-15) == 41   # 41 rays through the diagonal shared by the two front triangles
    o = np.array([0.0, -4.0, 0.0])
    t, face, _ = so.cast(v, f, o, d)
    hit = o + d * t[:, None]
    assert np.all(face >= 0) and np.allclose(hit[:, 1], -0.5, atol=1e-12)


def test_oracle_miss_cutoff_back_face_and_zero_area():
    v, f = _cube()
    o = np.array([0.0, -4.0, 0.0])
    t, face, _ = so.cast(v, f, o, np.array([[0.0, 0.0, 1.0], [0.0, -1.0, 0.0]]))   # beside and away from the cube
    assert np.all(face == -1) and np.all(np.isinf(t))
    up = np.array([[0.0, 1.0, 0.0]])
    assert so.cast(v, f, o, up, max_distance=3.4)[1][0] == -1          # the front face is 3.5 away
    t, face, _ = so.cast(v, f, o, up, max_distance=3.5)
    assert face[0] >= 0 and t[0] == 3.5
    # from inside, the ray meets the back side of the far face: no back-face culling
    t, face, _ = so.cast(v, f, np.zeros(3), up)
    assert face[0] in (6, 7) and abs(t[0] - 0.5) < 1e-15
    # a zero-area face (collinear vertices) across the ray is never hit; the face behind it is
    v2 = np.concatenate([v, [[-1.0, -1.0, 0.0], [1.0, -1.0, 0.0], [0.0, -1.0, 0.0]]]).astype(np.float32)
    f2 = np.concatenate([[[8, 9, 10]], f]).astype(np.int32)
    t, face, _ = so.cast(v2, f2, o, up)
    assert face[0] >= 1 and abs(t[0] - 3.5) < 1e-15
    # a triangle seen edge-on is not hit either (det == 0)
    v3 = np.array([[0.0, -1.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]], np.float32)
    assert so.cast(v3, np.array([[0, 1, 2]], np.int32), o, up)[1][0] == -1


def test_oracle_scanner_rays():
    o, d = so.scanner_rays(np.eye(3), [0.0, 4.0, 0.0])
    assert np.array_equal(o, [-0.0, -4.0, -0.0]) and d.shape == (176 * 144, 3)
    np.testing.assert_allclose(np.linalg.norm(d, axis=1), 1.0, atol=1e-15)
    assert np.all(d[:, 1] > 0)
    # the wide axis (columns) is z, column 0 at -z; row 0 at +x; the corner rays span the field of view
    assert d[0, 2] < 0 and d[0, 0] > 0 and d[-1, 2] > 0 and d[-1, 0] < 0
    half_w = np.degrees(np.arctan(d[:176, 2] / d[:176, 1]))
    half_h = np.degrees(np.arctan(d[::176, 0] / d[::176, 1]))
    assert abs(half_h[0] - (17.3 - 34.6 / 144 / 2)) < 0.02 and np.allclose(half_h, -half_h[::-1])
    assert abs(half_w[-1] - (21.8 - 43.6 / 176 / 2)) < 0.02 and np.allclose(half_w, -half_w[::-1])
    # a rotation of the pose rotates the rays
    R = trafo.quaternion_matrix(trafo.random_quaternion(np.array([0.3, 0.6, 0.9])))[:3, :3]
    o2, d2 = so.scanner_rays(R, [0.1, 4.0, -0.1])
    np.testing.assert_allclose(d2, d @ R, atol=1e-15)
    np.testing.assert_allclose(R @ o2 + [0.1, 4.0, -0.1], 0.0, atol=1e-15)


def test_sample_blensor_file_layout(tmp_path, monkeypatch):
    g = [_golden(i) for i in range(2)]
    root = tmp_path / 'ds'
    os.makedirs(str(root / '03_meshes'))
    v, f = _cube()
    for gi in g:
        mesh_io.write_ply(str(root / '03_meshes' / (str(gi['name']) + '.ply')), v, f)
    calls = []

    def fake_scan(verts, faces, rotations, locations, noise_sigma=0.0, seed=0, first_scan=0, **kw):
        calls.append((np.asarray(rotations), np.asarray(locations), noise_sigma, seed))
        S = len(locations)
        n = 150 if len(calls) == 1 else 50   # the second mesh stays below min_pts_size
        hps = np.full(S, n // S, np.int32)
        hps[0] += n - hps.sum()
        pts = torch.arange(3 * n, dtype=torch.float32).reshape(n, 3)
        return pts, pts, torch.zeros(n, dtype=torch.int32) + 2, torch.from_numpy(hps)

    monkeypatch.setattr(ops, 'range_scan', fake_scan)
    monkeypatch.setattr(make_dataset.sdf, '_device', lambda: torch.device('cpu'))
    args = (str(tmp_path), 'ds', 'blender', '03_meshes', '04_pts_raw', '04_pts', '04_pts_vis', '04_pcd', '04_blensor_py',
            '04_locations', '04_rotations', 5, 30, 8)
    make_dataset.sample_blensor(*args, min_pts_size=100)
    assert len(calls) == 2
    for k, gi in enumerate(sorted(g, key=lambda x: str(x['name']))):
        stem = str(gi['name'])
        rot, loc, sigma, seed = calls[k]
        assert np.array_equal(loc, gi['locations']) and sigma == gi['sigma']
        for R, q in zip(rot, gi['rotations']):
            assert np.array_equal(R, trafo.quaternion_matrix(q)[:3, :3])
        assert seed == make_dataset.filename_to_hash(str(root / '03_meshes' / (stem + '.ply')))
        assert np.array_equal(np.load(str(root / '04_locations' / (stem + '.npz')))['locations'], gi['locations'])
        assert np.array_equal(np.load(str(root / '04_rotations' / (stem + '.npz')))['rotations'], gi['rotations'])
        hps = np.load(str(root / '04_hits_per_scan' / (stem + '.npz')))['hits_per_scan']
        pts = np.load(str(root / '04_pts' / (stem + '.xyz.npy')))
        assert hps.dtype == np.int32 and len(hps) == gi['num_scans'] and hps.sum() == len(pts)
        assert pts.dtype == np.float32 and pts.shape[1] == 6
        assert np.array_equal(pts[:, 3:], np.tile(make_dataset.face_normals(v, f)[2], (len(pts), 1)))
        vis = root / '04_pts_vis' / (stem + '.xyz')
        assert vis.exists() == (len(pts) > 100)
        if vis.exists():
            assert np.array_equal(np.loadtxt(str(vis)).astype(np.float32), pts[:, :3])
    for d in ('04_pts_raw', '04_pcd', '04_blensor_py'):
        assert not (root / d).exists()
    # up-to-date outputs are skipped
    make_dataset.sample_blensor(*args, min_pts_size=100)
    assert len(calls) == 2
