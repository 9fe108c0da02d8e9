"""CPU tests of the closest-point evaluation stages: the float64 closest-point oracle (tests/closest_point_oracle.py)
against brute force, and the host parts of the distance maps and ground-truth normals against the unmodified
reference's results (tests/golden/distance_vis.npz, written by tests/golden/make_distance_vis_golden.py)."""
import numpy as np
import pytest

from oracle import mesh_sdf_oracle as msdf
import closest_point_oracle as cpo
from helpers import load_golden
from points2surf_b200 import mesh_io, point_cloud
from points2surf_b200.figure import distance_vis

CUTS = (0.9, 0.5, 0.0, 0.999, 1.0, None)


def _random_mesh(rng, nv=30, nf=60, degenerate=True):
    v = rng.normal(size=(nv, 3))
    f = np.stack([rng.choice(nv, 3, replace=False) for _ in range(nf)])
    if degenerate:   # a point, segments, a collinear triangle and duplicated faces (one reversed)
        v = np.concatenate([v, [v[0] + 0.5 * (v[1] - v[0])]])
        f = np.concatenate([f, [[2, 2, 2], [3, 4, 3], [5, 5, 6], [0, 1, nv]], f[:3], f[3:5, ::-1]])
    return v.astype(np.float32), f.astype(np.int32)


def _brute_force(v, f, q):
    """closest point on every face by the kernel's rule (plane projection when inside, else the first nearest edge),
    minimum over all faces -> (points [Q,3], dist [Q], face [Q], d2 [Q,F])"""
    v = v.astype(np.float64)
    q = q.astype(np.float64)
    d2 = np.empty((len(q), len(f)))
    pts = np.empty((len(q), len(f), 3))
    for j, (ia, ib, ic) in enumerate(f):
        a, b, c = v[ia], v[ib], v[ic]
        n = np.cross(b - a, c - a)
        cands = [cpo._seg_closest(q, a, b), cpo._seg_closest(q, b, c), cpo._seg_closest(q, c, a)]
        de = np.stack([((q - x) ** 2).sum(1) for x in cands], 1)
        k = np.argmin(de, 1)
        best = np.stack(cands, 1)[np.arange(len(q)), k]
        if (n != 0).any():
            inside = np.ones(len(q), bool)
            for s, e in ((a, b), (b, c), (c, a)):
                inside &= (np.cross(e - s, q - s) @ n) >= 0
            proj = q - ((q - a) @ n / (n @ n))[:, None] * n
            best = np.where(inside[:, None], proj, best)
        pts[:, j] = best
        d2[:, j] = ((q - best) ** 2).sum(1)
    face = np.argmin(d2, 1)
    idx = np.arange(len(q))
    return pts[idx, face], np.sqrt(d2[idx, face]), face, d2


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_oracle_matches_brute_force(seed):
    rng = np.random.RandomState(seed)
    v, f = _random_mesh(rng)
    fi = rng.randint(0, len(f), 40)
    a, b, c = (v[f[fi, k]].astype(np.float64) for k in range(3))
    r = rng.uniform(0, 1, (40, 2))
    r[r.sum(1) > 1] = 1 - r[r.sum(1) > 1]
    q = np.concatenate([rng.normal(size=(200, 3)) * 2, v[:10], 0.5 * (a + b), a + r[:, :1] * (b - a) + r[:, 1:] * (c - a),
                        rng.normal(size=(20, 3)) * 50]).astype(np.float32)
    cp, d, face, d2 = cpo.mesh_closest_point(v, f, q)
    bp, bd, bface, bd2 = _brute_force(v, f, q)
    assert np.abs(d - bd).max() <= 1e-12 * (1 + np.abs(q).max())
    # the face is the brute-force one up to ties, and the point lies on it
    gap = np.sqrt(bd2[np.arange(len(q)), face]) - bd
    assert np.abs(gap).max() <= 1e-12 * (1 + np.abs(q).max())
    same = face == bface
    assert same.mean() > 0.9
    assert np.abs(cp[same] - bp[same]).max() <= 1e-9 * (1 + np.abs(q).max())
    assert np.abs(np.sqrt(((cp - q) ** 2).sum(1)) - d).max() <= 1e-12 * (1 + np.abs(q).max())
    # the distances are the signed-distance oracle's: bit for bit on faces with area, within rounding elsewhere
    ds, fs, _ = msdf.mesh_signed_distance(v, f, q)
    assert np.abs(np.abs(ds) - d).max() <= 1e-14 * (1 + np.abs(q).max())
    zero = msdf._edges_zero_area(*(v[f[:, k]].astype(np.float64) for k in range(3)))
    nz = ~zero[face]
    assert np.array_equal(np.abs(ds)[nz & (fs == face)], d[nz & (fs == face)])
    # no point of the winning face is closer than the oracle's point
    rr = rng.uniform(0, 1, (len(q), 64, 2))
    rr[rr.sum(2) > 1] = 1 - rr[rr.sum(2) > 1]
    fa, fb, fc = (v[f[face, k]].astype(np.float64)[:, None] for k in range(3))
    s = fa + rr[..., :1] * (fb - fa) + rr[..., 1:] * (fc - fa)
    ds2 = np.sqrt(((s - q.astype(np.float64)[:, None]) ** 2).sum(2)).min(1)
    assert (ds2 >= d - 1e-12).all()


def test_oracle_degenerate_faces_are_edges():
    v = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [5, 5, 5]], np.float32)
    f = np.array([[0, 1, 2], [3, 3, 3]], np.int32)            # a collinear triangle and a point
    q = np.array([[0.5, 1, 0], [3, 0, 0], [5, 5, 6], [-1, -1, 0]], np.float32)
    cp, d, face, _ = cpo.mesh_closest_point(v, f, q)
    np.testing.assert_array_equal(cp, [[0.5, 0, 0], [2, 0, 0], [5, 5, 5], [0, 0, 0]])
    np.testing.assert_array_equal(face, [0, 0, 1, 0])
    np.testing.assert_allclose(d, [1, 1, 1, np.sqrt(2)], rtol=1e-15)


def test_normalization_target_matches_reference():
    g = load_golden('distance_vis.npz')
    dists = [g['dist_%d' % i] for i in range(3)]
    for k, cut in enumerate(CUTS):
        t = distance_vis.get_normalization_target(dists, cut_percentil=cut)
        assert t == g['target_%d' % k] and type(t) is np.float64
        assert distance_vis.get_normalization_target(dists[1:2], cut_percentil=cut) == g['target_single_%d' % k]


def test_stats_text_and_outputs_match_reference(tmp_path):
    g = load_golden('distance_vis.npz')
    v = np.random.RandomState(0).rand(1001, 3).astype(np.float32)
    f = np.array([[0, 1, 2]], np.int32)
    for i in range(3):
        d = g['dist_%d' % i]
        mesh_file = str(tmp_path / ('rec%d.ply' % i))
        distance_vis.visualize_mesh_with_distances(mesh_file, (v[:len(d)], f), d, g['target_0'], cut_percentil=0.9)
        assert open(mesh_file + '_stats.txt').read() == str(g['stats_%d' % i])
        assert np.array_equal(np.load(mesh_file + '_dist.npy'), d)
        vo, fo = mesh_io.read_ply(mesh_file + '_vis.ply')
        assert np.array_equal(vo, v[:len(d)]) and np.array_equal(fo, f)
        assert b'property uchar red' in open(mesh_file + '_vis.ply', 'rb').read(400)


def test_distance_colors_ramp():
    ramp = distance_vis.COLOR_RAMP
    c = distance_vis.distance_colors(np.array([0.0, 0.5, 1.0, 7.0, 0.999]), 1.0)
    np.testing.assert_array_equal(c[0], ramp[0])
    np.testing.assert_array_equal(c[1], ramp[127])     # int(0.5 * 255)
    np.testing.assert_array_equal(c[2], ramp[255])
    np.testing.assert_array_equal(c[3], ramp[255])     # beyond the target: clamped
    np.testing.assert_array_equal(c[4], ramp[254])
    assert ramp[0][2] > ramp[0][1] and ramp[127][1] > ramp[127][2] and ramp[255][0] > ramp[255][2]   # blue, green, yellow
    np.testing.assert_array_equal(distance_vis.distance_colors(np.zeros(3), 0.0), ramp[[0, 0, 0]])


@pytest.mark.parametrize('case', ['pts32_normals', 'pts32', 'pts64_normals', 'pts2d', 'ptsT'])
def test_write_xyz_matches_reference(tmp_path, case):
    g = load_golden('distance_vis.npz')
    args = {'pts32_normals': (g['xyz_pts32'], g['xyz_nrm64']), 'pts32': (g['xyz_pts32'], None),
            'pts64_normals': (g['xyz_pts64'], g['xyz_nrm64'][:5]), 'pts2d': (g['xyz_pts2d'], None),
            'ptsT': (g['xyz_ptsT'], None)}[case]
    path = str(tmp_path / 'sub' / (case + '.xyz'))
    point_cloud.write_xyz(path, args[0], normals=args[1])
    assert open(path).read() == str(g['xyz_text_' + case])


def test_source_shims_reexport_the_mirrors():
    from source.base import point_cloud as src_pc
    from source.figure import distance_vis as src_dv
    assert src_pc.get_closest_distance_batched is point_cloud.get_closest_distance_batched
    assert src_pc.write_xyz is point_cloud.write_xyz
    assert src_dv.make_distance_comparison is distance_vis.make_distance_comparison
    assert src_dv.get_normalization_target is distance_vis.get_normalization_target
