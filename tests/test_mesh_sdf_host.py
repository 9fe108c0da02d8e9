"""CPU: the training-target stage (make_dataset.py:447-538) -- the float64 signed-distance oracle against the reference's
own 05_query_dist, the host-side random stream of the query points against its 05_query_pts, the file-name hashes, and
the host helpers of the mirror (tests/golden/mesh_sdf.npz, written by tests/golden/make_mesh_sdf_golden.py)."""
import numpy as np
import pytest

from oracle import mesh_sdf_oracle as msdf
from points2surf_b200 import make_dataset, sdf, ops
from helpers import load_golden


@pytest.mark.parametrize('i', [0, 1, 2])
def test_oracle_matches_reference_distances(i):
    g = load_golden('mesh_sdf.npz')
    q, d_ref = g['ref_query_pts_%d' % i], g['ref_query_dist_%d' % i]
    # 150 far and 150 close points (the close half is where sign and distance are delicate)
    rng = np.random.RandomState(i)
    n = len(q) // 2
    sel = np.concatenate([rng.choice(n, 150, replace=False), n + rng.choice(len(q) - n, 150, replace=False)])
    d, face, w = msdf.mesh_signed_distance(g['verts_%d' % i], g['faces_%d' % i], q[sel])
    assert np.array_equal(np.sign(d), np.sign(d_ref[sel]))
    assert np.abs(np.abs(d) - np.abs(d_ref[sel])).max() <= 1e-5
    # the fixture's oracle columns are this oracle's output
    np.testing.assert_allclose(d, g['oracle_dist_%d' % i][sel], rtol=0, atol=1e-12)
    assert np.array_equal(face, g['oracle_face_%d' % i][sel])


@pytest.mark.parametrize('i', [0, 1, 2])
def test_far_points_are_the_reference_stream(i):
    g = load_golden('mesh_sdf.npz')
    q = g['ref_query_pts_%d' % i]
    rng = np.random.RandomState(int(g['hash_%d' % i]))
    offset, far = sdf._query_pts_rng_draws(rng, len(q), float(g['patch_radius']), float(g['far_query_pts_ratio']))
    assert far.shape == (len(q) // 2, 3) and offset.shape == (len(q) - len(q) // 2,)
    assert np.array_equal(far.astype(np.float32), q[:len(far)])
    assert np.abs(offset).max() <= float(g['patch_radius'])


def test_filename_to_hash_matches_reference(tmp_path):
    g = load_golden('mesh_sdf.npz')
    for i in range(3):
        p = tmp_path / str(g['name_%d' % i])
        p.write_bytes(b'')
        assert make_dataset.filename_to_hash(str(p)) == int(g['hash_%d' % i])
    with pytest.raises(ValueError):
        make_dataset.filename_to_hash(str(tmp_path / 'missing.ply'))


def test_oracle_degenerate_faces_and_ties():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 0, 0]], np.float64)
    f = np.array([[0, 1, 2], [0, 1, 3], [1, 1, 1], [0, 1, 2]])     # collinear, a point, a duplicate
    q = np.array([[0.25, 0.25, 1.0], [1.5, 0.0, 0.0], [1.0, 0.0, 0.0], [5.0, 0.0, 0.0]])
    d, face, w = msdf.mesh_signed_distance(v, f, q)
    np.testing.assert_allclose(np.abs(d), [1.0, 0.0, 0.0, 3.0], atol=1e-15)
    assert list(face) == [0, 1, 0, 1]           # lowest index among equal distances
    assert np.isfinite(w).all()


def test_orient_outward_flips_inverted_meshes():
    # a tetrahedron, outward, then every face reversed
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    f = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int32)
    assert sdf._orient_outward(v, f) is f
    assert np.array_equal(sdf._orient_outward(v, f[:, ::-1].copy()), f)
    _, _, w = msdf.mesh_signed_distance(v, f, np.array([[0.1, 0.1, 0.1]]))
    assert abs(w[0] - 1.0) < 1e-12


def test_mesh_arguments_are_validated():
    v = np.zeros((3, 3), np.float32)
    with pytest.raises(ops.P2SError):
        sdf._mesh_arrays((v, np.array([[0, 1, 3]])))
    with pytest.raises(ops.P2SError):
        sdf._mesh_arrays((v, np.zeros((0, 3), np.int32)))

    class M:
        vertices, faces = v, np.array([[0, 1, 2]])
    vv, ff = sdf._mesh_arrays(M())
    assert vv.dtype == np.float32 and ff.dtype == np.int32 and ff.shape == (1, 3)
