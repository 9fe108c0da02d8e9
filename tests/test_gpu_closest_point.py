"""GPU tests of p2s_mesh_closest_point_dev (csrc/meshsdf.cu, the unsigned variant of the slab kernel) against the float64
oracle (tests/closest_point_oracle.py), against the signed path it shares its arithmetic with, and for determinism."""
import numpy as np
import pytest
import torch

import closest_point_oracle as cpo
from points2surf_b200 import ops, point_cloud
from test_gpu_mesh_sdf import _fixture, _mc_mesh, _stress_points, _torus_50k, cu

pytestmark = pytest.mark.gpu


def _with_degenerate(f):
    """zero-area faces (a point, a segment) and duplicated faces appended"""
    point = np.stack([f[:20, 0], f[:20, 0], f[:20, 0]], 1)
    seg = np.stack([f[20:40, 0], f[20:40, 1], f[20:40, 0]], 1)
    return np.concatenate([f, point, seg, f[40:60], f[60:70, ::-1]]).astype(np.int32)


def _mesh(case):
    if case.startswith('abc'):
        fx = _fixture(int(case[3]))
        v, f = fx['verts'], fx['faces']
    else:
        kind, res = case.split('_')[:2]
        v, f = _mc_mesh(kind, int(res))
    if case.endswith('_degenerate'):
        f = _with_degenerate(f)
    return v, f


CASES = ['abc0', 'abc1', 'abc2', 'sphere_32', 'torus_40', 'sphere_24_degenerate', 'abc0_degenerate']


@pytest.mark.parametrize('case', CASES)
def test_against_float64_oracle(case):
    v, f = _mesh(case)
    q = _stress_points(v, f, np.random.RandomState(len(f)))
    cp, d, face = (t.cpu().numpy() for t in ops.mesh_closest_point(cu(v), cu(f), cu(q)))
    cp_o, d_o, face_o, d2_o = cpo.mesh_closest_point(v, f, q)
    # 1e-6, relative beyond |d| = 1: the far points (|d| up to ~150) come back in fp32 (half an ulp at 128 is 3.8e-6)
    assert (np.abs(d - d_o) <= 1e-6 * np.maximum(1.0, d_o)).all()
    # the face is the oracle's up to ties within 1e-12
    idx = np.arange(len(q))
    assert (np.sqrt(d2_o[idx, face]) - d_o <= 1e-12).all()
    # the point lies within 1e-6 (1 + |q|_inf) of the oracle's point on the same face
    scale = 1.0 + np.abs(q).max(1)
    same = face == face_o
    assert (np.abs(cp[same] - cp_o[same]).max(1) <= 1e-6 * scale[same]).all()
    on_face = cpo.closest_points_on_faces(v, f, q, face)
    assert (np.abs(cp - on_face).max(1) <= 1e-6 * scale).all()


@pytest.mark.parametrize('case', CASES)
def test_same_arithmetic_as_the_signed_distance(case):
    v, f = _mesh(case)
    q = _stress_points(v, f, np.random.RandomState(len(f) + 1))
    _, d, face = ops.mesh_closest_point(cu(v), cu(f), cu(q))
    ds, fs = ops.mesh_signed_distance(cu(v), cu(f), cu(q), return_face_ids=True)
    assert torch.equal(d, ds.abs()) and torch.equal(face, fs)


def test_large_torus_against_oracle_sample():
    v, f = _torus_50k()
    rng = np.random.RandomState(11)
    fi = rng.choice(len(f), 50000)
    a, b, c = v[f[fi, 0]], v[f[fi, 1]], v[f[fi, 2]]
    r = rng.uniform(0, 1, (50000, 2))
    r[r.sum(1) > 1] = 1 - r[r.sum(1) > 1]
    q = np.concatenate([a + r[:, :1] * (b - a) + r[:, 1:] * (c - a) + rng.normal(0, 0.01, (50000, 3)),
                        rng.uniform(-1, 1, (50000, 3))]).astype(np.float32)
    cp, d, face = (t.cpu().numpy() for t in ops.mesh_closest_point(cu(v), cu(f), cu(q)))
    sel = rng.choice(len(q), 400, replace=False)
    cp_o, d_o, face_o, d2_o = cpo.mesh_closest_point(v, f, q[sel])
    assert np.abs(d[sel] - d_o).max() <= 1e-6
    assert (np.sqrt(d2_o[np.arange(len(sel)), face[sel]]) - d_o <= 1e-12).all()
    on_face = cpo.closest_points_on_faces(v, f, q[sel], face[sel])
    assert np.abs(cp[sel] - on_face).max() <= 1e-6 * (1 + np.abs(q[sel]).max())


def test_deterministic_and_independent_of_the_query_split():
    fx = _fixture(1)
    v, f = cu(fx['verts']), cu(fx['faces'])
    q = np.concatenate([fx['ref_query_pts'], np.random.RandomState(5).uniform(-1, 1, (3001, 3)).astype(np.float32)])
    r1 = [t.cpu().numpy() for t in ops.mesh_closest_point(v, f, cu(q))]
    r2 = [t.cpu().numpy() for t in ops.mesh_closest_point(v, f, cu(q))]
    parts = [[t.cpu().numpy() for t in ops.mesh_closest_point(v, f, cu(q[a:b]))] for a, b in ((0, 999), (999, 1000),
                                                                                                (1000, len(q)))]
    for k in range(3):
        assert r1[k].tobytes() == r2[k].tobytes()
        assert r1[k].tobytes() == np.concatenate([p[k] for p in parts]).tobytes()


def test_errors_and_edge_cases():
    v = cu(np.eye(3, dtype=np.float32))
    f = cu(np.array([[0, 1, 2]], np.int32))
    q = cu(np.array([[0, 0, 0], [np.nan, 0, 0], [1, 0, 0]], np.float32))
    for bad in ([[0, 1, 3]], [[0, -1, 2]]):
        with pytest.raises(ops.P2SError):
            ops.mesh_closest_point(v, cu(np.array(bad, np.int32)), q)
    with pytest.raises(ops.P2SError):
        ops.mesh_closest_point(v, cu(np.zeros((0, 3), np.int32)), q)
    with pytest.raises(ops.P2SError):
        ops.mesh_closest_point(v.cpu(), f, q)
    cp, d, face = ops.mesh_closest_point(v, f, q)
    cp, d, face = cp.cpu().numpy(), d.cpu().numpy(), face.cpu().numpy()
    np.testing.assert_allclose(cp[0], [1 / 3, 1 / 3, 1 / 3], rtol=1e-6)
    assert np.isnan(cp[1]).all() and np.isnan(d[1]) and face[1] == -1
    assert np.array_equal(cp[2], [1, 0, 0]) and d[2] == 0 and face[2] == 0
    out = ops.mesh_closest_point(v, f, q[:0])
    assert [t.shape[0] for t in out] == [0, 0, 0]


def test_get_closest_distance_batched_mirror():
    fx = _fixture(2)
    q = fx['ref_query_pts'].astype(np.float64)
    pts, dists, faces = point_cloud.get_closest_distance_batched(q, (fx['verts'], fx['faces']), batch_size=7, workers=3)
    assert pts.shape == (len(q), 3) and pts.dtype == np.float64
    assert dists.shape == (len(q),) and dists.dtype == np.float64 and faces.dtype == np.int64
    cp, d, face = ops.mesh_closest_point(cu(fx['verts']), cu(fx['faces']), cu(fx['ref_query_pts']))
    assert np.array_equal(pts, cp.cpu().numpy().astype(np.float64))
    assert np.array_equal(dists, d.cpu().numpy().astype(np.float64)) and np.array_equal(faces, face.cpu().numpy())
    np.testing.assert_allclose(dists, np.abs(fx['oracle_dist']), atol=1e-6)
