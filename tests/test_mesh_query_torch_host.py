"""CPU: the float64 torch restatement of the mesh queries (tests/mesh_query_torch.py) against the NumPy oracles
(oracle/mesh_sdf_oracle.py, tests/closest_point_oracle.py) to 1e-12, on the abc_minimal fixtures and on random meshes with
zero-area (point, segment, collinear) and duplicated faces, and with chunks smaller than the query and face counts."""
import numpy as np
import pytest
import torch

import closest_point_oracle as cpo
import mesh_query_torch as mqt
from helpers import load_golden
from oracle import mesh_sdf_oracle as msdf
from test_closest_point_host import _random_mesh


def _abc_case(i, degenerate):
    g = load_golden('mesh_sdf.npz')
    v, f = g['verts_%d' % i], g['faces_%d' % i]
    rng = np.random.RandomState(i)
    q = g['ref_query_pts_%d' % i][rng.choice(len(g['ref_query_pts_%d' % i]), 120, replace=False)]
    q = np.concatenate([q, v[f[:10, 0]], 0.5 * (v[f[10:20, 0]] + v[f[10:20, 1]]), rng.normal(size=(10, 3)) * 20])
    if degenerate:   # a point, segments and duplicated faces (one reversed)
        f = np.concatenate([f, np.stack([f[:5, 0]] * 3, 1), np.stack([f[5:10, 0], f[5:10, 1], f[5:10, 0]], 1), f[20:30],
                            f[30:35, ::-1]])
    return v, f.astype(np.int32), q.astype(np.float32)


def _random_case(seed):
    rng = np.random.RandomState(seed)
    v, f = _random_mesh(rng)
    q = np.concatenate([rng.normal(size=(150, 3)) * 2, v, 0.5 * (v[f[:, 0]] + v[f[:, 1]]), rng.normal(size=(10, 3)) * 50])
    return v, f, q.astype(np.float32)


CASES = {'abc0': lambda: _abc_case(0, False), 'abc1_degenerate': lambda: _abc_case(1, True),
         'random0': lambda: _random_case(0), 'random1': lambda: _random_case(1), 'random2': lambda: _random_case(2),
         'ties': lambda: (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 0, 0]], np.float32),
                          np.array([[0, 1, 2], [0, 1, 3], [1, 1, 1], [0, 1, 2]], np.int32),
                          np.array([[0.25, 0.25, 1.0], [1.5, 0.0, 0.0], [1.0, 0.0, 0.0], [5.0, 0.0, 0.0],
                                    [0.25, 0.25, -1.0]], np.float32))}


@pytest.mark.parametrize('pairs', [1 << 22, 1000])
@pytest.mark.parametrize('case', sorted(CASES))
def test_torch_reference_equals_numpy_oracles(case, pairs):
    v, f, q = CASES[case]()
    r = {k: t.numpy() for k, t in mqt.mesh_query(torch.from_numpy(v), torch.from_numpy(f), q, pairs=pairs).items()}
    d_o, face_o, w_o = msdf.mesh_signed_distance(v, f, q)
    cp_o, du_o, fu_o, d2_o = cpo.mesh_closest_point(v, f, q)
    scale = 1.0 + np.abs(q).max(1)
    assert np.abs(r['d'] - du_o).max() <= 1e-12 * scale.max()
    assert np.abs(r['signed'] - d_o).max() <= 1e-12 * scale.max()
    off = du_o > 1e-6   # on the surface the winding number jumps: its value there is a matter of rounding
    assert np.abs(r['w'] - w_o)[off].max() <= 1e-12
    # the face is the oracles' up to float64 ties
    idx = np.arange(len(q))
    assert np.array_equal(face_o, fu_o)
    assert (np.sqrt(d2_o[idx, r['face']]) - du_o <= 1e-12 * scale).all()
    assert (r['face'] == face_o).mean() > 0.97
    # the point on the face it returns is the oracle's point on that face
    on_face = cpo.closest_points_on_faces(v, f, q, r['face'])
    assert np.abs(r['closest'] - on_face).max() <= 1e-12 * scale.max()
    np.testing.assert_allclose(mqt.face_dist2(torch.from_numpy(v), torch.from_numpy(f), q, r['face']).numpy(),
                               r['d'] ** 2, rtol=0, atol=1e-12 * scale.max() ** 2)


def test_ties_take_the_lowest_face():
    v, f, q = CASES['ties']()
    r = mqt.mesh_query(v, f, q, pairs=2)
    assert r['face'].tolist() == [0, 1, 0, 1, 0]
    np.testing.assert_allclose(r['d'].numpy(), [1, 0, 0, 3, 1], atol=1e-15)
    assert r['signed'][4] == -1.0 and r['signed'][1] == 0.0
