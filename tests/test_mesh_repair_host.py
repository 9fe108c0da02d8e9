"""CPU tests of the mesh repair oracle (oracle/mesh_repair_oracle.py, the rules of p2s_mesh_repair_dev in
include/p2s_b200.h) against hand-computed expectations and brute-force invariants."""
import collections

import numpy as np
import pytest

from oracle import mesh_repair_oracle as mro
from helpers import load_golden
import mesh_repair_cases as mrc


def edge_count(f):
    c = collections.Counter()
    for t in np.asarray(f).tolist():
        for k in range(3):
            c[frozenset((t[k], t[(k + 1) % 3]))] += 1
    return c


def half_edges(f):
    return collections.Counter((t[k], t[(k + 1) % 3]) for t in np.asarray(f).tolist() for k in range(3))


def assert_invariants(f_in, v_out, f_out, st):
    """no edge with more than two faces, one fan per vertex, and every fill face consistent with its neighbours"""
    assert max(edge_count(f_out).values()) <= 2
    for x, comps in mro.fans(np.asarray(f_out, np.int64)).items():
        assert len(comps) == 1, x
    kept = len(f_out) - st['faces_added']
    he = half_edges(f_out)
    for t in f_out[kept:].tolist():
        for k in range(3):
            a, b = t[k], t[(k + 1) % 3]
            assert he[(a, b)] == 1 and he[(b, a)] == 1, (a, b)   # closed against the old faces or the next fill face


def test_cube_holes_close_up_to_30_edges():
    v, f, sizes = mrc.cube_with_holes()
    assert sum(1 for c in edge_count(f).values() if c == 1) == sum(k * n for k, n in sizes.items())
    vo, fo, st = mro.mesh_repair(v, f)
    assert st['holes_closed'] == 5 and st['holes_left_open'] == 1
    assert st['faces_added'] == sum(k - 2 for k in sizes if k <= 30)        # a planar n-gon gains n - 2 faces
    assert st['faces_removed'] == 0 and st['vertices_split'] == 0
    assert np.array_equal(fo[:len(f)], f) and vo.tobytes() == v.tobytes()
    assert sum(1 for c in edge_count(fo).values() if c == 1) == 31            # only the 31-edge hole is open
    assert_invariants(f, vo, fo, st)
    _, _, st29 = mro.mesh_repair(v, f, max_hole_size=29)
    assert st29['holes_closed'] == 4 and st29['holes_left_open'] == 2


@pytest.mark.parametrize('k', [3, 4])
@pytest.mark.parametrize('tied', [False, True])
def test_nonmanifold_edges_drop_the_smallest_faces(k, tied):
    v, f = mrc.fins(k, tied)
    vo, fo, st = mro.mesh_repair(v, f)
    area = mro.area2(v.astype(np.float64), f.astype(np.int64))
    # brute force: keep the two largest, ties to the lower index
    expect = sorted(sorted(range(k), key=lambda i: (-area[i], i))[:2])
    assert np.array_equal(fo[:2], f[expect]) and st['faces_removed'] == k - 2
    # rule 2 is a no-op: after rule 1 no edge has more than two faces
    assert max(edge_count(fo[:2]).values()) <= 2
    assert_invariants(f, vo, fo, st)


def test_bowtie_vertex_is_split_into_one_copy():
    v, f = mrc.bowtie()
    vo, fo, st = mro.mesh_repair(v, f)
    assert st['vertices_split'] == 1 and len(vo) == len(v) + 1 and vo[-1].tobytes() == v[0].tobytes()
    assert (fo[:6] == f[:6]).all()                          # the fan of face 0 keeps vertex 0
    assert (fo[6:12, 0] == len(v)).all() and (fo[6:12, 1:] == f[6:12, 1:]).all()
    assert st['holes_closed'] == 2 and st['faces_added'] == 8
    assert_invariants(f, vo, fo, st)


def test_concave_planar_loop_skips_the_self_intersecting_ear():
    v, f = mrc.planar_annulus(mrc.CHEVRON)
    vo, fo, st = mro.mesh_repair(v, f)
    inner = fo[len(f):len(f) + 2]
    # the sharpest convex ear, at the tip (vertex 0), holds the notch (vertex 2): it must not be cut first
    P = np.array(mrc.CHEVRON)
    ang = {}
    for i in range(4):
        a, b = P[i - 1] - P[i], P[(i + 1) % 4] - P[i]
        if a[1] * b[0] - a[0] * b[1] > 0:
            ang[i] = np.arccos(a @ b / np.linalg.norm(a) / np.linalg.norm(b))
    assert min(ang, key=ang.get) == 0
    assert inner[0][1] != 0 and inner.tolist() == [[0, 1, 2], [3, 0, 2]]
    # the fill tiles the hole: its 2D area equals the polygon's and both faces are counter-clockwise
    x, y = P[:, 0], P[:, 1]
    poly = 0.5 * np.sum(x * np.roll(y, -1) - np.roll(x, -1) * y)
    tri = [0.5 * ((P[b] - P[a])[0] * (P[c] - P[a])[1] - (P[b] - P[a])[1] * (P[c] - P[a])[0]) for a, b, c in inner]
    assert min(tri) > 0 and np.isclose(sum(tri), poly)
    assert_invariants(f, vo, fo, st)


def test_loop_without_a_valid_ear_stays_open():
    v, f = mrc.spiked_pyramid()
    vo, fo, st = mro.mesh_repair(v, f)
    assert st['holes_left_open'] == 1 and st['holes_closed'] == 0 and st['faces_added'] == 0
    assert np.array_equal(fo, f)
    # brute force: each of the four ears of the square is crossed by a face around the loop
    P = [tuple(map(float, p)) for p in v]
    for a, b, c in [(3, 0, 1), (0, 1, 2), (1, 2, 3), (2, 3, 0)]:
        assert any(mro.tri_cross((P[a], P[b], P[c]), tuple(P[i] for i in t)) for t in f.tolist())
    # without the intersection test the same loop closes
    _, fo2, st2 = mro.mesh_repair(v, f, prevent_self_intersection=False)
    assert st2['holes_closed'] == 1 and st2['faces_added'] == 2


@pytest.mark.parametrize('i', [0, 1, 2])
def test_abc_minimal_with_deleted_faces_keeps_the_invariants(i):
    g = load_golden('mesh_sdf.npz')
    v, f = g['verts_%d' % i].astype(np.float32), g['faces_%d' % i].astype(np.int32)
    vo, fo, st = mro.mesh_repair(v, f)
    assert np.array_equal(fo, f) and st['faces_added'] == 0 and st['holes_left_open'] == 0
    f2 = mrc.delete_random_faces(f, seed=i)
    vo, fo, st = mro.mesh_repair(v, f2)
    assert st['holes_closed'] >= 1
    assert_invariants(f2, vo, fo, st)


def test_bad_input_raises():
    v, f = mrc.bowtie()
    with pytest.raises(ValueError):
        mro.mesh_repair(v, np.array([[0, 1, 99]]))
    with pytest.raises(ValueError):
        mro.mesh_repair(v, np.array([[0, 1, 1]]))
    with pytest.raises(ValueError):
        mro.mesh_repair(v, f, max_hole_size=129)
