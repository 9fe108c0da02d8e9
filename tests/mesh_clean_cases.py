"""Hand-built meshes for the mesh-cleaning tests (tests/test_mesh_clean_host.py on the oracle, tests/test_gpu_mesh_clean.py
on the kernel).  Each case is (verts, faces, expected report fields)."""
import numpy as np

TET_V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
TET_F = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int32)     # outward
CUBE_V = np.array([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], np.float32)
CUBE_F = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1],
                   [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]], np.int32)


def soup(v, f):
    return np.ascontiguousarray(v[f].reshape(-1, 3)), np.arange(3 * len(f), dtype=np.int32).reshape(-1, 3)


def flip(f, rows):
    f = f.copy()
    f[rows] = f[rows][:, ::-1]
    return f


def mobius(n=12, width=0.3):
    t = 2 * np.pi * np.arange(n) / n
    c = np.stack([np.cos(t), np.sin(t), 0 * t], 1)
    w = np.stack([np.cos(t / 2) * np.cos(t), np.cos(t / 2) * np.sin(t), np.sin(t / 2)], 1)
    v = np.concatenate([c + width * w, c - width * w]).astype(np.float32)     # a_i = i, b_i = n + i
    faces = []
    for i in range(n):
        a0, b0 = i, n + i
        a1, b1 = (i + 1, n + i + 1) if i + 1 < n else (n, 0)                  # the half twist swaps the sides
        faces += [(a0, b0, b1), (a0, b1, a1)]
    return v, np.array(faces, np.int32)


def pentagonal_bipyramid():
    t = 2 * np.pi * np.arange(5) / 5
    ring = np.stack([np.cos(t), np.sin(t), 0 * t], 1)
    v = np.concatenate([ring, [[0, 0, 1], [0, 0, -1]]]).astype(np.float32)
    top = [(i, (i + 1) % 5, 5) for i in range(5)]
    bottom = [((i + 1) % 5, i, 6) for i in range(5)]
    return v, np.array(top + bottom, np.int32)


def cases():
    """name -> (verts, faces, expected report fields)"""
    out = {}
    closed = dict(watertight=True, winding_consistent=True, boundary_edges=0, nonmanifold_edges=0)
    out['tet'] = (TET_V, TET_F, dict(closed, vertices_out=4, faces_out=4, merged_vertices=0, volume=1 / 6))
    out['tet_soup'] = soup(TET_V, TET_F) + (dict(closed, vertices_out=4, faces_out=4, merged_vertices=8),)
    out['cube'] = (CUBE_V, CUBE_F, dict(closed, vertices_out=8, faces_out=12, volume=1.0, faces_reversed=0))
    out['cube_soup'] = soup(CUBE_V, CUBE_F) + (dict(closed, vertices_out=8, faces_out=12, merged_vertices=28),)
    out['cube_one_reversed'] = (CUBE_V, flip(CUBE_F, [5]), dict(closed, faces_reversed=1, winding_consistent_before=False,
                                                               components=1, volume=1.0))
    out['cube_first_reversed'] = (CUBE_V, flip(CUBE_F, [0, 7, 11]), dict(closed, faces_reversed=3, volume=1.0))
    out['cube_inverted'] = (CUBE_V, CUBE_F[:, ::-1].copy(), dict(closed, faces_reversed=0, components=0, volume=-1.0))
    out['tet_missing_triangle'] = (TET_V, TET_F[:3], dict(closed, holes_filled=1, faces_added=1, faces_out=4,
                                                          watertight_before=True, volume=1 / 6))
    out['cube_missing_quad'] = (CUBE_V, CUBE_F[2:], dict(closed, holes_filled=1, faces_added=2, faces_out=12, volume=1.0))
    pv, pf = pentagonal_bipyramid()
    out['missing_pentagon'] = (pv, pf[5:], dict(watertight=False, holes_filled=0, faces_added=0, boundary_edges=5,
                                                vertices_out=6))
    out['duplicates'] = (CUBE_V, np.concatenate([CUBE_F, CUBE_F[[3]], CUBE_F[[6]][:, ::-1], CUBE_F[[3]]]),
                         dict(closed, duplicate_faces=3, faces_out=12))
    sv = np.concatenate([CUBE_V, [[3, 0, 0], [4, 0, 0], [5, 0, 0], [0, 0, 5], [1, 0, 5], [0.5, 1e-9, 5]]]).astype(np.float32)
    out['slivers'] = (sv, np.concatenate([CUBE_F, [[0, 0, 1], [8, 9, 10], [11, 12, 13]]]).astype(np.int32),
                      dict(closed, degenerate_faces=3, unreferenced_vertices=6, vertices_out=8, faces_out=12))
    nv = np.concatenate([CUBE_V, [[7, 7, 7], [np.nan, 0, 0], [8, 8, 8]]]).astype(np.float32)
    out['unreferenced_and_nan'] = (nv, np.concatenate([CUBE_F, [[0, 9, 1]]]).astype(np.int32),
                                   dict(closed, nonfinite_faces=1, unreferenced_vertices=3, vertices_out=8, faces_out=12))
    tv = np.concatenate([TET_V, CUBE_V + 3]).astype(np.float32)
    tf = np.concatenate([flip(TET_F, [2]), CUBE_F[:, ::-1] + 4]).astype(np.int32)
    out['two_bodies_one_inverted'] = (tv, tf, dict(closed, components=2, faces_reversed=13, volume=1 + 1 / 6))
    mv, mf = mobius()
    out['mobius'] = (mv, mf, dict(watertight=False, winding_consistent=False, components=1, nonorientable_components=1,
                                  faces_reversed=0, holes_filled=0, boundary_edges=24))
    fv = np.concatenate([TET_V, [[0.5, -1, -1]]]).astype(np.float32)
    out['three_face_edge'] = (fv, np.concatenate([TET_F, [[0, 1, 4]]]).astype(np.int32),
                              dict(watertight=False, nonmanifold_edges=1, boundary_edges=2, holes_filled=0))
    return out


def canonical(v, f):
    """faces as coordinate triples rotated to start at their smallest vertex (orientation kept), sorted"""
    t = np.asarray(v, np.float64)[np.asarray(f)]
    keys = [tuple(map(tuple, tri)) for tri in t]
    rot = [min(k[i:] + k[:i] for i in range(3)) for k in keys]
    return sorted(rot)
