"""Hand-built meshes for the mesh repair tests (test_mesh_repair_host.py, test_gpu_mesh_repair.py).  Every builder
returns (verts [V,3] float32, faces [F,3] int32) with exactly representable coordinates."""
import numpy as np


def grid_cube(n=10):
    """the surface of [0, n]^3 as six n x n grids of quads, two outward triangles per quad.  -> (verts, faces, quads)
    where quads[side][i][j] = (face index of the first triangle, of the second)."""
    verts, index = [], {}

    def vid(p):
        if p not in index:
            index[p] = len(verts)
            verts.append(p)
        return index[p]

    faces, quads = [], []
    # (origin, axis u, axis v) with u x v pointing out of the cube
    sides = [((0, 0, 0), (0, 1, 0), (1, 0, 0)), ((0, 0, n), (1, 0, 0), (0, 1, 0)),
             ((0, 0, 0), (1, 0, 0), (0, 0, 1)), ((0, n, 0), (0, 0, 1), (1, 0, 0)),
             ((0, 0, 0), (0, 0, 1), (0, 1, 0)), ((n, 0, 0), (0, 1, 0), (0, 0, 1))]
    for o, u, w in sides:
        q = []
        for i in range(n):
            row = []
            for j in range(n):
                def p(a, b):
                    return vid(tuple(o[k] + a * u[k] + b * w[k] for k in range(3)))
                a, b, c, d = p(i, j), p(i + 1, j), p(i + 1, j + 1), p(i, j + 1)
                row.append((len(faces), len(faces) + 1))
                faces += [(a, b, c), (a, c, d)]
            q.append(row)
        quads.append(q)
    return np.array(verts, np.float32), np.array(faces, np.int32), quads


def cube_with_holes():
    """grid_cube(10) with holes of 3, 4, 5, 12, 30 and 31 boundary edges (the last stays open at MaxHoleSize 30).
    -> (verts, faces, {hole size: number of such holes})"""
    v, f, q = grid_cube(10)
    drop = [q[0][2][2][0]]                                          # 3: one triangle
    drop += list(q[0][6][6])                                        # 4: one quad
    drop += list(q[1][2][2]) + [q[1][3][2][1]]                      # 5: a quad and a triangle of its neighbour
    drop += [t for i in range(4, 7) for j in range(4, 7) for t in q[2][i][j]]              # 12: 3 x 3 quads
    drop += [t for i in range(1, 8) for j in range(1, 9) for t in q[3][i][j]]              # 30: 7 x 8 quads
    drop += [t for i in range(1, 8) for j in range(1, 9) for t in q[4][i][j]] + [q[4][8][4][1]]   # 31
    keep = np.ones(len(f), bool)
    keep[drop] = False
    return v, f[keep], {3: 1, 4: 1, 5: 1, 12: 1, 30: 1, 31: 1}


def fins(k, tied):
    """k <= 4 faces on the edge (0, 1), fin i of height 1 + i (all of height 1, equal areas, when tied)"""
    v = [(0, 0, 0), (4, 0, 0)]
    f = []
    for i, (y, z) in enumerate([(1, 0), (0, 1), (-1, 0), (0, -1)][:k]):
        h = 1.0 if tied else 1.0 + i
        v.append((2, h * y, h * z))
        f.append((0, 1, 2 + i) if i % 2 == 0 else (1, 0, 2 + i))
    return np.array(v, np.float32), np.array(f, np.int32)


def _cone(apex_z, base_z, n, first):
    v = [(0.0, 0.0, apex_z)] if first else []
    ring = []
    for i in range(n):
        ang = 2 * np.pi * i / n
        ring.append((round(2 * np.cos(ang), 3), round(2 * np.sin(ang), 3), base_z))
    return v + ring


def bowtie():
    """two cones sharing their apex (vertex 0): one vertex with two fans, and two 6-edge holes (the cone bases)"""
    v = _cone(0.0, 2.0, 6, True) + _cone(0.0, -2.0, 6, False)
    f = [(0, 1 + i, 1 + (i + 1) % 6) for i in range(6)] + [(0, 7 + (i + 1) % 6, 7 + i) for i in range(6)]
    return np.array(v, np.float32), np.array(f, np.int32)


CHEVRON = [(6.0, 0.0), (0.0, 1.0), (1.0, 0.0), (0.0, -1.0)]   # counter-clockwise; the sharp tip's ear holds the notch


def planar_annulus(poly, centre=(0.5, 0.0), scale=3.0):
    """a flat ring of faces (z = 0) around the hole `poly` (counter-clockwise, star-shaped about `centre`), normals +z"""
    n = len(poly)
    inner = [(x, y, 0.0) for x, y in poly]
    outer = [(centre[0] + scale * (x - centre[0]), centre[1] + scale * (y - centre[1]), 0.0) for x, y in poly]
    f = []
    for i in range(n):
        j = (i + 1) % n
        f += [(i, n + i, n + j), (i, n + j, j)]
    return np.array(inner + outer, np.float32), np.array(f, np.int32)


def spiked_pyramid():
    """an open pyramid over the square hole (0,0)-(1,1) at z = 0 with apex E above it; two spikes reach from E through
    the hole's plane so that every ear of the square is pierced by an edge E-S of a face around a loop vertex: the loop
    has no valid ear and stays open."""
    v = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0.5, 0.5, 1.0), (0.7, 0.1, -1.0), (0.4, 0.8, -1.0)]
    A, B, C, D, E, S, S2 = range(7)
    f = [(A, B, S), (B, E, S), (E, A, S), (B, C, E), (C, D, S2), (D, E, S2), (E, C, S2), (D, A, E)]
    return np.array(v, np.float32), np.array(f, np.int32)


def cases():
    """name -> (verts, faces)"""
    out = {'cube_holes': cube_with_holes()[:2], 'bowtie': bowtie(), 'chevron': planar_annulus(CHEVRON),
           'no_valid_ear': spiked_pyramid()}
    for k in (3, 4):
        for tied in (False, True):
            out['fins%d_%s' % (k, 'tied' if tied else 'distinct')] = fins(k, tied)
    return out


def delete_random_faces(f, seed, n_sets=4, size=3):
    """remove `n_sets` random patches of `size` edge-connected faces (grown breadth-first from a random face)"""
    rng = np.random.RandomState(seed)
    f = np.asarray(f)
    by_edge = {}
    for i, t in enumerate(f.tolist()):
        for k in range(3):
            by_edge.setdefault(frozenset((t[k], t[(k + 1) % 3])), []).append(i)
    keep = np.ones(len(f), bool)
    for _ in range(n_sets):
        patch, queue = [], [int(rng.randint(len(f)))]
        while queue and len(patch) < size:
            i = queue.pop(0)
            if i in patch:
                continue
            patch.append(i)
            t = f[i].tolist()
            queue += [j for k in range(3) for j in by_edge[frozenset((t[k], t[(k + 1) % 3]))] if j != i]
        keep[patch] = False
    return f[keep]
