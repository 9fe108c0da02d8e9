"""Closed test meshes of the solid voxelisation (csrc/inside.cu, oracle/inside_oracle.py): an icosphere, a torus, the
three abc_minimal meshes of tests/golden/mesh_sdf.npz, and an axis-aligned box and an octahedron whose corners, edges
and (for the box) faces lie exactly on voxel centres of a res-16 grid."""
import os

import numpy as np

from oracle import inside_oracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def icosphere(radius=0.45, level=4):
    t = (1.0 + 5 ** 0.5) / 2.0
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t),
         (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
         (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7),
         (9, 8, 1)]
    v = [np.array(p, np.float64) / np.linalg.norm(p) for p in v]
    for _ in range(level):
        mid = {}

        def m(a, b):
            key = (min(a, b), max(a, b))
            if key not in mid:
                p = v[a] + v[b]
                v.append(p / np.linalg.norm(p))
                mid[key] = len(v) - 1
            return mid[key]
        nf = []
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        f = nf
    return (np.array(v) * radius).astype(np.float32), np.array(f, np.int32)


def torus(R=0.5, r=0.2, n=48, m=24):
    u = np.arange(n) * 2 * np.pi / n
    w = np.arange(m) * 2 * np.pi / m
    U, W = np.meshgrid(u, w, indexing='ij')
    v = np.stack([(R + r * np.cos(W)) * np.cos(U), (R + r * np.cos(W)) * np.sin(U), r * np.sin(W)], -1).reshape(-1, 3)
    f = []
    for i in range(n):
        for j in range(m):
            a, b = i * m + j, ((i + 1) % n) * m + j
            c, d = ((i + 1) % n) * m + (j + 1) % m, i * m + (j + 1) % m
            f += [(a, b, c), (a, c, d)]
    return v.astype(np.float32), np.array(f, np.int32)


def abc(i):
    g = np.load(os.path.join(GOLDEN, 'mesh_sdf.npz'))
    return g['verts_%d' % i], g['faces_%d' % i]


# the two lattice meshes live on the voxel centres of this grid, where the centres are exact dyadic numbers
LATTICE_RES = 16


def box(lo=(3, 3, 2), hi=(12, 12, 13)):
    """Axis-aligned box from voxel centre lo to voxel centre hi (index triples of the res-16 grid), outward faces.  Its
    top and bottom faces lie on centre planes, its side faces (parallel to z) on centre lines, and the diagonals of the
    top and bottom squares pass through centres."""
    c = inside_oracle.centres(LATTICE_RES)
    x = (c[lo[0]], c[hi[0]])
    y = (c[lo[1]], c[hi[1]])
    z = (c[lo[2]], c[hi[2]])
    v = np.array([(x[i], y[j], z[k]) for i in (0, 1) for j in (0, 1) for k in (0, 1)], np.float32)   # index 4i + 2j + k
    f = [(0, 1, 3), (0, 3, 2), (4, 6, 7), (4, 7, 5), (0, 4, 5), (0, 5, 1), (2, 3, 7), (2, 7, 6), (0, 2, 6), (0, 6, 4),
         (1, 5, 7), (1, 7, 3)]
    return v, np.array(f, np.int32)


def box_inside(lo=(3, 3, 2), hi=(12, 12, 13)):
    """What geometry and the tie rule say: the half-open index box [lo, hi) (a centre on the lower x or y face is moved
    into the box by (eps, eps^2), one on the upper face out of it; a voxel centre on the top face is below no crossing
    of it, one on the bottom face below the bottom crossing too)."""
    R = LATTICE_RES
    out = np.zeros((R, R, R), np.uint8)
    out[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = 1
    return out


def octahedron(centre=7, half=4, height=0.3):
    """Octahedron around voxel centre (centre, centre) of the res-16 grid: equator corners `half` columns away along x
    and y (so all four projected equator edges run through centres, and the four edges to each apex along a row or a
    column of centres), apexes `height` above and below the centre plane c(centre)."""
    c = inside_oracle.centres(LATTICE_RES)
    m = c[centre]
    zc = np.float32(m)
    v = np.array([(c[centre + half], m, zc), (c[centre - half], m, zc), (m, c[centre + half], zc),
                  (m, c[centre - half], zc), (m, m, np.float32(zc + height)), (m, m, np.float32(zc - height))], np.float32)
    f = [(0, 2, 4), (2, 1, 4), (1, 3, 4), (3, 0, 4), (2, 0, 5), (1, 2, 5), (3, 1, 5), (0, 3, 5)]
    return v, np.array(f, np.int32)


def octahedron_inside(centre=7, half=4, height=0.3):
    """Inside iff |x - m| + |y - m| < a (L1 radius r in columns, exact on the lattice) and |z - zc| < height (1 - r / half);
    the heights never meet a voxel centre, and columns on the boundary (r = half) have zero height."""
    R = LATTICE_RES
    c = inside_oracle.centres(R).astype(np.float64)
    i = np.arange(R)
    r = np.abs(i[:, None] - centre) + np.abs(i[None, :] - centre)
    h = np.where(r < half, height * (1.0 - r / half), -1.0)
    dz = np.abs(c - c[centre])
    return (dz[None, None, :] < h[:, :, None]).astype(np.uint8)


def closed_cases():
    """name -> (verts, faces) of every closed test mesh"""
    out = {'sphere': icosphere(), 'torus': torus(), 'box': box(), 'octahedron': octahedron()}
    for i in range(3):
        out['abc%d' % i] = abc(i)
    return out
