"""Float64 closest point on a triangle mesh: the Voronoi regions of oracle/mesh_sdf_oracle.py (Ericson, Real-Time Collision
Detection, 5.1.5) extended to return the point, for the tests of p2s_mesh_closest_point_dev.  The squared distances are
the same expressions as mesh_sdf_oracle._closest_dist2, so they equal it bit for bit (tests/test_closest_point_host.py
checks that).  Zero-area faces (float64 cross product of the edges exactly 0) are their three edges, the first nearest of
ab, bc, ca.  Ties between faces -> lowest face index."""
import numpy as np

from oracle import mesh_sdf_oracle as msdf


def _seg_closest(p, a, b):
    u = b - a
    w = p - a
    uu = (u * u).sum(-1)
    with np.errstate(divide='ignore', invalid='ignore'):
        t = np.where(uu > 0, (u * w).sum(-1) / np.where(uu > 0, uu, 1.0), 0.0)
    t = np.clip(t, 0.0, 1.0)
    return a + t[..., None] * u


def _region_closest(p, a, b, c):
    """p [P,1,3], a,b,c [1,F,3] -> closest points [P,F,3] by the closest-point regions (mesh_sdf_oracle._closest_dist2)."""
    ab, ac, ap = b - a, c - a, p - a
    d1, d2 = (ab * ap).sum(-1), (ac * ap).sum(-1)
    bp = p - b
    d3, d4 = (ab * bp).sum(-1), (ac * bp).sum(-1)
    cp = p - c
    d5, d6 = (ab * cp).sum(-1), (ac * cp).sum(-1)
    va, vb, vc = d3 * d6 - d5 * d4, d5 * d2 - d1 * d6, d1 * d4 - d3 * d2
    with np.errstate(divide='ignore', invalid='ignore'):
        den = va + vb + vc
        v, w = vb / den, vc / den
        q = a + ab * v[..., None] + ac * w[..., None]
        t_ab = d1 / (d1 - d3)
        t_ac = d2 / (d2 - d6)
        t_bc = (d4 - d3) / ((d4 - d3) + (d5 - d6))
    q = np.where(((va <= 0) & (d4 - d3 >= 0) & (d5 - d6 >= 0))[..., None], b + (c - b) * t_bc[..., None], q)
    q = np.where(((vb <= 0) & (d2 >= 0) & (d6 <= 0))[..., None], a + ac * t_ac[..., None], q)
    q = np.where(((d6 >= 0) & (d5 <= d6))[..., None], c, q)
    q = np.where(((vc <= 0) & (d1 >= 0) & (d3 <= 0))[..., None], a + ab * t_ab[..., None], q)
    q = np.where(((d3 >= 0) & (d4 <= d3))[..., None], b, q)
    q = np.where(((d1 <= 0) & (d2 <= 0))[..., None], a, q)
    return q


def _edges_closest(p, a, b, c):
    best = None
    for s, e in ((a, b), (b, c), (c, a)):
        q = np.broadcast_to(_seg_closest(p, s, e), np.broadcast_shapes(p.shape, a.shape))
        d = ((p - q) ** 2).sum(-1)
        if best is None:
            best, bq = d, q.copy()
        else:
            closer = d < best
            best = np.where(closer, d, best)
            bq = np.where(closer[..., None], q, bq)
    return bq


def closest_points_on_faces(verts, faces, query, face_idx):
    """The closest point [Q,3] of every query on the face face_idx[q] (float64)."""
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)[np.asarray(face_idx, np.int64)]
    p = np.asarray(query, np.float64)[:, None, :]
    a, b, c = v[f[:, 0]][:, None], v[f[:, 1]][:, None], v[f[:, 2]][:, None]
    zero = msdf._edges_zero_area(a, b, c)[:, 0]
    q = _region_closest(p, a, b, c)[:, 0]
    if zero.any():
        q[zero] = _edges_closest(p[zero], a[zero], b[zero], c[zero])[:, 0]
    return q


def mesh_closest_point(verts, faces, query, chunk_pairs=2_000_000):
    """-> (closest [Q,3] f64, distance [Q] f64, face [Q] int64, squared distances of every face [Q,F] f64)."""
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)
    q = np.asarray(query, np.float64)
    if len(f) == 0 or f.min() < 0 or f.max() >= len(v):
        raise ValueError('face index outside [0, V) or empty mesh')
    a, b, c = v[f[:, 0]][None], v[f[:, 1]][None], v[f[:, 2]][None]
    zero = msdf._edges_zero_area(a, b, c)[0]
    d2 = np.empty((len(q), len(f)))
    step = max(1, chunk_pairs // len(f))
    for i in range(0, len(q), step):
        p = q[i:i + step, None, :]
        cp = _region_closest(p, a, b, c)
        if zero.any():
            cp[:, zero] = _edges_closest(p, a[:, zero], b[:, zero], c[:, zero])
        d2[i:i + step] = ((p - cp) ** 2).sum(-1)
    face = np.argmin(d2, axis=1)                    # first minimum: lowest face index on ties
    return closest_points_on_faces(v, f, q, face), np.sqrt(d2[np.arange(len(q)), face]), face, d2
