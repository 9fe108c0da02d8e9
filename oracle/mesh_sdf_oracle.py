"""CPU restatement (float64 NumPy) of the training-target signed distance: trimesh.proximity.signed_distance as called by
sdf.get_signed_distance (source/sdf.py:318-348) -- the distance to the nearest triangle, positive inside.

Distance: exact closest point on each triangle by its Voronoi regions (Ericson, Real-Time Collision Detection, 5.1.5),
a different formulation from the kernel's (plane / edge), so that the two check each other.  Zero-area faces (float64
cross product of the edges exactly 0) are their three edges.  Ties -> lowest face index.
Sign: generalised winding number w (Jacobson et al. 2013), solid angles by Van Oosterom & Strackee (1983); zero-area
faces contribute 0.  Inside (w > 0.5) and on the surface (|d| <= 1e-8) are positive, like trimesh.
Pinned against the reference's own 05_query_dist on the abc_minimal meshes (tests/golden/mesh_sdf.npz)."""
import numpy as np


def _edges_zero_area(a, b, c):
    n = np.cross(b - a, c - a)
    return (n == 0.0).all(axis=-1)


def _seg_dist2(p, a, b):
    u = b - a
    w = p - a
    uu = (u * u).sum(-1)
    with np.errstate(divide='ignore', invalid='ignore'):
        t = np.where(uu > 0, (u * w).sum(-1) / np.where(uu > 0, uu, 1.0), 0.0)
    t = np.clip(t, 0.0, 1.0)
    d = w - t[..., None] * u
    return (d * d).sum(-1)


def _closest_dist2(p, a, b, c):
    """p [P,1,3], a,b,c [1,F,3] -> squared distances [P,F] by the closest-point regions."""
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
        q = a + ab * v[..., None] + ac * w[..., None]                                   # interior
        t_ab = d1 / (d1 - d3)
        t_ac = d2 / (d2 - d6)
        t_bc = (d4 - d3) / ((d4 - d3) + (d5 - d6))
    # Ericson's test order A, B, AB, C, AC, BC, interior: apply the regions from the last to the first so that the
    # first region that holds wins
    q = np.where(((va <= 0) & (d4 - d3 >= 0) & (d5 - d6 >= 0))[..., None], b + (c - b) * t_bc[..., None], q)
    q = np.where(((vb <= 0) & (d2 >= 0) & (d6 <= 0))[..., None], a + ac * t_ac[..., None], q)
    q = np.where(((d6 >= 0) & (d5 <= d6))[..., None], c, q)
    q = np.where(((vc <= 0) & (d1 >= 0) & (d3 <= 0))[..., None], a + ab * t_ab[..., None], q)
    q = np.where(((d3 >= 0) & (d4 <= d3))[..., None], b, q)
    q = np.where(((d1 <= 0) & (d2 <= 0))[..., None], a, q)
    return ((p - q) ** 2).sum(-1)


def _half_solid_angles(p, a, b, c):
    A, B, C = a - p, b - p, c - p
    la, lb, lc = (np.sqrt((X * X).sum(-1)) for X in (A, B, C))
    det = (A * np.cross(B, C)).sum(-1)
    den = la * lb * lc + (A * B).sum(-1) * lc + (B * C).sum(-1) * la + (C * A).sum(-1) * lb
    return np.arctan2(det, den)


def mesh_signed_distance(verts, faces, query, chunk_pairs=2_000_000):
    """-> (signed distance [Q] f64, closest face [Q] int64, winding number [Q] f64).  verts / query are taken as given
    (pass the fp32 arrays the kernel sees, widened to float64 exactly)."""
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)
    q = np.asarray(query, np.float64)
    if len(f) == 0 or f.min() < 0 or f.max() >= len(v):
        raise ValueError('face index outside [0, V) or empty mesh')
    a, b, c = v[f[:, 0]][None], v[f[:, 1]][None], v[f[:, 2]][None]
    zero = _edges_zero_area(a, b, c)[0]
    good = ~zero
    ag, bg, cg = a[:, good], b[:, good], c[:, good]
    dist = np.empty(len(q))
    face = np.empty(len(q), np.int64)
    wind = np.empty(len(q))
    step = max(1, chunk_pairs // len(f))
    for i in range(0, len(q), step):
        p = q[i:i + step, None, :]
        d2 = np.full((p.shape[0], len(f)), np.inf)
        d2[:, good] = _closest_dist2(p, ag, bg, cg)
        if zero.any():
            az, bz, cz = a[:, zero], b[:, zero], c[:, zero]
            d2[:, zero] = np.minimum(np.minimum(_seg_dist2(p, az, bz), _seg_dist2(p, bz, cz)), _seg_dist2(p, cz, az))
        j = np.argmin(d2, axis=1)                   # first minimum: lowest face index on ties
        face[i:i + step] = j
        dist[i:i + step] = np.sqrt(d2[np.arange(len(j)), j])
        wind[i:i + step] = _half_solid_angles(p, ag, bg, cg).sum(1) / (2.0 * np.pi)
    inside = (wind > 0.5) | (dist <= 1e-8)
    return np.where(inside, dist, -dist), face, wind
