"""TEST INFRASTRUCTURE ONLY -- the point-to-mesh queries of include/p2s_b200.h (p2s_mesh_signed_distance_dev,
p2s_mesh_closest_point_dev) restated in float64 torch, chunked over queries x faces, so that they run on the device the
mesh is on and can check csrc/meshsdf.cu at sizes where the NumPy oracles (oracle/mesh_sdf_oracle.py,
tests/closest_point_oracle.py) take minutes.

Shares nothing with the kernel but the definition: the closest point of a triangle by its Voronoi regions (Ericson,
Real-Time Collision Detection, 5.1.5, the NumPy oracles' formulation, not the kernel's plane / edge one); zero-area faces
(float64 cross product of the edges exactly 0) are their three edges, the first nearest of ab, bc, ca; ties between faces
-> lowest face index; the generalised winding number from Van Oosterom & Strackee's solid angles, zero-area faces
contribute 0; inside (w > 0.5) and on the surface (|d| <= 1e-8) are positive.  tests/test_mesh_query_torch_host.py pins
it to the NumPy oracles."""
import math

import torch


def _dot(x, y):
    return x[..., 0] * y[..., 0] + x[..., 1] * y[..., 1] + x[..., 2] * y[..., 2]


def _seg_closest(p, a, b):
    u = b - a
    uu = _dot(u, u)
    t = torch.where(uu > 0, _dot(u, p - a) / torch.where(uu > 0, uu, torch.ones_like(uu)), torch.zeros_like(uu))
    return a + t.clamp(0.0, 1.0)[..., None] * u


def _region_closest(p, a, b, c):
    """p [P,1,3] (or [P,3] with a, b, c [P,3]), faces a, b, c [1,F,3] -> closest points by the closest-point regions"""
    ab, ac = b - a, c - a
    d1, d2 = _dot(ab, p - a), _dot(ac, p - a)
    d3, d4 = _dot(ab, p - b), _dot(ac, p - b)
    d5, d6 = _dot(ab, p - c), _dot(ac, p - c)
    va, vb, vc = d3 * d6 - d5 * d4, d5 * d2 - d1 * d6, d1 * d4 - d3 * d2
    den = va + vb + vc
    q = a + ab * (vb / den)[..., None] + ac * (vc / den)[..., None]                       # interior
    e = lambda m, x: torch.where(m[..., None], x, q)                                      # noqa: E731
    # Ericson's test order A, B, AB, C, AC, BC, interior: applied from the last to the first, the first that holds wins
    q = e((va <= 0) & (d4 - d3 >= 0) & (d5 - d6 >= 0), b + (c - b) * ((d4 - d3) / ((d4 - d3) + (d5 - d6)))[..., None])
    q = e((vb <= 0) & (d2 >= 0) & (d6 <= 0), a + ac * (d2 / (d2 - d6))[..., None])
    q = e((d6 >= 0) & (d5 <= d6), c.expand_as(q))
    q = e((vc <= 0) & (d1 >= 0) & (d3 <= 0), a + ab * (d1 / (d1 - d3))[..., None])
    q = e((d3 >= 0) & (d4 <= d3), b.expand_as(q))
    q = e((d1 <= 0) & (d2 <= 0), a.expand_as(q))
    return q


def _edges_closest(p, a, b, c):
    best, bq = None, None
    for s, t in ((a, b), (b, c), (c, a)):
        q = _seg_closest(p, s, t)
        d = _dot(p - q, p - q)
        if best is None:
            best, bq = d, q
        else:
            closer = d < best
            best = torch.where(closer, d, best)
            bq = torch.where(closer[..., None], q, bq)
    return bq


def _closest(p, a, b, c, zero):
    """closest points of p on faces a, b, c (broadcast), zero: the faces' zero-area flags (broadcast like a[..., 0])"""
    q = _region_closest(p, a, b, c)
    if bool(zero.any()):
        q = torch.where(zero[..., None], _edges_closest(p, a, b, c), q)
    return q


def _corners(verts, faces):
    v = torch.as_tensor(verts).to(torch.float64)
    f = torch.as_tensor(faces).to(device=v.device, dtype=torch.int64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    n = torch.cross(b - a, c - a, dim=1)
    return a, b, c, (n == 0).all(dim=1)


def closest_on_faces(verts, faces, query, face_idx):
    """closest point [Q,3] float64 of every query on the face face_idx[q]"""
    a, b, c, zero = _corners(verts, faces)
    p = torch.as_tensor(query).to(device=a.device, dtype=torch.float64)
    j = torch.as_tensor(face_idx).to(device=a.device, dtype=torch.int64)
    return _closest(p, a[j], b[j], c[j], zero[j])


def face_dist2(verts, faces, query, face_idx):
    """squared distance [Q] float64 of every query to the face face_idx[q]"""
    q = closest_on_faces(verts, faces, query, face_idx)
    p = torch.as_tensor(query).to(device=q.device, dtype=torch.float64)
    return _dot(p - q, p - q)


def mesh_query(verts, faces, query, pairs=1 << 22):
    """-> dict of float64 / int64 tensors on the mesh's device: d (unsigned distance [Q]), face [Q] (lowest index on
    ties), w (winding number [Q]), signed [Q] (the kernel's sign rule), closest [Q,3] (the point on `face`)."""
    a, b, c, zero = _corners(verts, faces)
    p_all = torch.as_tensor(query).to(device=a.device, dtype=torch.float64)
    Q, F = p_all.shape[0], a.shape[0]
    fs = max(1, min(F, pairs))
    qs = max(1, pairs // fs)
    best = torch.full((Q,), math.inf, dtype=torch.float64, device=a.device)
    face = torch.full((Q,), -1, dtype=torch.int64, device=a.device)
    wind = torch.zeros((Q,), dtype=torch.float64, device=a.device)
    for q0 in range(0, Q, qs):
        p = p_all[q0:q0 + qs, None, :]
        for f0 in range(0, F, fs):
            fa, fb, fc, fz = (x[None, f0:f0 + fs] for x in (a, b, c, zero))
            cp = _closest(p, fa, fb, fc, fz)
            d2 = _dot(p - cp, p - cp)
            m, j = d2.min(dim=1)                     # first minimum: lowest face index of the block on ties
            upd = m < best[q0:q0 + qs]                # strict: earlier blocks (lower faces) win ties
            best[q0:q0 + qs] = torch.where(upd, m, best[q0:q0 + qs])
            face[q0:q0 + qs] = torch.where(upd, j + f0, face[q0:q0 + qs])
            A, B, C = fa - p, fb - p, fc - p
            la, lb, lc = (torch.sqrt(_dot(X, X)) for X in (A, B, C))
            det = _dot(A, torch.cross(B.expand_as(C), C, dim=-1))
            den = la * lb * lc + _dot(A, B) * lc + _dot(B, C) * la + _dot(C, A) * lb
            wind[q0:q0 + qs] += torch.where(fz, torch.zeros_like(det), torch.atan2(det, den)).sum(dim=1)
    wind /= 2.0 * math.pi
    d = torch.sqrt(best)
    closest = _closest(p_all, a[face], b[face], c[face], zero[face])
    signed = torch.where((wind > 0.5) | (d <= 1e-8), d, -d)
    return dict(d=d, face=face, w=wind, signed=signed, closest=closest)
