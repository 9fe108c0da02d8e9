"""Oriented point clouds with analytic normals for the screened Poisson tests and tools/poisson_bench.py."""
import numpy as np

SPHERE_CENTER = np.array([0.1, -0.2, 0.3])
SPHERE_RADIUS = 0.8
TORUS_CENTER = np.array([-0.05, 0.1, 0.0])
TORUS_R, TORUS_r = 0.6, 0.25


def sphere(n, seed=0):
    """-> (pts [n,3] float32, outward unit normals [n,3] float32), uniform on the sphere"""
    d = np.random.RandomState(seed).normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return (SPHERE_CENTER + SPHERE_RADIUS * d).astype(np.float32), d.astype(np.float32)


def torus(n, seed=0):
    """-> (pts, outward unit normals) of the torus around z, area-uniform (rejection on the tube angle)"""
    rs = np.random.RandomState(seed)
    u, v = np.empty(0), np.empty(0)
    while len(u) < n:
        uu, vv = rs.uniform(0, 2 * np.pi, 2 * n), rs.uniform(0, 2 * np.pi, 2 * n)
        keep = rs.uniform(0, 1, 2 * n) < (TORUS_R + TORUS_r * np.cos(vv)) / (TORUS_R + TORUS_r)
        u, v = np.concatenate([u, uu[keep]]), np.concatenate([v, vv[keep]])
    u, v = u[:n], v[:n]
    nrm = np.stack([np.cos(v) * np.cos(u), np.cos(v) * np.sin(u), np.sin(v)], 1)
    ring = TORUS_R * np.stack([np.cos(u), np.sin(u), np.zeros_like(u)], 1)
    return (TORUS_CENTER + ring + TORUS_r * nrm).astype(np.float32), nrm.astype(np.float32)


def torus_distance(p):
    """unsigned distance of points [n,3] to the analytic torus"""
    q = np.asarray(p, np.float64) - TORUS_CENTER
    return np.abs(np.hypot(np.hypot(q[:, 0], q[:, 1]) - TORUS_R, q[:, 2]) - TORUS_r)


def closed_manifold(faces):
    """every undirected edge is used by exactly two faces"""
    f = np.asarray(faces, np.int64)
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), axis=1)
    _, cnt = np.unique(e, axis=0, return_counts=True)
    return bool((cnt == 2).all())


def euler_characteristic(verts, faces):
    f = np.asarray(faces, np.int64)
    e = np.unique(np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), axis=1), axis=0)
    return len(np.unique(f)) - len(e) + len(f)


def signed_volume(verts, faces):
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)
    return float(np.einsum('ij,ij->i', v[f[:, 0]], np.cross(v[f[:, 1]], v[f[:, 2]])).sum() / 6.0)
