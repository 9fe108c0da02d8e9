"""CPU oracle of the oriented point normals (include/p2s_b200.h, "point normals"), written from the rules stated there:
cKDTree neighbours, float64 eigh plane fit with the same degeneracy and pre-sign rules, edge costs with the same operation
order, Kruskal with union-find under the total order (cost bits, min id, max id), rooting and signs by BFS.  Tests only."""
import collections

import numpy as np
from scipy.spatial import cKDTree


def dist2(p, q):
    """(dx*dx + dy*dy) + dz*dz in float64 on the fp32 coordinates (no FMA: NumPy rounds every operation)."""
    d = p.astype(np.float64) - q.astype(np.float64)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def neighbours(pts, k):
    """ids [N,k] int32: the k nearest points of every point, itself included, ascending (distance, id)."""
    pts = np.ascontiguousarray(pts, np.float32)
    n = len(pts)
    extra = min(n, k + 16)                    # room to resolve ties at the k-th distance by id
    _, cand = cKDTree(pts.astype(np.float64)).query(pts.astype(np.float64), k=extra)
    d = dist2(pts[cand], pts[:, None, :])
    order = np.lexsort((cand, d), axis=1)
    ids = np.take_along_axis(cand, order, 1)
    ds = np.take_along_axis(d, order, 1)
    if extra < n and (ds[:, k - 1] == ds[:, -1]).any():
        raise ValueError('more than 16 points tie at a k-th neighbour distance')
    return ids[:, :k].astype(np.int32)


def plane_fit(pts, ids):
    """-> (normals [N,3] fp32 with the pre-sign rule, zero where degenerate; gap ratio (l1 - l0) / l2 [N], 0 where l2 = 0)."""
    p = np.ascontiguousarray(pts, np.float32).astype(np.float64)[ids]          # [N,k,3]
    d = p - p.mean(axis=1, keepdims=True)
    w, v = np.linalg.eigh(np.einsum('nki,nkj->nij', d, d))
    l0, l1, l2 = w[:, 0], w[:, 1], w[:, 2]
    ok = (l2 > 0) & (l1 - l0 > 1e-9 * l2)
    n = v[:, :, 0]
    n = (n / np.linalg.norm(n, axis=1, keepdims=True)).astype(np.float32)
    n = presign(n)
    n[~ok] = 0
    gap = np.where(l2 > 0, (l1 - l0) / np.where(l2 > 0, l2, 1.0), 0.0)
    return n, gap


def presign(n):
    """The component of largest magnitude (lowest axis on ties) becomes positive."""
    n = np.array(n, np.float32)
    big = n[np.arange(len(n)), np.argmax(np.abs(n), axis=1)]
    n[big < 0] *= -1
    return n


def dot(a, b):
    a, b = a.astype(np.float64), b.astype(np.float64)
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def edges(normals, ids):
    """The graph's edges sorted by the total order -> (lo [E], hi [E], cost [E] float64), each undirected edge once."""
    n, k = ids.shape
    i = np.repeat(np.arange(n, dtype=np.int64), k)
    j = ids.reshape(-1).astype(np.int64)
    valid = np.any(normals != 0, axis=1)
    keep = (i != j) & valid[i] & valid[j]
    lo, hi = np.minimum(i, j)[keep], np.maximum(i, j)[keep]
    pair = np.unique(lo * n + hi)
    lo, hi = pair // n, pair % n
    cost = np.maximum(1.0 - np.abs(dot(normals[lo], normals[hi])), 0.0) + 0.0
    order = np.lexsort((hi, lo, cost.view(np.uint64)))
    return lo[order], hi[order], cost[order]


def spanning_forest(n, lo, hi):
    """Kruskal over edges already in the total order -> boolean mask of the forest's edges."""
    parent = list(range(n))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    take = np.zeros(len(lo), bool)
    for e, (a, b) in enumerate(zip(lo.tolist(), hi.tolist())):
        ra, rb = find(a), find(b)
        if ra != rb:
            parent[ra] = rb
            take[e] = True
    return take


def orient(pts, normals, ids):
    """-> (oriented normals [N,3] fp32, forest parents [N] int32 (root: itself, no normal: -1), stats dict)."""
    pts = np.ascontiguousarray(pts, np.float32)
    normals = np.ascontiguousarray(normals, np.float32)
    n = len(pts)
    lo, hi, _ = edges(normals, ids)
    take = spanning_forest(n, lo, hi)
    adj = collections.defaultdict(list)
    for a, b in zip(lo[take].tolist(), hi[take].tolist()):
        adj[a].append(b)
        adj[b].append(a)
    valid = np.any(normals != 0, axis=1)
    parents = np.full(n, -1, np.int32)
    out = normals.copy()
    # roots in (largest z, lowest id) order: the first unreached point of that order is its component's root
    z = pts[:, 2] + np.float32(0)
    components = 0
    for r in np.lexsort((np.arange(n), -z.astype(np.float64))).tolist():
        if not valid[r] or parents[r] >= 0:
            continue
        components += 1
        parents[r] = r
        lead = next((c for c in (out[r, 2], out[r, 1], out[r, 0]) if c != 0), 0.0)
        if lead < 0:
            out[r] = -out[r]
        queue = collections.deque([r])
        while queue:
            a = queue.popleft()
            for b in adj[a]:
                if parents[b] >= 0:
                    continue
                parents[b] = a
                if dot(out[a], normals[b]) < 0:
                    out[b] = -normals[b]
                queue.append(b)
    flipped = int((np.any(out != normals, axis=1)).sum())
    return out, parents, dict(components=components, degenerate=int((~valid).sum()), flipped=flipped)


def point_normals(pts, k=10, mode='propagate', viewpoint=None):
    """-> (normals [N,3] fp32, ids [N,k] int32)."""
    pts = np.ascontiguousarray(pts, np.float32)
    ids = neighbours(pts, k)
    n, _ = plane_fit(pts, ids)
    if mode == 'viewpoint':
        v = np.asarray(viewpoint, np.float64)[None, :] - pts.astype(np.float64)
        nd = n.astype(np.float64)
        d = (nd[:, 0] * v[:, 0] + nd[:, 1] * v[:, 1]) + nd[:, 2] * v[:, 2]
        n = n.copy()
        n[d < 0] *= -1
        return n, ids
    return orient(pts, n, ids)[0], ids
