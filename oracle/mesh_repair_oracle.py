"""TEST INFRASTRUCTURE ONLY -- float64 NumPy / Python restatement of the mesh repair of csrc/meshrepair.cu
(p2s_mesh_repair_dev, rules in include/p2s_b200.h).  It shares no code with the kernel: edges are Python dicts, fans are
found by a breadth-first search per vertex, loops by walking the boundary, ears by sorting the candidates.  Every float64
product, sum, quotient and square root is evaluated in the kernel's order, so kernel and oracle agree bit for bit."""
import collections
import math

import numpy as np

STATS_FIELDS = ('vertices_in', 'faces_in', 'vertices_out', 'faces_out', 'faces_removed', 'vertices_split', 'holes_closed',
                'holes_left_open', 'faces_added')
MAX_LOOP = 128


def area2(v, tri):
    """|(b - a) x (c - a)|^2 per face of tri [n,3], float64."""
    a, b, c = v[tri[:, 0]], v[tri[:, 1]], v[tri[:, 2]]
    u, w = b - a, c - a
    nx = u[:, 1] * w[:, 2] - u[:, 2] * w[:, 1]
    ny = u[:, 2] * w[:, 0] - u[:, 0] * w[:, 2]
    nz = u[:, 0] * w[:, 1] - u[:, 1] * w[:, 0]
    return (nx * nx + ny * ny) + nz * nz


def edge_faces(W):
    """undirected edge (lo, hi) -> [face, ...] ascending"""
    e = collections.defaultdict(list)
    for i, t in enumerate(W.tolist()):
        for k in range(3):
            a, b = t[k], t[(k + 1) % 3]
            e[(min(a, b), max(a, b))].append(i)
    return e


def remove_nonmanifold_faces(v, f):
    """rule 1 -> keep flags [F]"""
    a2 = area2(v, f)
    keep = np.ones(len(f), bool)
    for fl in edge_faces(f).values():
        if len(fl) > 2:
            for g in sorted(fl, key=lambda g: (a2[g], -g))[:len(fl) - 2]:
                keep[g] = False
    return keep


def fans(W):
    """rule 3 -> {vertex: [fan, ...]}, each fan a sorted list of faces, fans ordered by their lowest face"""
    ef = edge_faces(W)
    around = collections.defaultdict(list)
    for i, t in enumerate(W.tolist()):
        for x in t:
            around[x].append(i)
    out = {}
    for x, fl in around.items():
        adj = collections.defaultdict(list)
        for i in fl:
            for y in W[i].tolist():
                if y != x:
                    g = ef[(min(x, y), max(x, y))]
                    if len(g) == 2:
                        j = g[0] if g[1] == i else g[1]
                        adj[i].append(j)
        seen, comps = set(), []
        for s in fl:
            if s in seen:
                continue
            comp, queue = [], [s]
            seen.add(s)
            while queue:
                i = queue.pop()
                comp.append(i)
                for j in adj[i]:
                    if j not in seen:
                        seen.add(j)
                        queue.append(j)
            comps.append(sorted(comp))
        out[x] = sorted(comps)
    return out


def split_vertices(W, V):
    """-> (renumbered faces, source vertex of every copy)"""
    heads = []
    fan_of = fans(W)
    for x, comps in fan_of.items():
        for comp in comps[1:]:
            lo = comp[0]
            heads.append((lo, W[lo].tolist().index(x), x, comp))
    heads.sort()
    Wn = W.copy()
    src = []
    for p, (lo, _, x, comp) in enumerate(heads):
        for i in comp:
            Wn[i][W[i] == x] = V + p
        src.append(x)
    return Wn, np.array(src, np.int64)


# ---- float64 geometry, scalar, in the kernel's order
def _sub(a, b):
    return (a[0] - b[0], a[1] - b[1], a[2] - b[2])


def _dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def _cross(u, w):
    return (u[1] * w[2] - u[2] * w[1], u[2] * w[0] - u[0] * w[2], u[0] * w[1] - u[1] * w[0])


def orient3(a, b, c, d):
    if a == b or a == c or a == d or b == c or b == d or c == d:
        return 0.0
    return _dot(_cross(_sub(b, a), _sub(c, a)), _sub(d, a))


def seg_cross(p, q, a, b, c):
    o1, o2 = orient3(a, b, c, p), orient3(a, b, c, q)
    if not ((o1 > 0 and o2 < 0) or (o1 < 0 and o2 > 0)):
        return False
    s = (orient3(p, q, a, b), orient3(p, q, b, c), orient3(p, q, c, a))
    return all(x > 0 for x in s) or all(x < 0 for x in s)


def tri_cross(T, S):
    return any(seg_cross(T[i], T[(i + 1) % 3], *S) for i in range(3)) or \
        any(seg_cross(S[i], S[(i + 1) % 3], *T) for i in range(3))


def orient2(a, b, q):
    return (b[0] - a[0]) * (q[1] - a[1]) - (b[1] - a[1]) * (q[0] - a[0])


def frame(P):
    """Newell normal of the loop P [(x,y,z)] and the 2D coordinates, or None for a zero normal"""
    nx = ny = nz = 0.0
    L = len(P)
    for i in range(L):
        a, b = P[i], P[(i + 1) % L]
        nx = nx + (a[1] - b[1]) * (a[2] + b[2])
        ny = ny + (a[2] - b[2]) * (a[0] + b[0])
        nz = nz + (a[0] - b[0]) * (a[1] + b[1])
    n = (nx, ny, nz)
    nl = math.sqrt(_dot(n, n))
    if nl == 0.0:
        return None
    ax, ay, az = abs(nx), abs(ny), abs(nz)
    u = (0.0, nz, -ny) if (ax <= ay and ax <= az) else ((-nz, 0.0, nx) if ay <= az else (ny, -nx, 0.0))
    ul = math.sqrt(_dot(u, u))
    u = (u[0] / ul, u[1] / ul, u[2] / ul)
    w = _cross((nx / nl, ny / nl, nz / nl), u)
    return [(_dot(p, u), _dot(p, w)) for p in P]


def ear_cut(ring, P, ring_faces, mesh_edges, psi):
    """-> fill faces [(a, b, c) vertex ids] in cutting order, or None when no convex ear is valid"""
    st = frame(P)
    if st is None:
        return None
    idx = list(range(len(ring)))
    out = []
    while len(idx) >= 3:
        m = len(idx)
        cands = []
        for j in range(m):
            a, b, c = idx[j - 1], idx[j], idx[(j + 1) % m]
            px, py = st[a][0] - st[b][0], st[a][1] - st[b][1]
            qx, qy = st[c][0] - st[b][0], st[c][1] - st[b][1]
            if not (py * qx - px * qy > 0.0):
                continue
            cs = (px * qx + py * qy) / (math.sqrt(px * px + py * py) * math.sqrt(qx * qx + qy * qy))
            cands.append((-cs, ring[b], j))
        cut = None
        for _, _, j in sorted(cands):
            a, b, c = idx[j - 1], idx[j], idx[(j + 1) % m]
            ok = not any(orient2(st[a], st[b], st[q]) >= 0 and orient2(st[b], st[c], st[q]) >= 0 and
                         orient2(st[c], st[a], st[q]) >= 0 for q in idx if q not in (a, b, c))
            if ok and m > 3:
                ok = frozenset((ring[a], ring[c])) not in mesh_edges
            if ok and psi:
                T = (P[a], P[b], P[c])
                pos = dict(zip(ring, P))
                ok = not any(tri_cross(T, S) for S in ring_faces) and \
                    not any(tri_cross(T, (pos[x], pos[y], pos[z])) for x, y, z in out)
            if ok:
                cut = j
                break
        if cut is None:
            return None
        a, b, c = idx[cut - 1], idx[cut], idx[(cut + 1) % len(idx)]
        out.append((ring[a], ring[b], ring[c]))
        del idx[cut]
    return out


def loops(Wn):
    """boundary loops: [(owner, walk [vertex ids])] by ascending owner (the loop's lowest vertex)"""
    nb = collections.defaultdict(list)    # vertex -> [(neighbour, the face runs neighbour -> vertex)]
    for (a, b), fl in edge_faces(Wn).items():
        if len(fl) == 1:
            t = Wn[fl[0]].tolist()
            k = t.index(a)
            a_to_b = t[(k + 1) % 3] == b
            nb[a].append((b, not a_to_b))
            nb[b].append((a, a_to_b))
    assert all(len(x) == 2 for x in nb.values()), 'a boundary vertex without two boundary edges'
    seen, out = set(), []
    for v in sorted(nb):
        if v in seen:
            continue
        (n0, in0), (n1, in1) = nb[v]
        cur = (n0 if in0 else n1) if in0 != in1 else min(n0, n1)
        walk, prev = [v], v
        while cur != v:
            walk.append(cur)
            x, y = nb[cur][0][0], nb[cur][1][0]
            prev, cur = cur, (y if x == prev else x)
        seen.update(walk)
        out.append((v, walk))
    return out


def mesh_repair(verts, faces, max_hole_size=30, prevent_self_intersection=True):
    """-> (verts [V',3] float32, faces [F',3] int32, stats dict) as p2s_mesh_repair_dev; ValueError on bad input."""
    v32 = np.asarray(verts, np.float32).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    V, F = len(v32), len(f)
    if F and (f.min() < 0 or f.max() >= V):
        raise ValueError('face index outside [0, V)')
    if F and ((f[:, 0] == f[:, 1]) | (f[:, 1] == f[:, 2]) | (f[:, 0] == f[:, 2])).any():
        raise ValueError('face with a repeated vertex index')
    if not 0 <= max_hole_size <= MAX_LOOP:
        raise ValueError('max_hole_size outside [0, 128]')
    v = v32.astype(np.float64)
    W = f[remove_nonmanifold_faces(v, f)] if F else f
    Wn, src = split_vertices(W, V)
    vout = np.concatenate([v32, v32[src]]) if len(src) else v32.copy()
    pos = [tuple(p) for p in vout.astype(np.float64).tolist()]
    around = collections.defaultdict(list)
    for i, t in enumerate(Wn.tolist()):
        for x in t:
            around[x].append(i)
    mesh_edges = {frozenset(e) for e in edge_faces(Wn)}
    fills, closed, left_open = [], 0, 0
    for _, ring in loops(Wn):
        if len(ring) > max_hole_size:
            left_open += 1
            continue
        ring_faces = []
        if prevent_self_intersection:
            ring_faces = [tuple(pos[x] for x in Wn[i].tolist()) for i in sorted({i for x in ring for i in around[x]})]
        out = ear_cut(ring, [pos[x] for x in ring], ring_faces, mesh_edges, prevent_self_intersection)
        if out is None:
            left_open += 1
        else:
            closed += 1
            fills += out
    fout = np.concatenate([Wn, np.array(fills, np.int64).reshape(-1, 3)]).astype(np.int32)
    stats = dict(vertices_in=V, faces_in=F, vertices_out=len(vout), faces_out=len(fout), faces_removed=F - len(W),
                 vertices_split=len(src), holes_closed=closed, holes_left_open=left_open, faces_added=len(fills))
    return vout, fout, stats
