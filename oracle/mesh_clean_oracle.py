"""TEST INFRASTRUCTURE ONLY -- float64 NumPy restatement of the mesh repair of csrc/meshclean.cu (p2s_mesh_clean_dev,
rules in include/p2s_b200.h).  It shares no code with the kernel: vertices are welded with np.unique, components and
face parities are found by an explicit breadth-first search, holes by walking the boundary in Python.  Every float64
product, sum and square root is evaluated in the kernel's order, and signed volumes are reduced in the kernel's fixed
order (fixed_sum), so kernel and oracle agree bit for bit."""
import collections

import numpy as np

WELD_SCALE = 1e8
KEY_LIMIT = 9e10
MIN_ALTITUDE = 1e-8
SUM_LANES = 256

REPORT_FIELDS = ('vertices_in', 'faces_in', 'vertices_out', 'faces_out', 'merged_vertices', 'unreferenced_vertices',
                 'nonfinite_faces', 'degenerate_faces', 'duplicate_faces', 'boundary_edges', 'nonmanifold_edges',
                 'holes_filled', 'faces_added', 'components', 'nonorientable_components', 'faces_reversed',
                 'watertight_before', 'winding_consistent_before', 'watertight', 'winding_consistent', 'volume')


def llround(y):
    """C llround (halves away from zero) of float64 values, exactly."""
    r = np.trunc(y)
    frac = y - r
    return (r + (frac >= 0.5) - (frac <= -0.5)).astype(np.int64)


def fixed_sum(d):
    """The kernel's order: lane t of 256 adds elements t, t + 256, ... in turn, then the lanes are halved pairwise."""
    d = np.asarray(d, np.float64)
    acc = np.zeros(SUM_LANES)
    for row in np.concatenate([d, np.zeros((-len(d)) % SUM_LANES)]).reshape(-1, SUM_LANES):
        acc = acc + row
    h = SUM_LANES // 2
    while h:
        acc[:h] = acc[:h] + acc[h:2 * h]
        h //= 2
    return float(acc[0])


def _norm(x, y, z):
    return np.sqrt((x * x + y * y) + z * z)


def low_altitude(v, tri):
    """2 area / longest edge <= 1e-8 (or a zero-length longest edge), float64, per face of tri [n,3]."""
    a, b, c = v[tri[:, 0]], v[tri[:, 1]], v[tri[:, 2]]
    u, w, e = b - a, c - a, c - b
    nx = u[:, 1] * w[:, 2] - u[:, 2] * w[:, 1]
    ny = u[:, 2] * w[:, 0] - u[:, 0] * w[:, 2]
    nz = u[:, 0] * w[:, 1] - u[:, 1] * w[:, 0]
    longest = np.maximum(np.maximum(_norm(*u.T), _norm(*e.T)), _norm(*w.T))
    with np.errstate(divide='ignore', invalid='ignore'):
        return (longest == 0.0) | (_norm(nx, ny, nz) / longest <= MIN_ALTITUDE)


def det3(v, tri):
    """v0 . (v1 x v2) per face, float64."""
    a, b, c = v[tri[:, 0]], v[tri[:, 1]], v[tri[:, 2]]
    cx = b[:, 1] * c[:, 2] - b[:, 2] * c[:, 1]
    cy = b[:, 2] * c[:, 0] - b[:, 0] * c[:, 2]
    cz = b[:, 0] * c[:, 1] - b[:, 1] * c[:, 0]
    return (a[:, 0] * cx + a[:, 1] * cy) + a[:, 2] * cz


def classify(W):
    """-> dict: the half-edge starts u, per undirected edge its half-edges (ascending), counts and the edge totals."""
    u = W.reshape(-1)
    w = W[:, [1, 2, 0]].reshape(-1)
    key = np.minimum(u, w) * (1 << 32) + np.maximum(u, w)
    order = np.argsort(key, kind='stable')
    _, start, counts = np.unique(key[order], return_index=True, return_counts=True)
    two = counts == 2
    h0, h1 = order[start[two]], order[start[two] + 1]
    return {'u': u, 'w': w, 'order': order, 'start': start, 'counts': counts, 'h0': h0, 'h1': h1,
            'boundary': int((counts == 1).sum()), 'nonmanifold': int((counts > 2).sum()),
            'inconsistent': int((u[h0] == u[h1]).sum())}


def fill_holes(W, e):
    """Fill faces [k,3] and the number of loops filled (rules 6 of include/p2s_b200.h)."""
    nb = collections.defaultdict(list)       # vertex -> [(neighbour, the face runs vertex -> neighbour)]
    for h in e['order'][e['start'][e['counts'] == 1]]:
        a, b = int(e['u'][h]), int(e['w'][h])
        nb[a].append((b, True))
        nb[b].append((a, False))

    def other(p, prev):
        if len(nb[p]) != 2:
            return -1
        x, y = nb[p][0][0], nb[p][1][0]
        return y if x == prev else x

    fills, loops = [], 0
    for v in sorted(nb):
        if len(nb[v]) != 2:
            continue
        p0, out = min(nb[v])
        p1 = other(p0, v)
        p2 = other(p1, p0) if p1 >= 0 else -1
        if p1 < 0 or p2 < 0:
            continue
        if p2 == v:
            if v < min(p0, p1):
                loops += 1
                fills.append((v, p1, p0) if out else (v, p0, p1))
            continue
        if other(p2, p1) == v and v < min(p0, p1, p2):
            loops += 1
            fills += [(v, p1, p0), (v, p2, p1)] if out else [(v, p0, p1), (v, p1, p2)]
    return np.array(fills, np.int64).reshape(-1, 3), loops


def orient(v, W, e):
    """Rule 7 on W in place -> (components, non-orientable components, faces reversed)."""
    n = len(W)
    f0, f1 = e['h0'] // 3, e['h1'] // 3
    rel = (e['u'][e['h0']] == e['u'][e['h1']]).astype(np.int64)
    adj = [[] for _ in range(n)]
    for a, b, r in zip(f0.tolist(), f1.tolist(), rel.tolist()):
        adj[a].append((b, r))
        adj[b].append((a, r))
    comp = np.full(n, -1, np.int64)
    parity = np.zeros(n, np.int64)
    roots = []
    for s in range(n):
        if comp[s] >= 0 or not adj[s]:
            continue
        roots.append(s)
        comp[s] = s
        queue = collections.deque([s])
        while queue:
            x = queue.popleft()
            for y, r in adj[x]:
                if comp[y] < 0:
                    comp[y] = s
                    parity[y] = parity[x] ^ r
                    queue.append(y)
    bad = set(comp[f0[(parity[f0] ^ parity[f1]) != rel]].tolist())
    flip = {}
    for r in roots:
        faces = np.nonzero(comp == r)[0]
        tri = W[faces].copy()
        tri[parity[faces] == 1] = tri[parity[faces] == 1][:, ::-1]
        flip[r] = fixed_sum(det3(v, tri)) < 0.0
    rev = np.array([comp[f] >= 0 and comp[f] not in bad and bool(parity[f]) != flip[comp[f]] for f in range(n)], bool)
    W[rev] = W[rev][:, ::-1]
    return len(roots), len(bad), int(rev.sum())


def mesh_clean(verts, faces):
    """-> (verts [V',3] float32, faces [F',3] int32, report dict) as p2s_mesh_clean_dev; ValueError on bad input."""
    v32 = np.asarray(verts, np.float32).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    V, F = len(v32), len(f)
    if F and (f.min() < 0 or f.max() >= V):
        raise ValueError('face index outside [0, V)')
    v = v32.astype(np.float64)
    finite = np.isfinite(v).all(1)
    if (np.abs(v[finite]) >= KEY_LIMIT).any():
        raise ValueError('finite vertex coordinate with |x| >= 9e10')
    rep = np.arange(V)
    fi = np.nonzero(finite)[0]
    nkeys = 0
    if len(fi):
        _, first, inv = np.unique(llround(v[fi] * WELD_SCALE), axis=0, return_index=True, return_inverse=True)
        rep[fi] = fi[first[inv.reshape(-1)]]
        nkeys = len(first)
    R = dict.fromkeys(REPORT_FIELDS, 0)
    R.update(vertices_in=V, faces_in=F, merged_vertices=V - nkeys - int((~finite).sum()))

    nonfinite = ~finite[f].all(1) if F else np.zeros(0, bool)
    r = rep[f]
    ok = ~nonfinite
    degenerate = np.zeros(F, bool)
    degenerate[ok] = ((r[ok, 0] == r[ok, 1]) | (r[ok, 1] == r[ok, 2]) | (r[ok, 0] == r[ok, 2]) |
                      low_altitude(v, r[ok]))
    cand = np.nonzero(ok & ~degenerate)[0]
    alive = np.zeros(F, bool)
    if len(cand):
        _, first = np.unique(np.sort(r[cand], axis=1), axis=0, return_index=True)
        alive[cand[first]] = True
    R.update(nonfinite_faces=int(nonfinite.sum()), degenerate_faces=int(degenerate.sum()),
             duplicate_faces=int(len(cand) - alive.sum()))

    W = r[alive].reshape(-1, 3)
    A = len(W)
    e = classify(W)
    if e['boundary']:
        fills, loops = fill_holes(W, e)
        if len(fills):
            W = np.concatenate([W, fills])
            e = classify(W)
        R['holes_filled'] = loops
    R.update(faces_added=len(W) - A, boundary_edges=e['boundary'], nonmanifold_edges=e['nonmanifold'],
             watertight_before=e['boundary'] == 0 and e['nonmanifold'] == 0,
             winding_consistent_before=e['inconsistent'] == 0)
    if e['inconsistent']:
        R['components'], R['nonorientable_components'], R['faces_reversed'] = orient(v, W, e)
        e = classify(W)
    R.update(watertight=e['boundary'] == 0 and e['nonmanifold'] == 0, winding_consistent=e['inconsistent'] == 0)

    used = np.unique(W)
    R.update(vertices_out=len(used), faces_out=len(W), unreferenced_vertices=V - R['merged_vertices'] - len(used),
             volume=fixed_sum(det3(v, W)) / 6.0 if len(W) else 0.0)
    return v32[used], np.searchsorted(used, W).astype(np.int32).reshape(-1, 3), R
