"""TEST INFRASTRUCTURE ONLY -- float64 SciPy restatement of the screened Poisson system that
points2surf_b200/csrc/poisson.cu solves (the formulation is stated in include/p2s_b200.h, p2s_poisson_solve_dev).

The system is assembled from the 1D hat-function matrices with Kronecker products and a sparse trilinear
interpolation matrix (N x nodes, 8 entries per row), and solved directly (spsolve) at depth <= 5 or by conjugate
gradients to a 1e-12 relative residual above.  It shares no code with the kernel: the kernel applies the same operator
matrix-free through per-cell screening matrices and multigrid.

Node (i, j, k) has the linear index (i R + j) R + k, R = 2^depth + 1 (np.kron's order, and the kernel's)."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla


def matrices_1d(n):
    """-> (M, K, D) [n+1, n+1] CSR: int phi_i phi_j, int phi_i' phi_j', int phi_i phi_j' on nodes 0..n, h = 1/n."""
    h = 1.0 / n
    R = n + 1
    ends = np.zeros(R, bool)
    ends[[0, n]] = True
    off = np.ones(n)
    M = sp.diags([np.where(ends, h / 3.0, 2.0 * h / 3.0), off * (h / 6.0), off * (h / 6.0)], [0, 1, -1])
    K = sp.diags([np.where(ends, 1.0 / h, 2.0 / h), off * (-1.0 / h), off * (-1.0 / h)], [0, 1, -1])
    dd = np.zeros(R)
    dd[0], dd[n] = -0.5, 0.5
    D = sp.diags([dd, off * 0.5, off * -0.5], [0, 1, -1])
    return M.tocsr(), K.tocsr(), D.tocsr()


def kron3(a, b, c):
    return sp.kron(a, sp.kron(b, c, format='csr'), format='csr')


def stiffness(n):
    M, K, _ = matrices_1d(n)
    return (kron3(K, M, M) + kron3(M, K, M) + kron3(M, M, K)).tocsr()


def prolongation(nc):
    """P [(2nc+1)^3, (nc+1)^3]: coarse hat functions in terms of the fine ones (1D: 1/2, 1, 1/2)."""
    nf = 2 * nc
    rows, cols, vals = [], [], []
    for I in range(nc + 1):
        for a, w in ((-1, 0.5), (0, 1.0), (1, 0.5)):
            i = 2 * I + a
            if 0 <= i <= nf:
                rows.append(i)
                cols.append(I)
                vals.append(w)
    p1 = sp.csr_matrix((vals, (rows, cols)), shape=(nf + 1, nc + 1))
    return kron3(p1, p1, p1)


def frame(pts, scale):
    """-> (origin [3] float64, edge): the cube of edge scale * largest extent centred on the bounding box."""
    pts = np.asarray(pts, np.float32)
    lo = pts.min(0).astype(np.float64)
    hi = pts.max(0).astype(np.float64)
    edge = float(np.float32(scale)) * float((hi - lo).max())
    return 0.5 * (lo + hi) - 0.5 * edge, edge


def prepare(pts, normals, depth, scale=1.1):
    """Points with nonzero normals in grid coordinates g = (p - origin) / edge * 2^depth, their unit normals, finest
    cells and area weights (4h)^2 / (points in the depth-2 cell)."""
    pts = np.asarray(pts, np.float32)
    nrm = np.asarray(normals, np.float32)
    if len(pts) == 0 or not (np.isfinite(pts).all() and np.isfinite(nrm).all()):
        raise ValueError('empty or non-finite input')
    n = 2 ** depth
    origin, edge = frame(pts, scale)
    if edge <= 0:
        raise ValueError('zero extent')
    keep = ~(nrm == 0).all(1)
    g = (pts[keep].astype(np.float64) - origin) / edge * n
    nk = nrm[keep].astype(np.float64)
    un = nk / np.sqrt((nk * nk).sum(1))[:, None]
    cell = np.clip(np.floor(g).astype(np.int64), 0, n - 1)
    dc = cell // 4
    dkey = (dc[:, 0] * n + dc[:, 1]) * n + dc[:, 2]
    _, inv, cnt = np.unique(dkey, return_inverse=True, return_counts=True)
    area = (4.0 / n) ** 2 / cnt[inv.reshape(-1)]
    return dict(n=n, origin=origin, edge=edge, g=g, un=un, cell=cell, area=area, dropped=int((~keep).sum()))


def interpolation(g, cell, n):
    """B [N, (n+1)^3]: the 8 trilinear weights of every point in its cell."""
    R = n + 1
    t = g - cell
    rows, cols, vals = [], [], []
    N = len(g)
    for m in range(8):
        o = np.array([m & 1, (m >> 1) & 1, m >> 2])
        w = np.prod(np.where(o[None, :] == 1, t, 1.0 - t), axis=1)
        c = cell + o[None, :]
        rows.append(np.arange(N))
        cols.append((c[:, 0] * R + c[:, 1]) * R + c[:, 2])
        vals.append(w)
    return sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(N, R ** 3))


def assemble(pts, normals, depth, point_weight=4.0, scale=1.1):
    """-> dict(L, S, b, B (interpolation), area, ...) of the system (L + S) chi = b."""
    q = prepare(pts, normals, depth, scale)
    n = q['n']
    M, K, D = matrices_1d(n)
    L = (kron3(K, M, M) + kron3(M, K, M) + kron3(M, M, K)).tocsr()
    B = interpolation(q['g'], q['cell'], n)
    alpha = float(np.float32(point_weight)) * n
    S = (alpha * (B.T @ sp.diags(q['area']) @ B)).tocsr()
    V = (B.T @ (q['area'][:, None] * q['un'])) * float(n) ** 3
    b = kron3(D, M, M).T @ V[:, 0] + kron3(M, D, M).T @ V[:, 1] + kron3(M, M, D).T @ V[:, 2]
    q.update(L=L, S=S, b=b, B=B, V=V)
    return q


def solve(pts, normals, depth, point_weight=4.0, scale=1.1):
    """-> dict(chi [(n+1)^3], values = iso - chi, iso, residual, origin, edge, dropped, occupied_cells)."""
    q = assemble(pts, normals, depth, point_weight, scale)
    A = (q['L'] + q['S']).tocsr()
    b = q['b']
    if depth <= 5:
        chi = spla.spsolve(A.tocsc(), b)
    else:
        dinv = sp.diags(1.0 / A.diagonal())
        chi, info = spla.cg(A, b, rtol=1e-12, atol=0.0, maxiter=20000, M=dinv)
        if info != 0:
            raise RuntimeError('CG did not converge (%d)' % info)
    a = q['area']
    iso = float(a @ (q['B'] @ chi) / a.sum())
    n = q['n']
    cells = np.unique((q['cell'][:, 0] * n + q['cell'][:, 1]) * n + q['cell'][:, 2])
    return dict(chi=chi, values=iso - chi, iso=iso, residual=float(np.linalg.norm(b - A @ chi) / np.linalg.norm(b)),
                origin=q['origin'], edge=q['edge'], dropped=q['dropped'], occupied_cells=len(cells), n=n)


def to_world(verts_mc, R, origin, edge):
    """Marching-cubes vertices ((i + 0.5) / R - 0.5) * 2 of an R^3 node grid -> world: origin + edge i / (R - 1)."""
    i = (np.asarray(verts_mc, np.float64) / 2.0 + 0.5) * R - 0.5
    return np.asarray(origin)[None, :] + edge * i / (R - 1)
