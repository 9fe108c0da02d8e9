"""TEST INFRASTRUCTURE ONLY -- the screened Poisson system of include/p2s_b200.h (p2s_poisson_solve_dev) restated in
float64 torch, matrix-free, so that it runs on the device the inputs are on and can check points2surf_b200/csrc/poisson.cu
at depths 7-9, where oracle/poisson_oracle.py's sparse assembly and solve take minutes to hours.

The point side (grid coordinates, cells, area weights, unit normals, dropped points) is poisson_oracle.prepare.  The rest
shares nothing with the kernel but the formulation:
  L x     K(x)M(x)M + M(x)K(x)M + M(x)M(x)K as 1D tridiagonal products along the axes of an [R, R, R] tensor
  S x     alpha B^T (a * B x) by a gather and an index_add_, alpha = float32(point_weight) 2^depth
  b       D^T(x)M(x)M V_x + M(x)D^T(x)M V_y + M(x)M(x)D^T V_z with V = n^3 B^T (a * un)
  solve   conjugate gradients preconditioned by the exact inverse of L (DCT-I diagonalises the 1D M and K), plus the
          exact correction of the constant mode, which L does not see and S does; until the recomputed residual
          ||b - A chi|| / ||b|| <= tol.  point_weight 0 is the singular Neumann system: the constant is projected out of b
          and of every iterate, and chi is returned with mean zero (values = iso - chi does not depend on it).
Node (i, j, k) is entry [i, j, k], linear index (i R + j) R + k, R = 2^depth + 1 (the kernel's and poisson_oracle's)."""
import math
import time

import numpy as np
import torch

from oracle import poisson_oracle as po


def _tri(x, ax, d0, dm, dn, lo, up):
    """y_i = d_i x_i + lo x_{i-1} + up x_{i+1} along axis `ax` (nodes 0..n), d_0 = d0, d_n = dn, dm in between"""
    n = x.shape[ax] - 1
    y = x * dm
    y.narrow(ax, 0, 1).copy_(x.narrow(ax, 0, 1) * d0)
    y.narrow(ax, n, 1).copy_(x.narrow(ax, n, 1) * dn)
    y.narrow(ax, 1, n).add_(x.narrow(ax, 0, n), alpha=lo)
    y.narrow(ax, 0, n).add_(x.narrow(ax, 1, n), alpha=up)
    return y


class System:
    """(L + S) chi = b of one cloud on `device`.  pts, normals: [N, 3] float32 arrays (NumPy or torch)."""

    def __init__(self, pts, normals, depth, point_weight=4.0, scale=1.1, device='cpu'):
        pts = pts.cpu().numpy() if torch.is_tensor(pts) else np.asarray(pts)
        normals = normals.cpu().numpy() if torch.is_tensor(normals) else np.asarray(normals)
        q = po.prepare(pts, normals, depth, scale)
        n = q['n']
        h = 1.0 / n
        self.n, self.R, self.h, self.dev = n, n + 1, h, torch.device(device)
        self.origin, self.edge, self.dropped = q['origin'], q['edge'], q['dropped']
        self.points_used = len(q['g'])
        self.occupied_cells = len(np.unique((q['cell'][:, 0] * n + q['cell'][:, 1]) * n + q['cell'][:, 2]))
        self.M = (h / 3.0, 2.0 * h / 3.0, h / 3.0, h / 6.0, h / 6.0)       # (d_0, d_mid, d_n, lower, upper)
        self.K = (1.0 / h, 2.0 / h, 1.0 / h, -1.0 / h, -1.0 / h)
        self.DT = (-0.5, 0.0, 0.5, 0.5, -0.5)                               # D^T, D(i, i +- 1) = +-1/2
        self.alpha = float(np.float32(point_weight)) * n
        # the 8 trilinear nodes and weights of every point (corner m = (m & 1, m >> 1 & 1, m >> 2))
        g = torch.from_numpy(q['g']).to(self.dev)
        cell = torch.from_numpy(q['cell']).to(self.dev)
        t = g - cell
        o = torch.tensor([[m & 1, (m >> 1) & 1, m >> 2] for m in range(8)], device=self.dev)
        c = cell[:, None, :] + o[None]                                       # [N, 8, 3]
        self.idx = (c[..., 0] * self.R + c[..., 1]) * self.R + c[..., 2]
        self.w = torch.where(o[None] == 1, t[:, None, :], 1.0 - t[:, None, :]).prod(2)
        self.a = torch.from_numpy(q['area']).to(self.dev)
        un = torch.from_numpy(q['un']).to(self.dev)
        V = [self._bt(self.a * un[:, k]) * float(n) ** 3 for k in range(3)]
        self.b = _tri(_tri(_tri(V[0], 0, *self.DT), 1, *self.M), 2, *self.M)
        self.b += _tri(_tri(_tri(V[1], 0, *self.M), 1, *self.DT), 2, *self.M)
        self.b += _tri(_tri(_tri(V[2], 0, *self.M), 1, *self.M), 2, *self.DT)
        del V
        # 1^T A 1 = 1^T S 1 (L 1 = 0, the hat functions sum to 1)
        self.const_energy = self.alpha * float(self.a.sum())

    # ---- operators on [R, R, R] float64 tensors
    def _b(self, x):
        """B x: chi at every point"""
        return (x.reshape(-1)[self.idx] * self.w).sum(1)

    def _bt(self, y):
        """B^T y as an [R, R, R] tensor"""
        out = torch.zeros(self.R ** 3, dtype=torch.float64, device=self.dev)
        out.index_add_(0, self.idx.reshape(-1), (self.w * y[:, None]).reshape(-1))
        return out.view(self.R, self.R, self.R)

    def stiffness(self, x):
        mz = _tri(x, 2, *self.M)
        out = _tri(_tri(mz, 1, *self.M), 0, *self.K)
        t = _tri(mz, 1, *self.K)
        del mz
        t += _tri(_tri(x, 2, *self.K), 1, *self.M)
        out += _tri(t, 0, *self.M)
        return out

    def screening(self, x):
        return self._bt(self.alpha * self.a * self._b(x))

    def apply(self, x):
        """(L + S) x"""
        out = self.stiffness(x)
        out += self.screening(x)
        return out

    def mass3(self, x):
        """M(x)M(x)M x"""
        return _tri(_tri(_tri(x, 0, *self.M), 1, *self.M), 2, *self.M)

    def diagonal(self):
        """diag(L + S)"""
        dM = torch.full((self.R,), self.M[1], dtype=torch.float64, device=self.dev)
        dK = torch.full((self.R,), self.K[1], dtype=torch.float64, device=self.dev)
        dM[0] = dM[-1] = self.M[0]
        dK[0] = dK[-1] = self.K[0]
        d = (dK[:, None, None] * dM[None, :, None] * dM[None, None, :] + dM[:, None, None] * dK[None, :, None]
             * dM[None, None, :] + dM[:, None, None] * dM[None, :, None] * dK[None, None, :]).reshape(-1)
        d.index_add_(0, self.idx.reshape(-1), (self.alpha * self.a[:, None] * self.w * self.w).reshape(-1))
        return d.view(self.R, self.R, self.R)

    def interpolate(self, x):
        """sum a chi(p) / sum a"""
        return float((self.a * self._b(x)).sum() / self.a.sum())


class DCTInverse:
    """(L + beta M(x)M(x)M)^-1 on the (n+1)^3 grid, beta >= 0.  With C_ik = cos(pi i k / n) and W = diag(1/2, 1, .., 1, 1/2),
    K C = W C diag(lk) and M C = W C diag(lm), lk = (2 - 2 cos t_k) / h, lm = h (2 + cos t_k) / 3, t_k = pi k / n; and
    C W C = (n / 2) W^-1.  So the inverse is (2/n)^3 C3 diag(W3 / Lambda) C3 with C3 = C(x)C(x)C applied axis by axis (a
    dense [R, R] product: exact to rounding, and R <= 513).  beta = 0 drops the k = 0 mode (Lambda = 0 there): the result
    then inverts L on everything but the constant."""

    def __init__(self, n, beta=0.0, device='cpu'):
        R, h = n + 1, 1.0 / n
        k = torch.arange(R, dtype=torch.float64, device=device)
        self.C = torch.cos(math.pi * torch.outer(k, k) / n)
        ct = torch.cos(math.pi * k / n)
        lk, lm = (2.0 - 2.0 * ct) / h, h * (2.0 + ct) / 3.0
        w = torch.ones(R, dtype=torch.float64, device=device)
        w[0] = w[-1] = 0.5
        lam = (lk[:, None, None] * lm[None, :, None] * lm[None, None, :] + lm[:, None, None] * lk[None, :, None]
               * lm[None, None, :] + lm[:, None, None] * lm[None, :, None] * lk[None, None, :]
               + beta * lm[:, None, None] * lm[None, :, None] * lm[None, None, :])
        ww = w[:, None, None] * w[None, :, None] * w[None, None, :]
        self.scale = torch.where(lam > 0, (2.0 / n) ** 3 * ww / torch.where(lam > 0, lam, 1.0), 0.0)
        self.R = R

    def _c3(self, x):
        R = self.R
        x = x @ self.C                                        # axis 2 (C is symmetric)
        x = torch.matmul(self.C, x)                           # axis 1
        return (self.C @ x.reshape(R, R * R)).view(R, R, R)   # axis 0

    def __call__(self, x):
        y = self._c3(x)
        y *= self.scale
        return self._c3(y)


def solve(pts, normals, depth, point_weight=4.0, scale=1.1, device='cpu', tol=1e-11, max_iters=5000):
    """-> dict(chi, values = iso - chi, iso, residual, iterations, seconds, and the report fields of ops.poisson_solve:
    origin, edge, grid_res, occupied_cells, points_used, dropped_points).  chi and values are [R, R, R] float64 on
    `device`.  Raises RuntimeError when CG does not reach `tol` in `max_iters` iterations."""
    dev = torch.device(device)
    sync = torch.cuda.synchronize if dev.type == 'cuda' else (lambda: None)
    sync()
    t0 = time.perf_counter()
    A = System(pts, normals, depth, point_weight, scale, dev)
    P0 = DCTInverse(A.n, 0.0, dev)
    singular = A.const_energy == 0.0

    def project(x):
        if singular:
            x -= x.mean()
        return x

    def precondition(r):
        z = P0(r)
        if singular:
            return project(z)
        z += float(r.sum()) / A.const_energy
        return z

    b = project(A.b.clone())
    bn = float(torch.linalg.vector_norm(b))
    x = torch.zeros_like(b)
    it, rel = 0, 0.0
    if bn > 0:
        r = b.clone()
        z = precondition(r)
        p = z.clone()
        rz = float(torch.vdot(r.reshape(-1), z.reshape(-1)))
        while True:
            q = A.apply(p)
            step = rz / float(torch.vdot(p.reshape(-1), q.reshape(-1)))
            x.add_(p, alpha=step)
            r.add_(q, alpha=-step)
            del q
            it += 1
            if float(torch.linalg.vector_norm(r)) <= tol * bn:
                # the recursive residual drifts from the true one: stop on the recomputed residual, else continue from it
                r = project(b - A.apply(x))
                rel = float(torch.linalg.vector_norm(r)) / bn
                if rel <= tol:
                    break
            if it >= max_iters:
                raise RuntimeError('reference CG: residual %.3g after %d iterations' % (rel, it))
            z = precondition(r)
            rz_new = float(torch.vdot(r.reshape(-1), z.reshape(-1)))
            p.mul_(rz_new / rz).add_(z)
            rz = rz_new
            del z
        del r, p
    if singular:
        x -= x.mean()
    iso = A.interpolate(x)
    sync()
    return dict(chi=x, values=iso - x, iso=iso, residual=rel, iterations=it, seconds=time.perf_counter() - t0,
                origin=tuple(float(v) for v in A.origin), edge=A.edge, grid_res=A.R, occupied_cells=A.occupied_cells,
                points_used=A.points_used, dropped_points=A.dropped, n=A.n)
