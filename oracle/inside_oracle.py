"""CPU restatement (NumPy, exact int64 edge functions) of the solid voxelisation of csrc/inside.cu
(p2s_mesh_inside_grid_dev): the inside flag of every voxel centre of a res^3 grid over [-1, 1]^3 is the parity of the
faces that the ray from the centre towards +z crosses.

The rule is watertight, so a closed mesh (every edge shared by exactly two faces) crosses every column an even number of
times whatever the coordinates:
  - x and y in fixed point, X = rint(double(x) * 2^26), for the vertices and the column centres alike (|x|, |y| < 16 keeps
    every edge function below 2^63); z stays fp32.
  - a column crosses a face iff its three projected edge functions E(u -> v) = (u - p) x (v - p), evaluated on the edge's
    canonical vertex order (lower vertex index first) and negated where the face runs the other way, have one sign; the
    two faces of an edge see exactly negated values.
  - ties (E == 0: the column centre on a projected edge or vertex) take the sign at the centre moved by (eps, eps^2):
    -sign(v.y - u.y), else sign(v.x - u.x) -- a top-left rule.  Every column sees one generic point of the projection, so
    a closed surface covers it an even number of times.
  - faces with zero projected area (parallel to z, or with a repeated vertex) cross nothing.
  - crossing height z = (E_bc z_a + E_ca z_b + E_ab z_c) / (E_bc + E_ca + E_ab) in float64, left to right; the crossing
    flips the voxels with centre c(k) < z.
On a closed mesh the parity is the winding number mod 2 (overlapping closed components, winding number 2, are outside).
The kernel must equal this bit for bit."""
import numpy as np

FIX_SCALE = 2.0 ** 26
MAX_XY = 16.0


def centres(res):
    """c(i) = float32(((double)i + 0.5) / res * 2 - 1), the voxel centres of ops.query_points."""
    return ((np.arange(res, dtype=np.float64) + 0.5) / res * 2.0 - 1.0).astype(np.float32)


def _fix(x):
    return np.rint(np.asarray(x, np.float32).astype(np.float64) * FIX_SCALE).astype(np.int64)


def _edge(ux, uy, vx, vy, px, py):
    """-> (E exact int64, sign at p + (eps, eps^2))"""
    e = (ux - px) * (vy - py) - (uy - py) * (vx - px)
    dx, dy = vx - ux, vy - uy
    tie = np.where(dy != 0, -np.sign(dy), np.sign(dx))
    return e, np.where(e != 0, np.sign(e), tie)


def crossings(verts, faces, res):
    """-> (column index ix * res + iy [H] int64, crossing height z [H] float64) of every face crossing a column."""
    v = np.asarray(verts, np.float32).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    if len(f) and (f.min() < 0 or f.max() >= len(v)):
        raise ValueError('face index outside [0, V)')
    if len(v) and not (np.all(np.abs(v[:, :2]) < MAX_XY) and np.all(np.isfinite(v[:, 2]))):
        raise ValueError('vertex with |x| or |y| >= 16 or a non-finite coordinate')
    X, Y, Z = _fix(v[:, 0]), _fix(v[:, 1]), v[:, 2].astype(np.float64)
    fx, fy = X[f], Y[f]
    area = (fx[:, 1] - fx[:, 0]) * (fy[:, 2] - fy[:, 0]) - (fy[:, 1] - fy[:, 0]) * (fx[:, 2] - fx[:, 0])
    f, fx, fy = f[area != 0], fx[area != 0], fy[area != 0]
    cf = _fix(centres(res))
    # candidate columns: centres inside the face's fixed-point bounding box
    i0 = np.searchsorted(cf, fx.min(1), 'left')
    i1 = np.searchsorted(cf, fx.max(1), 'right')
    j0 = np.searchsorted(cf, fy.min(1), 'left')
    j1 = np.searchsorted(cf, fy.max(1), 'right')
    ni, nj = np.maximum(i1 - i0, 0), np.maximum(j1 - j0, 0)
    n = ni * nj
    face = np.repeat(np.arange(len(f)), n)
    t = np.arange(n.sum()) - np.repeat(np.cumsum(n) - n, n)
    i = i0[face] + t // np.maximum(nj[face], 1)
    j = j0[face] + t % np.maximum(nj[face], 1)
    px, py = cf[i], cf[j]
    ids, gx, gy = f[face], fx[face], fy[face]
    e, s = [], []
    for k in range(3):
        a, b = k, (k + 1) % 3
        fwd = ids[:, a] < ids[:, b]
        u = np.where(fwd, a, b)
        w = np.where(fwd, b, a)
        r = np.arange(len(ids))
        ek, sk = _edge(gx[r, u], gy[r, u], gx[r, w], gy[r, w], px, py)
        e.append(np.where(fwd, ek, -ek))
        s.append(np.where(fwd, sk, -sk))
    hit = (s[0] == s[1]) & (s[1] == s[2])
    z = Z[ids[hit]]
    w0, w1, w2 = e[1][hit].astype(np.float64), e[2][hit].astype(np.float64), e[0][hit].astype(np.float64)
    zh = (w0 * z[:, 0] + w1 * z[:, 1] + w2 * z[:, 2]) / (w0 + w1 + w2)
    return i[hit] * res + j[hit], zh


def inside_grid(verts, faces, res):
    """-> (inside [res, res, res] uint8 indexed [ix, iy, iz], crossings per column [res, res] int64)."""
    col, zh = crossings(verts, faces, res)
    k0 = np.searchsorted(centres(res).astype(np.float64), zh, 'left')    # voxel centres below the crossing
    cnt = np.zeros((res * res, res + 1), np.int64)
    np.add.at(cnt, (col, k0), 1)
    above = np.cumsum(cnt[:, ::-1], axis=1)[:, ::-1]                       # [:, k] = crossings with k0 >= k
    inside = (above[:, 1:] % 2).astype(np.uint8)                          # voxel k flips for every k0 > k
    return inside.reshape(res, res, res), np.bincount(col, minlength=res * res).reshape(res, res)
