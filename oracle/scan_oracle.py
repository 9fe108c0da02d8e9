"""CPU restatement (float64 NumPy) of the simulated time-of-flight scan of csrc/scan.cu, without noise: the scanner model
of include/p2s_b200.h (origin, looking along +y, wide axis z, rays through the pixel centres of a uniform image-plane grid) and the
watertight ray-triangle test of Woop, Benthin & Wald (2013), nearest hit in (0, max_distance], ties -> lowest face,
zero-area faces never hit.  The rays are computed with the same operations in the same order as the kernel.

Besides t and the face, every ray gets a barycentric margin: the smallest |min barycentric coordinate| over the faces
whose plane it crosses within range.  Below ~1e-6 the ray passes within rounding of a face's edge, where a
different but equally valid evaluation order may decide hit / miss or the face differently."""
import math

import numpy as np


def scanner_rays(rotation, location, res_x=176, res_y=144, lens_angle_w=43.6, lens_angle_h=34.6):
    """-> origin [3], directions [res_y * res_x, 3] in model space, pixels in (row, col) order."""
    R = np.asarray(rotation, np.float64)
    loc = np.asarray(location, np.float64)
    tan_w = math.tan(float(np.float32(lens_angle_w)) * (math.pi / 360.0))
    tan_h = math.tan(float(np.float32(lens_angle_h)) * (math.pi / 360.0))
    pix = np.arange(res_x * res_y)
    row, col = pix // res_x, pix % res_x
    u = (2.0 * (col + 0.5) / res_x - 1.0) * tan_w
    v = (1.0 - 2.0 * (row + 0.5) / res_y) * tan_h
    n = np.sqrt(u * u + 1.0 + v * v)
    s0, s1, s2 = v / n, 1.0 / n, u / n          # the wide axis (columns, u) is z, the rows (v) run along x
    d = np.stack([R[0, i] * s0 + R[1, i] * s1 + R[2, i] * s2 for i in range(3)], 1)
    o = np.array([-(R[0, i] * loc[0] + R[1, i] * loc[1] + R[2, i] * loc[2]) for i in range(3)])
    return o, d


def _shear_frame(d):
    ar = np.arange(len(d))
    ad = np.abs(d)
    kz = np.where(ad[:, 1] > ad[:, 0], 1, 0)
    kz = np.where(ad[:, 2] > ad[ar, kz], 2, kz)
    kx = np.where(kz == 2, 0, kz + 1)
    ky = np.where(kx == 2, 0, kx + 1)
    dz = d[ar, kz]
    neg = dz < 0
    kx, ky = np.where(neg, ky, kx), np.where(neg, kx, ky)
    return kx, ky, kz, d[ar, kx] / dz, d[ar, ky] / dz, 1.0 / dz


def cast(verts, faces, origin, dirs, max_distance=10.0, chunk_pairs=2_000_000):
    """Nearest hit of every ray (origin [3] or [n,3], dirs [n,3]) -> (t [n] f64, inf on a miss; face [n] int64, -1 on a
    miss; margin [n] f64)."""
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)
    if len(f) == 0 or f.min() < 0 or f.max() >= len(v):
        raise ValueError('face index outside [0, V) or empty mesh')
    tri = v[f]                                                   # [F, 3 vertices, 3]
    zero = (np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]) == 0.0).all(-1)
    dirs = np.asarray(dirs, np.float64)
    o = np.broadcast_to(np.asarray(origin, np.float64), dirs.shape)
    n = len(dirs)
    t_out = np.full(n, np.inf)
    f_out = np.full(n, -1, np.int64)
    m_out = np.full(n, np.inf)
    tmax = float(np.float32(max_distance))
    step = max(1, chunk_pairs // len(f))
    for i in range(0, n, step):
        dd, oo = dirs[i:i + step], o[i:i + step]
        kx, ky, kz, Sx, Sy, Sz = _shear_frame(dd)
        ar = np.arange(len(dd))
        # [r, F, 3 vertices] permuted coordinates relative to the origin
        px = tri[:, :, kx].transpose(2, 0, 1) - oo[ar, kx][:, None, None]
        py = tri[:, :, ky].transpose(2, 0, 1) - oo[ar, ky][:, None, None]
        pz = tri[:, :, kz].transpose(2, 0, 1) - oo[ar, kz][:, None, None]
        X = px - Sx[:, None, None] * pz
        Y = py - Sy[:, None, None] * pz
        Ax, Bx, Cx = X[..., 0], X[..., 1], X[..., 2]
        Ay, By, Cy = Y[..., 0], Y[..., 1], Y[..., 2]
        U = Cx * By - Cy * Bx
        V = Ax * Cy - Ay * Cx
        W = Bx * Ay - By * Ax
        det = U + V + W
        sz = Sz[:, None]
        T = U * (sz * pz[..., 0]) + V * (sz * pz[..., 1]) + W * (sz * pz[..., 2])
        with np.errstate(divide='ignore', invalid='ignore'):
            t = T / det
            bmin = np.minimum(np.minimum(U, V), W) / det
            bmin = np.where(det < 0, np.maximum(np.maximum(U, V), W) / det, bmin)
        mixed = ((U < 0) | (V < 0) | (W < 0)) & ((U > 0) | (V > 0) | (W > 0))
        valid = ~zero[None] & (det != 0)
        in_range = valid & (t > 0) & (t <= tmax)
        hit = in_range & ~mixed
        th = np.where(hit, t, np.inf)
        j = np.argmin(th, axis=1)                      # first minimum: lowest face on ties
        tb = th[ar, j]
        t_out[i:i + step] = tb
        f_out[i:i + step] = np.where(np.isfinite(tb), j, -1)
        m_out[i:i + step] = np.where(in_range, np.abs(bmin), np.inf).min(axis=1)
    return t_out, f_out, m_out


def box_survivors(verts, origin, dirs, max_distance=10.0):
    """Indices of the rays that reach the padded bounding box of the vertices within max_distance (the kernel's cull)."""
    v = np.asarray(verts, np.float64)
    lo, hi = v.min(0), v.max(0)
    pad = 1e-6 * max(np.abs(lo).max(), np.abs(hi).max()) + 1e-30
    lo, hi = lo - pad, hi + pad
    with np.errstate(divide='ignore', invalid='ignore'):
        t0, t1 = (lo - origin) / dirs, (hi - origin) / dirs
    ok = ~np.isnan(t0) & ~np.isnan(t1)
    tn = np.fmin(t0, t1).max(1, initial=0.0, where=ok)
    tf = np.fmax(t0, t1).min(1, initial=float(np.float32(max_distance)), where=ok)
    return np.nonzero(tn <= tf)[0]


def range_scan(verts, faces, rotations, locations, res_x=176, res_y=144, lens_angle_w=43.6, lens_angle_h=34.6,
               max_distance=10.0):
    """Noise-free scans -> list over scans of dict(t [npix], face [npix], margin [npix], origin [3], dirs [npix, 3]).
    Rays that miss the padded bounding box of the vertices are not cast (they cannot hit)."""
    out = []
    for R, loc in zip(rotations, locations):
        o, d = scanner_rays(R, loc, res_x, res_y, lens_angle_w, lens_angle_h)
        sel = box_survivors(verts, o, d, max_distance)
        t = np.full(len(d), np.inf)
        face = np.full(len(d), -1, np.int64)
        margin = np.full(len(d), np.inf)
        if len(sel):
            t[sel], face[sel], margin[sel] = cast(verts, faces, o, d[sel], max_distance)
        out.append({'t': t, 'face': face, 'margin': margin, 'origin': o, 'dirs': d})
    return out
