"""GPU: the screened Poisson kernel (ops.poisson_solve) against the float64 torch reference (oracle/poisson_torch.py) on
the device, at the depths and parameters production runs with (depth 8 for eval_dataset --spsr, depth 7 with
point_weight 2 for --spsr_estimated_normals) and at the edges of what the ABI accepts: depths 2-4 and 9, point_weight 0
and 16, scale 1.0 and 2.0, iters 1 and 64, uneven area weights, a flat cloud, dropped points and tiny clouds.

Every case holds the kernel to: max |d values| <= 1e-4 range(chi); the sign of values wherever the reference's |values|
exceeds that; every zero crossing of the reference on a grid edge (where it changes by >= 1e-3 range(chi)) moved by
<= 0.01 h; |d iso| <= 1e-4 range(chi); the
report's frame and counts equal to the reference's; and a converged solve (residual <= 1e-5 in < 100 iterations)."""
import time

import numpy as np
import pytest
import torch

from oracle import poisson_oracle as po
from oracle import poisson_torch as pt
from points2surf_b200 import ops
import poisson_cases as pc
from test_gpu_poisson import _abc_samples, cu

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
TOL = 1e-4          # of range(chi), for values and iso
CROSS_TOL = 0.01    # of h, for the zero crossings
# ... on the edges where the reference changes by >= 1e-3 range(chi).  On flatter edges float64 itself does not place the
# crossing to 0.01 h: the flat disc's chi equals iso on its whole plane by symmetry, so rounding alone sets the signs there
CROSS_MIN_STEP = 1e-3


def _dropped_sphere(n):
    pts, nrm = pc.sphere(n, seed=1)
    nrm = nrm.copy()
    nrm[::7] = 0
    return pts, nrm


def _uneven(depth, n=20000):
    """a sparse sphere (10 % of the points) and a dense disc tangent to it (90 %) inside one depth-(d-2) cell"""
    pts, nrm = pc.sphere(n // 10, seed=21)
    origin, edge = po.frame(pts, 1.1)
    c = 2 ** (depth - 2)
    d = np.array([0.48, 0.6, 0.64])
    d /= np.linalg.norm(d)
    cell = np.floor((pc.SPHERE_CENTER + pc.SPHERE_RADIUS * d - origin) / edge * c)
    centre = origin + (cell + 0.5) * edge / c
    e1 = np.cross(d, [0.0, 0.0, 1.0])
    e1 /= np.linalg.norm(e1)
    e2 = np.cross(d, e1)
    rs = np.random.RandomState(22)
    m = n - len(pts)
    r, phi = 0.3 * edge / c * np.sqrt(rs.uniform(0, 1, m)), rs.uniform(0, 2 * np.pi, m)
    disc = centre + (r * np.cos(phi))[:, None] * e1 + (r * np.sin(phi))[:, None] * e2
    return (np.concatenate([pts, disc.astype(np.float32)]),
            np.concatenate([nrm, np.repeat(d[None].astype(np.float32), m, 0)]))


def _flat(n=20000):
    """a planar disc: zero extent in z"""
    rs = np.random.RandomState(23)
    r, phi = 0.7 * np.sqrt(rs.uniform(0, 1, n)), rs.uniform(0, 2 * np.pi, n)
    pts = np.stack([r * np.cos(phi), r * np.sin(phi), np.full(n, 0.1)], 1).astype(np.float32)
    return pts, np.repeat(np.array([[0.0, 0.0, 1.0]], np.float32), n, 0)


def _estimated_normals(n):
    pts, _ = _abc_samples(n)
    return pts, ops.point_normals(cu(pts), k=10).cpu().numpy()


def _cloud(kind, depth):
    return {
        'abc': lambda: _abc_samples(50000),
        'abc_est': lambda: _estimated_normals(50000),
        'sphere': lambda: pc.sphere(20000, seed=1),
        'torus': lambda: pc.torus(20000, seed=2),
        'sphere200k': lambda: pc.sphere(200000, seed=1),
        'torus200k': lambda: pc.torus(200000, seed=2),
        'sphere1M': lambda: pc.sphere(1000000, seed=1),
        'uneven': lambda: _uneven(depth),
        'flat': _flat,
        'dropped': lambda: _dropped_sphere(200000),
        'tiny2': lambda: pc.sphere(2, seed=5),
        'tiny9': lambda: pc.sphere(9, seed=5),
    }[kind]()


# (cloud, depth, point_weight, scale, iters, run twice for bitwise identity)
CASES = [
    ('abc', 8, 4.0, 1.1, 8, False),          # eval_dataset --spsr
    ('sphere200k', 8, 4.0, 1.1, 8, True),
    ('torus200k', 8, 4.0, 1.1, 8, False),
    ('abc_est', 7, 2.0, 1.1, 8, False),      # eval_dataset --spsr_estimated_normals
    ('sphere', 2, 4.0, 1.1, 8, False),       # the coarse level alone
    ('torus', 2, 4.0, 1.1, 8, False),
    ('sphere', 3, 4.0, 1.1, 8, False),
    ('torus', 3, 4.0, 1.1, 8, False),
    ('sphere', 4, 4.0, 1.1, 8, False),
    ('torus', 4, 4.0, 1.1, 8, False),
    ('sphere1M', 9, 4.0, 1.1, 8, True),      # the largest grid
    ('sphere', 6, 0.0, 1.1, 8, False),       # unscreened: singular Neumann system
    ('abc', 6, 0.0, 1.1, 8, False),
    ('sphere200k', 8, 0.0, 1.1, 8, False),
    ('abc', 8, 0.0, 1.1, 8, False),
    ('torus', 7, 16.0, 1.1, 8, False),       # strong screening
    ('sphere', 6, 4.0, 1.0, 8, False),       # extreme points on the cube's faces
    ('sphere200k', 8, 4.0, 1.0, 8, False),
    ('torus', 7, 4.0, 2.0, 8, False),        # loose frame
    ('abc', 8, 4.0, 1.1, 1, False),          # smoother extremes
    ('abc', 8, 4.0, 1.1, 64, False),
    ('uneven', 7, 4.0, 1.1, 8, False),
    ('flat', 7, 4.0, 1.1, 8, False),
    ('dropped', 8, 4.0, 1.1, 8, False),
    ('tiny2', 3, 4.0, 1.1, 8, False),
    ('tiny9', 3, 4.0, 1.1, 8, False),
]


def _timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def _worst(err):
    """-> (max, (i, j, k)) of an [R, R, R] tensor"""
    k = int(err.reshape(-1).argmax())
    R = err.shape[0]
    return float(err.reshape(-1)[k]), (k // (R * R), (k // R) % R, k % R)


def _crossings(kv, rv, min_step):
    """-> (largest shift of a zero crossing on a grid edge, in h, its (axis, i, j, k), number of crossings): every edge
    where the reference changes sign strictly and by at least min_step, crossing at t = v0 / (v0 - v1) of the edge"""
    worst, where, count = 0.0, None, 0
    n = rv.shape[0] - 1
    for ax in range(3):
        r0, r1 = rv.narrow(ax, 0, n), rv.narrow(ax, 1, n)
        m = ((r0 * r1) < 0) & ((r0 - r1).abs() >= min_step)
        count += int(m.sum())
        if not bool(m.any()):
            continue
        k0, k1 = kv.narrow(ax, 0, n)[m], kv.narrow(ax, 1, n)[m]
        shift = (k0 / (k0 - k1) - r0[m] / (r0[m] - r1[m])).abs()
        shift = torch.where(torch.isfinite(shift), shift, torch.full_like(shift, float('inf')))
        j = int(shift.argmax())
        if float(shift[j]) > worst or where is None:
            worst = float(shift[j])
            ijk = m.nonzero()[j].tolist()
            where = (ax,) + tuple(ijk)
    return worst, where, count


@pytest.mark.parametrize('kind,depth,pw,scale,iters,twice', CASES,
                         ids=['%s-d%d-pw%g-s%g-it%d' % c[:5] for c in CASES])
def test_kernel_against_float64_reference(kind, depth, pw, scale, iters, twice):
    pts, nrm = _cloud(kind, depth)
    if kind == 'uneven':
        q = po.prepare(pts, nrm, depth)
        assert np.unique(q['cell'] // 4, axis=0, return_counts=True)[1].max() >= 0.9 * len(pts)
    (vals, rep), tk = _timed(lambda: ops.poisson_solve(cu(pts), cu(nrm), depth, pw, scale, iters))
    if twice:
        v2, r2 = ops.poisson_solve(cu(pts), cu(nrm), depth, pw, scale, iters)
        assert torch.equal(vals, v2)
        assert {k: v for k, v in rep.items() if k != 'stage_ms'} == {k: v for k, v in r2.items() if k != 'stage_ms'}
        del v2
    ref = pt.solve(pts, nrm, depth, pw, scale, device=DEV)
    rv, kv = ref['values'], vals.double()
    rng = float(ref['chi'].max() - ref['chi'].min())
    bound = TOL * rng
    dv = (kv - rv).abs()
    ev, at = _worst(dv)
    flips = int(((rv.abs() > bound) & (torch.sign(kv) != torch.sign(rv))).sum())
    cross, cross_at, ncross = _crossings(kv, rv, CROSS_MIN_STEP * rng)
    diso = abs(rep['iso'] - ref['iso'])
    print('%s d=%d pw=%g scale=%g iters=%d: |dvalues| %.3g of bound at %s, crossing shift %.3g of bound at %s '
          '(%d crossings), |diso| %.3g of bound, %d sign flips; kernel %d it, residual %.2e, %.3f s; reference %d it, '
          'residual %.1e, %.2f s'
          % (kind, depth, pw, scale, iters, ev / bound, at, cross / CROSS_TOL, cross_at, ncross, diso / bound, flips,
             rep['iterations'], rep['residual'], tk, ref['iterations'], ref['residual'], ref['seconds']))
    assert rep['residual'] <= 1e-5 and rep['iterations'] < 100
    assert ev <= bound
    assert flips == 0
    assert ncross > 0 and cross <= CROSS_TOL
    assert diso <= bound
    assert rep['origin'] == ref['origin'] and rep['edge'] == ref['edge']
    for k in ('grid_res', 'occupied_cells', 'points_used', 'dropped_points'):
        assert rep[k] == ref[k], k
    del ref, rv, kv, dv, vals
    torch.cuda.empty_cache()
