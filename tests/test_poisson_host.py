"""CPU: the float64 screened Poisson oracle (oracle/poisson_oracle.py) against a brute-force element-by-element
assembly, the Galerkin identities its multigrid hierarchy rests on, a sphere extracted with the marching-cubes oracle,
and the reading of meshlab filter scripts."""
import itertools

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import mc_oracle
from oracle import poisson_oracle as po
from points2surf_b200 import eval_dataset
import poisson_cases as pc

_GAUSS = (0.5 - 0.5 / np.sqrt(3.0), 0.5 + 0.5 / np.sqrt(3.0))   # 2-point Gauss on [0, 1], weights 1/2


def _random_cloud(n, seed):
    rs = np.random.RandomState(seed)
    p = rs.uniform(-1, 1, (n, 3)).astype(np.float32)
    nrm = rs.normal(size=(n, 3)).astype(np.float32)
    return p, nrm


def _brute_force(pts, normals, depth, point_weight, scale):
    """L, b, S by integrating every cell with 2-point Gauss quadrature (exact for these polynomial degrees) and by
    evaluating every hat function at every point"""
    q = po.prepare(pts, normals, depth, scale)
    n, R = q['n'], q['n'] + 1
    h = 1.0 / n
    corners = [(m & 1, (m >> 1) & 1, m >> 2) for m in range(8)]

    def basis(s, m):
        return np.prod([s[a] if corners[m][a] else 1.0 - s[a] for a in range(3)])

    def grad(s, m):
        g = []
        for a in range(3):
            d = 1.0 if corners[m][a] else -1.0
            g.append(d / h * np.prod([s[b] if corners[m][b] else 1.0 - s[b] for b in range(3) if b != a]))
        return np.array(g)

    # S and V from the hat functions evaluated directly
    alpha = float(np.float32(point_weight)) * n
    S = np.zeros((R ** 3, R ** 3))
    V = np.zeros((R ** 3, 3))
    for g, un, a in zip(q['g'], q['un'], q['area']):
        nodes, w = [], []
        for k in itertools.product(*[range(max(0, int(np.floor(x)) - 1), min(n, int(np.floor(x)) + 2) + 1) for x in g]):
            b = np.prod(np.maximum(0.0, 1.0 - np.abs(g - np.array(k))))
            if b > 0:
                nodes.append((k[0] * R + k[1]) * R + k[2])
                w.append(b)
        w = np.array(w)
        S[np.ix_(nodes, nodes)] += alpha * a * np.outer(w, w)
        V[nodes] += a * np.outer(w, un) / h ** 3
    L = np.zeros((R ** 3, R ** 3))
    b = np.zeros(R ** 3)
    for c in itertools.product(range(n), repeat=3):
        ids = [((c[0] + o[0]) * R + c[1] + o[1]) * R + c[2] + o[2] for o in corners]
        for s in itertools.product(_GAUSS, repeat=3):
            wq = h ** 3 / 8.0
            G = np.array([grad(s, m) for m in range(8)])
            Bv = np.array([basis(s, m) for m in range(8)])
            L[np.ix_(ids, ids)] += wq * G @ G.T
            Vs = Bv @ V[ids]                     # V at the quadrature point
            b[ids] += wq * G @ Vs
    return L, b, S


@pytest.mark.parametrize('depth', [2, 3])
def test_kronecker_assembly_equals_element_assembly(depth):
    pts, nrm = _random_cloud(60, depth)
    sys_ = po.assemble(pts, nrm, depth, point_weight=4.0, scale=1.1)
    L, b, S = _brute_force(pts, nrm, depth, 4.0, 1.1)
    for name, got, want in (('L', sys_['L'].toarray(), L), ('S', sys_['S'].toarray(), S), ('b', sys_['b'], b)):
        assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max()), name


@pytest.mark.parametrize('depth', [2, 5])
def test_stiffness_annihilates_constants(depth):
    L = po.stiffness(2 ** depth)
    assert np.abs(L @ np.ones(L.shape[0])).max() <= 1e-12 * abs(L.diagonal()).max()


def test_galerkin_identities():
    depth = 4
    n = 2 ** depth
    pts, nrm = _random_cloud(500, 7)
    fine = po.assemble(pts, nrm, depth, point_weight=4.0)
    P = po.prolongation(n // 2)
    Lc = (P.T @ fine['L'] @ P).toarray()
    assert np.abs(Lc - po.stiffness(n // 2).toarray()).max() <= 1e-12 * np.abs(Lc).max()
    # the screening term of the coarse basis at the same points, with the same alpha and area weights
    gc = fine['g'] / 2.0
    Bc = po.interpolation(gc, np.clip(np.floor(gc).astype(np.int64), 0, n // 2 - 1), n // 2)
    Sc = (float(np.float32(4.0)) * n * (Bc.T @ sp.diags(fine['area']) @ Bc)).toarray()
    got = (P.T @ fine['S'] @ P).toarray()
    assert np.abs(got - Sc).max() <= 1e-12 * np.abs(Sc).max()


def test_oracle_sphere_radial_error():
    depth = 5
    pts, nrm = pc.sphere(20000, seed=3)
    r = po.solve(pts, nrm, depth)
    assert r['residual'] < 1e-10
    R = r['n'] + 1
    chi = r['chi'].reshape(R, R, R)
    # chi grows along the outward normal: below iso inside, above it outside
    centre = np.round((pc.SPHERE_CENTER - r['origin']) / r['edge'] * r['n']).astype(int)
    assert chi[tuple(centre)] < r['iso'] < chi[0, 0, 0]
    v, f = mc_oracle.marching_cubes(r['values'].reshape(R, R, R).astype(np.float32), 0.0)
    w = po.to_world(v, R, r['origin'], r['edge'])
    h = r['edge'] / r['n']
    err = np.abs(np.linalg.norm(w - pc.SPHERE_CENTER, axis=1) - pc.SPHERE_RADIUS)
    assert err.mean() <= 0.25 * h, (err.mean() / h, err.max() / h)
    assert pc.closed_manifold(f) and pc.signed_volume(w, f) > 0


def test_prepare_drops_zero_normals_and_rejects_bad_input():
    pts, nrm = _random_cloud(100, 1)
    nrm[[3, 50]] = 0
    assert po.prepare(pts, nrm, 4)['dropped'] == 2
    nrm[7, 1] = np.nan
    with pytest.raises(ValueError):
        po.prepare(pts, nrm, 4)


_MLX = '''<!DOCTYPE FilterScript>
<FilterScript>
 <xmlfilter name="Surface Reconstruction: Screened Poisson">
  <xmlparam value="0" name="cgDepth"/>
  <xmlparam value="{depth}" name="depth"/>
  <xmlparam value="5" name="fullDepth"/>
  <xmlparam value="{iters}" name="iters"/>
  <xmlparam value="{pw}" name="pointWeight"/>
  <xmlparam value="1.5" name="samplesPerNode"/>
  <xmlparam value="{scale}" name="scale"/>
 </xmlfilter>
</FilterScript>
'''


def test_read_poisson_filter(tmp_path):
    f = tmp_path / 'poisson.mlx'
    f.write_text(_MLX.format(depth=7, iters=5, pw=2.5, scale=1.25))
    assert eval_dataset.read_poisson_filter(str(f)) == dict(depth=7, point_weight=2.5, scale=1.25, iters=5)
    f.write_text(_MLX.format(depth=8, iters=8, pw=4, scale=1.1))
    assert eval_dataset.read_poisson_filter(str(f)) == eval_dataset.POISSON_MLX_DEFAULTS
    g = tmp_path / 'normals_poisson.mlx'
    g.write_text('<!DOCTYPE FilterScript>\n<FilterScript>\n <filter name="Compute normals for point sets">\n'
                 '  <Param type="RichInt" name="K" value="10"/>\n </filter>\n'
                 ' <xmlfilter name="Screened Poisson Surface Reconstruction">\n'
                 '  <xmlparam name="depth" value="8"/>\n </xmlfilter>\n</FilterScript>\n')
    with pytest.raises(ValueError):
        eval_dataset.read_poisson_filter(str(g))
    h = tmp_path / 'clean.mlx'
    h.write_text('<FilterScript>\n <filter name="Close Holes"/>\n</FilterScript>\n')
    with pytest.raises(ValueError):
        eval_dataset.read_poisson_filter(str(h))
