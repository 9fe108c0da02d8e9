"""CPU: the matrix-free float64 torch restatement of the screened Poisson system (oracle/poisson_torch.py) against the
SciPy assembly and solve of oracle/poisson_oracle.py, at every point_weight and scale it is used with on the GPU,
including the singular unscreened system, and its DCT preconditioner against the operator it inverts."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla
import torch

from oracle import poisson_oracle as po
from oracle import poisson_torch as pt
import poisson_cases as pc

PARAMS = [(pw, scale) for pw in (0.0, 0.5, 2.0, 4.0, 16.0) for scale in (1.0, 1.1, 2.0)]


def _cloud(kind, n=1500):
    if kind == 'sphere':
        return pc.sphere(n, seed=11)
    if kind == 'torus':
        return pc.torus(n, seed=12)
    pts, nrm = pc.sphere(n, seed=13)       # every 7th normal zero: those points are dropped
    nrm = nrm.copy()
    nrm[::7] = 0
    return pts, nrm


def _grid(s, x):
    return torch.from_numpy(np.ascontiguousarray(x)).view(s.R, s.R, s.R)


def _rel(got, want):
    return float(np.abs(np.asarray(got).reshape(-1) - want).max() / np.abs(want).max())


@pytest.mark.parametrize('kind', ['sphere', 'torus', 'dropped'])
@pytest.mark.parametrize('depth', [2, 3, 4, 5])
def test_operator_rhs_and_diagonal_equal_scipy_assembly(depth, kind):
    pts, nrm = _cloud(kind)
    x = np.random.RandomState(depth).normal(size=(2 ** depth + 1) ** 3)
    for pw, scale in PARAMS:
        q = po.assemble(pts, nrm, depth, pw, scale)
        A = (q['L'] + q['S']).tocsr()
        s = pt.System(pts, nrm, depth, pw, scale)
        assert s.points_used == len(q['g']) and s.dropped == q['dropped']
        for name, got, want in (('(L + S) x', s.apply(_grid(s, x)), A @ x), ('b', s.b, q['b']),
                                ('diag', s.diagonal(), A.diagonal()), ('L x', s.stiffness(_grid(s, x)), q['L'] @ x)):
            assert _rel(got, want) <= 1e-13, (name, pw, scale, _rel(got, want))


@pytest.mark.parametrize('kind', ['sphere', 'torus', 'dropped'])
@pytest.mark.parametrize('depth', [2, 3, 4, 5])
def test_solution_equals_spsolve(depth, kind):
    pts, nrm = _cloud(kind)
    combos = [(0.5, 1.1), (4.0, 1.0), (4.0, 1.1), (16.0, 2.0)]
    if depth == 5:       # one spsolve takes ~25 s here: one combination per cloud
        combos = [combos[['dropped', 'sphere', 'torus'].index(kind) + 1]]
    for pw, scale in combos:
        ref = po.solve(pts, nrm, depth, pw, scale)          # spsolve at these depths
        got = pt.solve(pts, nrm, depth, pw, scale)
        rng = np.ptp(ref['chi'])
        err = float(np.abs(got['chi'].reshape(-1).numpy() - ref['chi']).max()) / rng
        assert got['residual'] <= 1e-11 and err <= 1e-10, (pw, scale, err, got['residual'])
        assert abs(got['iso'] - ref['iso']) <= 1e-10 * rng
        assert got['origin'] == tuple(ref['origin']) and got['edge'] == ref['edge']
        assert got['occupied_cells'] == ref['occupied_cells'] and got['dropped_points'] == ref['dropped']
        assert got['grid_res'] == 2 ** depth + 1 and got['points_used'] == len(pts) - ref['dropped']


@pytest.mark.parametrize('kind', ['sphere', 'torus', 'dropped'])
@pytest.mark.parametrize('depth', [2, 3, 4])
def test_unscreened_system(depth, kind):
    """point_weight 0: L 1 = 0 and 1^T b = 0 (the Neumann system is singular but consistent); the solution has a residual
    <= 1e-11 and equals, up to a constant, spsolve of the system with node 0 pinned to 0"""
    pts, nrm = _cloud(kind)
    for scale in (1.0, 1.1, 2.0):
        q = po.assemble(pts, nrm, depth, 0.0, scale)
        s = pt.System(pts, nrm, depth, 0.0, scale)
        one = torch.ones(s.R, s.R, s.R, dtype=torch.float64)
        assert float(s.apply(one).abs().max()) <= 1e-13 * float(s.diagonal().max())
        assert abs(float(s.b.sum())) <= 1e-13 * float(s.b.abs().sum())
        got = pt.solve(pts, nrm, depth, 0.0, scale)
        assert got['residual'] <= 1e-11
        A = q['L'].tocsc()[1:, 1:]
        chi = np.concatenate([[0.0], spla.spsolve(A, q['b'][1:])])
        chi -= chi.mean()
        err = float(np.abs(got['chi'].reshape(-1).numpy() - chi).max()) / np.ptp(chi)
        assert err <= 1e-10, (scale, err)
        # values = iso - chi does not depend on the constant
        iso = float(q['area'] @ (q['B'] @ chi) / q['area'].sum())
        assert np.abs(got['values'].reshape(-1).numpy() - (iso - chi)).max() <= 1e-10 * np.ptp(chi)


@pytest.mark.parametrize('n', [4, 16, 32])
def test_dct_preconditioner_inverts_screened_stiffness(n):
    pts, nrm = pc.sphere(100, seed=3)
    s = pt.System(pts, nrm, int(np.log2(n)), 0.0)
    x = torch.from_numpy(np.random.RandomState(n).normal(size=(n + 1,) * 3))
    for beta in (0.5, 3.0, 1e3):
        y = s.stiffness(x) + beta * s.mass3(x)
        err = float((pt.DCTInverse(n, beta)(y) - x).abs().max() / x.abs().max())
        assert err <= 1e-12, (beta, err)
    # beta = 0 inverts L on everything but the constant
    d = pt.DCTInverse(n, 0.0)(s.stiffness(x)) - x
    assert float((d - d.mean()).abs().max() / x.abs().max()) <= 1e-12


def test_tiny_clouds():
    """2 and 9 points: a few nodes carry all the screening, most of the grid none"""
    for N in (2, 9):
        pts, nrm = pc.sphere(N, seed=5)
        ref = po.solve(pts, nrm, 3)
        got = pt.solve(pts, nrm, 3)
        assert got['residual'] <= 1e-11
        assert np.abs(got['chi'].reshape(-1).numpy() - ref['chi']).max() <= 1e-10 * np.ptp(ref['chi'])
