"""The two references of the mesh-stage GPU tests against the plain ones they restate.

* oracle/sign_torch.py (sign propagation as a full torch recomputation, used on the GPU at 256^3 and 512^3) against
  oracle/p2s_oracle.propagate_sign on torch-CPU: identical volumes and iteration counts.
* oracle/mc_oracle.marching_cubes (vectorised, streamed over x-slabs) against the cell-by-cell `_marching_cubes_loop`:
  identical vertex and face arrays."""
import numpy as np
import pytest
import torch

from oracle import p2s_oracle as orc
from oracle import mc_oracle as mc
from oracle import mc_topo
from oracle import sign_torch as st
from helpers import load_golden

THRS = [-1.0, 0.0, 0.5, 1.0, 12.5, 13.0, 124.5, 125.0, 125.5, 126.0, 200.0, float('inf'), float('nan')]


def _centres(res):
    g = np.arange(res, dtype=np.float64)
    return np.meshgrid(g, g, g, indexing='ij')


def make_sign_volume(kind, res, rng):
    """float32 volume with unknowns (exact zeros) of one of the kinds the reconstruction and its edge cases produce."""
    X, Y, Z = _centres(res)
    if kind == 'band':           # a signed-distance band around a sphere, with noise
        c = rng.uniform(0.3, 0.7, 3) * res
        r = rng.uniform(0.2, 0.45) * res
        d = np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) - r
        d += rng.choice([0.0, 0.3, 1.0]) * rng.standard_normal(d.shape)
        vol = np.where(np.abs(d) < rng.uniform(1.0, 3.0), -d / res, 0.0)
    elif kind == 'full':         # every voxel known: no iteration
        vol = rng.standard_normal((res,) * 3)
        vol[vol == 0] = 1.0
    elif kind == 'sparse':       # random +-1 at a low or high density
        p = rng.choice([0.02, 0.1, 0.3])
        vol = np.where(rng.uniform(size=(res,) * 3) < p, rng.choice([-1.0, 1.0], (res,) * 3), 0.0)
    elif kind == 'plate':        # a known plate near one face: the front crosses the whole volume
        vol = np.zeros((res,) * 3)
        vol[min(1, res - 1)] = 1.0
    else:                        # 'checker': a known +-1 checkerboard (zero votes) beside a band: stalls with unknowns left
        vol = np.zeros((res,) * 3)
        h = max(1, res // 2)
        vol[:h] = np.where((X + Y + Z)[:h] % 2 == 0, 1.0, -1.0)
        vol[h:, :max(1, res // 3)] = 0.5
    return vol.astype(np.float32)


def _sign_cases():
    rng = np.random.RandomState(20261016)
    kinds = ['band', 'full', 'sparse', 'plate', 'checker']
    cases = []
    for i in range(70):
        res = int(rng.randint(2, 41))
        cases.append((kinds[i % len(kinds)], res, int(rng.randint(1, 12)), THRS[i % len(THRS)], int(rng.randint(1 << 30))))
    cases.append(('band', 128, 5, 13.0, 7))
    return cases


SIGN_CASES = _sign_cases()


def test_sign_cases_cover_the_edges():
    res = [c[1] for c in SIGN_CASES]
    assert len(SIGN_CASES) >= 60 and min(res) == 2 and 128 in res
    assert {c[2] for c in SIGN_CASES} == set(range(1, 12))
    assert {str(c[3]) for c in SIGN_CASES} == {str(t) for t in THRS}
    assert any(c[1] < c[2] for c in SIGN_CASES)                      # volumes smaller than the window


@pytest.fixture(scope='module')
def sign_outcomes():
    return {}


@pytest.mark.parametrize('kind,res,sigma,thr,seed', SIGN_CASES)
def test_propagate_sign_torch_matches_numpy_oracle(kind, res, sigma, thr, seed, sign_outcomes):
    vol = make_sign_volume(kind, res, np.random.RandomState(seed))
    ref, it_ref = orc.propagate_sign(vol.astype(np.float64), sigma, thr)
    got, it = st.propagate_sign_torch(torch.from_numpy(vol), sigma, thr)
    assert it == it_ref
    assert np.array_equal(got.numpy().astype(np.float64), ref)
    assert np.array_equal(st.box_sum_nearest(torch.from_numpy(np.sign(vol).astype(np.int8)), sigma).numpy(),
                          orc._box_sum_nearest(np.sign(vol).astype(np.int8), sigma))
    sign_outcomes[(kind, res, sigma, str(thr), seed)] = (it, int((ref == 0).sum()))


def test_sign_outcomes_include_no_iteration_long_runs_and_stalls(sign_outcomes):
    if len(sign_outcomes) < len(SIGN_CASES):
        pytest.skip('needs the whole parametrised test above')
    outs = list(sign_outcomes.values())
    assert any(it == 0 for it, _ in outs)
    assert any(it >= 10 for it, _ in outs)
    assert sum(1 for it, left in outs if it > 0 and left > 0) >= 3   # stopped with unknowns left


def test_sdf_to_volume_torch_matches_numpy_oracle():
    g = load_golden('volume.npz')
    for name in ('sphere', 'noisy'):
        res = int(g[name + '_res'])
        idx = orc.model_space_to_volume_space(g[name + '_qpts'], res)
        lin = torch.from_numpy((idx[:, 0] * res + idx[:, 1]) * res + idx[:, 2])
        vol, it = st.sdf_to_volume(lin, torch.from_numpy(g[name + '_dist']), res, 5, 13)
        assert np.array_equal(vol.numpy().astype(np.float64), orc.sdf_to_volume(g[name + '_dist'], g[name + '_qpts'], res, 5, 13))
        assert it == int(g[name + '_iters'])
    assert st.sdf_to_volume(lin, torch.zeros(len(lin)), res, 5, 13) == (None, -1)


# ------------------------------------------------------------------ marching cubes: vectorised vs cell-by-cell
def _mc_volumes():
    rng = np.random.RandomState(5)
    noise = rng.standard_normal((17, 17, 17)).astype(np.float32)
    noise[[0, -1]] = -1; noise[:, [0, -1]] = -1; noise[:, :, [0, -1]] = -1
    R = 24
    g = (np.arange(R) + 0.5) / R * 2 - 1
    X, Y, Z = np.meshgrid(g, g, g, indexing='ij')
    sphere = (0.6 - np.sqrt(X ** 2 + Y ** 2 + Z ** 2)).astype(np.float32)
    # values drawn from a few levels, so that exact zeros, values exactly at the level and tied saddles (A*C == B*D) abound
    ties = rng.choice(np.float32([-1.0, -0.7, -0.5, 0.0, 0.3, 0.5, 1.0]), (16, 16, 16)).astype(np.float32)
    small = rng.standard_normal((2, 2, 2)).astype(np.float32)
    return {'all_cases_0': mc_topo.all_cases_volume(0), 'all_cases_3': mc_topo.all_cases_volume(3), 'noise': noise,
            'sphere': sphere, 'inside_out': -sphere, 'propagated': np.clip(load_golden('volume.npz')['noisy_vol'], -1, 1).astype(np.float32),
            'ties': ties, 'r2': small}


MC_VOLUMES = _mc_volumes()


@pytest.mark.parametrize('name', sorted(MC_VOLUMES))
@pytest.mark.parametrize('level', [0.0, 0.3, -0.7])
def test_vectorised_marching_cubes_matches_cell_loop(name, level):
    vol = MC_VOLUMES[name]
    v0, f0 = mc._marching_cubes_loop(vol, level)
    for slab in (1 << 22, 1, 3 * vol.shape[0] ** 2):              # one slab; one plane per slab; three planes per slab
        v1, f1 = mc.marching_cubes(vol, level, slab_voxels=slab)
        assert v1.dtype == np.float32 and f1.dtype == np.int32
        assert np.array_equal(v0, v1) and np.array_equal(f0, f1), (name, level, slab)
    if name in ('sphere', 'inside_out', 'noise', 'propagated') and level == 0.0:
        assert len(f0) and mc.mesh_is_closed(f0)


def test_vectorised_marching_cubes_reports_the_flip():
    _, f, flipped = mc.marching_cubes(MC_VOLUMES['sphere'], 0.0, return_flipped=True)
    _, fi, flipped_i = mc.marching_cubes(MC_VOLUMES['inside_out'], 0.0, return_flipped=True)
    assert flipped != flipped_i and len(f) and len(fi)
    assert mc.marching_cubes(np.full((5, 5, 5), -1.0, np.float32), 0.0, return_flipped=True)[1].shape == (0, 3)
