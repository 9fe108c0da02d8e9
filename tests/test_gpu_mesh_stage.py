"""The mesh stage (csrc/volume.cu, csrc/mc.cu) bit for bit at the resolutions the benchmark (256^3) and the sharded job
(512^3) run, on every kernel path.

Sign propagation: the kernel against oracle/sign_torch.py (a full recomputation per iteration, on the GPU): torch.equal on
the volumes and equal iteration counts.  Cases on the row-vector path (sigma 5, res % 32 == 0) also run in a subprocess
with P2S_VOL_NOVEC=1 (read once per process), which puts them on the packed-word path.  One res-128 case closes the chain
kernel = restatement = NumPy oracle.
Marching cubes: the kernel against the vectorised oracle/mc_oracle.py: identical vertex and face arrays, closed meshes,
and a counting call that returns the counts of the emitting call."""
import ctypes as C
import functools
import hashlib
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

from oracle import p2s_oracle as orc
from oracle import mc_oracle as mc
from oracle import sign_torch as st
from points2surf_b200 import ops, synth

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN, INF = float('nan'), float('inf')


# ------------------------------------------------------------------ inputs
@functools.lru_cache(maxsize=None)
def _cloud(kind):
    if kind == 'shells':        # two nested spheres, radii 0.3 and 0.6
        s = synth.make_cloud('sphere', 10000, seed=0)
        return np.concatenate([s * np.float32(0.6), s * np.float32(1.2)])
    return synth.make_cloud(kind, 10000, seed=0)


@functools.lru_cache(maxsize=None)
def _query(kind, res):
    return ops.query_grid(torch.from_numpy(_cloud(kind)).to(DEV), res, 3)


def _distance(kind, q):
    """analytic signed distance, positive inside"""
    r = q.norm(dim=1)
    if kind == 'sphere':
        return 0.5 - r
    if kind == 'torus':
        return 0.18 - torch.sqrt((q[:, :2].norm(dim=1) - 0.45) ** 2 + q[:, 2] ** 2)
    if kind == 'box':
        return 0.45 - q.abs().amax(dim=1)
    if kind == 'shells':
        return torch.minimum(0.6 - r, r - 0.3)
    raise ValueError(kind)


def _from_volume(vol):
    """scatter every nonzero voxel of a dense volume"""
    flat = vol.reshape(-1)
    lin = torch.nonzero(flat).reshape(-1)
    return lin.to(torch.int32), flat[lin].contiguous()


def _volume_case(kind, res, seed):
    g = torch.Generator(device='cpu').manual_seed(seed)
    if kind == 'plate':         # one known plane near a face: the front crosses the whole volume
        vol = torch.zeros((res,) * 3, device=DEV)
        vol[1] = 0.5
    elif kind == 'random30':    # +-1 at 30 % density: every tile is on the work list in the first iterations
        u = torch.rand((res,) * 3, generator=g).to(DEV)
        vol = torch.where(u < 0.15, 1.0, torch.where(u < 0.3, -1.0, 0.0))
    elif kind == 'stall':
        # a plate and a known +-1 checkerboard block, whose votes are 0: the stop rule counts them, so propagation stops
        # with unknowns left once fewer unknowns remain than the block holds.  The block is about a fifth of what the front
        # decides per iteration, so that happens near the far face and not in the first iterations.
        vol = torch.zeros((res,) * 3, device=DEV)
        vol[1] = 0.5
        k = int(round((0.4 * res * res) ** (1.0 / 3.0)))
        i = torch.arange(k, device=DEV)
        cb = ((i[:, None, None] + i[None, :, None] + i[None, None, :]) % 2) * 2.0 - 1.0
        vol[res - k - 4:res - 4, 4:4 + k, 4:4 + k] = cb
    elif kind == 'small':       # random signed values at 40 % density
        u = torch.rand((res,) * 3, generator=g)
        vol = torch.where(u < 0.4, torch.randn((res,) * 3, generator=g), torch.zeros(())).to(DEV)
        vol[res // 2, res // 2, res // 2] = 0.25      # at least one known voxel
    else:
        raise ValueError(kind)
    return _from_volume(vol)


def case_name(kind, res, sigma, thr, noise=0.0):
    return '%s_%d_s%d_t%s%s' % (kind, res, sigma, thr, '_n%g' % noise if noise else '')


def _parse(name):
    parts = name.split('_')
    kind, res, sigma, thr = parts[0], int(parts[1]), int(parts[2][1:]), float(parts[3][1:])
    noise = float(parts[4][1:]) if len(parts) > 4 else 0.0
    return kind, res, sigma, thr, noise


def build_case(name):
    """-> (lin int32, dist float32 on the GPU, res, sigma, thr)"""
    kind, res, sigma, thr, noise = _parse(name)
    if kind in ('plate', 'random30', 'stall', 'small'):
        lin, dist = _volume_case(kind, res, 1000 * res + sigma)
    else:
        lin = _query(kind, res)
        dist = _distance(kind, ops.query_points(lin, res))
        if noise:
            g = torch.Generator(device='cpu').manual_seed(res)
            dist = dist + noise * torch.randn(dist.shape, generator=g).to(DEV)
        dist = dist.contiguous()
    return lin, dist, res, sigma, thr


def run_kernel(name):
    lin, dist, res, sigma, thr = build_case(name)
    return ops.sdf_to_volume(lin, dist, res, sigma, thr)


def digest(vol):
    return hashlib.blake2b(vol.cpu().numpy().tobytes(), digest_size=16).hexdigest()


_REF = {}


def reference(name):
    """the restatement's volume and iteration count; digest, iterations and unknowns left are cached per case"""
    lin, dist, res, sigma, thr = build_case(name)
    vol, it = st.sdf_to_volume(lin, dist, res, sigma, thr)
    _REF[name] = (digest(vol), it, int((vol == 0).sum()))
    return vol, it


def reference_digest(name):
    if name not in _REF:
        reference(name)
    return _REF[name]


# ------------------------------------------------------------------ cases
ROW_CASES = []      # sigma 5, res % 32 == 0: the row-vector path
for _res in (256, 512):
    ROW_CASES += [case_name(k, _res, 5, 13.0) for k in ('sphere', 'torus', 'box', 'shells', 'plate', 'stall')]
    ROW_CASES += [case_name('sphere', _res, 5, 13.0, n) for n in (0.005, 0.02)]
    ROW_CASES += [case_name('random30', _res, 5, 1.0)]
ROW_CASES += [case_name('sphere', 256, 5, t) for t in (-1.0, 0.0, 0.5, 20.0, 124.5, 125.0, 125.5, 126.0, INF, NAN)]
ROW_CASES += [case_name('sphere', 512, 5, t) for t in (-1.0, 0.0, 0.5, 20.0, 126.0, NAN)]
OFF_ROW_CASES = [case_name('sphere', r, 5, 13.0) for r in (252, 300, 255, 257)]          # packed-word / byte paths
OFF_ROW_CASES += [case_name('sphere', 256, s, 13.0) for s in (3, 7, 11)]
SMALL_CASES = [case_name('small', r, s, t) for r in (2, 3, 4, 5, 7, 8) for s in (5, 7, 11) for t in (1.0, 13.0)]


def _check(name):
    vol, it = run_kernel(name)
    ref, it_ref = reference(name)
    assert it == it_ref, (name, it, it_ref)
    assert torch.equal(vol, ref), (name, int((vol != ref).sum()))
    return it


@pytest.mark.parametrize('name', ROW_CASES)
def test_row_vector_path_matches_restatement(name):
    it = _check(name)
    kind, res, _, thr, noise = _parse(name)
    _, _, left = _REF[name]
    print('%s: %d iterations, %d voxels left at 0' % (name, it, left))
    if kind == 'plate':
        assert it >= res // 2 - 2                        # the front travels through the whole volume
    if kind == 'stall':
        assert it > 10 and left > 0                      # stopped by the second rule with unknowns left
    if kind == 'sphere' and thr == 13.0 and not noise:
        assert it >= 40


_NOVEC_WORKER = r"""
import json, sys
sys.path.insert(0, %(root)r)
sys.path.insert(0, %(tests)r)
import test_gpu_mesh_stage as m
out = {}
for name in sys.argv[2:]:
    vol, it = m.run_kernel(name)
    out[name] = [m.digest(vol), it]
json.dump(out, open(sys.argv[1], 'w'))
"""


@pytest.fixture(scope='module')
def novec_results(tmp_path_factory):
    path = str(tmp_path_factory.mktemp('novec') / 'novec.json')
    env = dict(os.environ, P2S_VOL_NOVEC='1')
    r = subprocess.run([sys.executable, '-c', _NOVEC_WORKER % dict(root=ROOT, tests=os.path.join(ROOT, 'tests')), path]
                       + ROW_CASES, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    with open(path) as f:
        return json.load(f)


@pytest.mark.parametrize('name', ROW_CASES)
def test_packed_word_path_on_row_vector_cases_matches_restatement(novec_results, name):
    d, it, _ = reference_digest(name)
    assert novec_results[name] == [d, it]


@pytest.mark.parametrize('name', OFF_ROW_CASES)
def test_large_volumes_off_the_row_vector_path_match_restatement(name):
    _check(name)


@pytest.mark.parametrize('name', SMALL_CASES)
def test_volumes_smaller_than_the_window_match_restatement(name):
    _check(name)


def test_workspace_reuse_across_sizes():
    # a new thread starts with an empty per-device scratch workspace, whatever ran before
    names = [case_name('sphere', 512, 5, 13.0), case_name('sphere', 24, 5, 13.0), case_name('sphere', 257, 5, 13.0),
             case_name('sphere', 512, 5, 13.0), case_name('sphere', 24, 5, 13.0)]
    got, err = [], []

    def work():
        try:
            for n in names:
                vol, it = run_kernel(n)
                got.append((digest(vol), it))
            torch.cuda.synchronize()
        except Exception as e:      # reported on the main thread
            err.append(e)
    t = threading.Thread(target=work)
    t.start()
    t.join()
    assert not err, err
    for n, g in zip(names, got):
        assert g == reference_digest(n)[:2], n
    assert got[0] == got[3] and got[1] == got[4]


def test_anchor_res128_against_numpy_oracle():
    name = case_name('sphere', 128, 5, 13.0)
    it = _check(name)
    lin, dist, res, _, _ = build_case(name)
    idx = orc.query_grid_indices(_cloud('sphere'), res, 3)
    assert np.array_equal(lin.cpu().numpy().astype(np.int64), (idx[:, 0] * res + idx[:, 1]) * res + idx[:, 2])
    vol_ref = orc.add_samples_to_volume(np.zeros((res,) * 3), orc.query_grid(_cloud('sphere'), res, 3), dist.cpu().numpy())
    vol_ref, it_ref = orc.propagate_sign(vol_ref, 5, 13.0)
    vol, _ = run_kernel(name)
    assert it == it_ref and np.array_equal(vol.cpu().numpy().astype(np.float64), np.clip(vol_ref, -1.0, 1.0))


@pytest.mark.parametrize('bad', [-1, 'V'])
def test_scatter_rejects_out_of_range_voxel_index(bad):
    # the reference raises IndexError for an index >= res and wraps a negative one; the kernel reports both as an error
    name = case_name('sphere', 64, 5, 13.0)
    lin, dist, res, sigma, thr = build_case(name)
    lin_bad = lin.clone()
    lin_bad[len(lin) // 2] = res ** 3 if bad == 'V' else bad
    with pytest.raises(ops.P2SError, match='voxel index'):
        ops.sdf_to_volume(lin_bad, dist, res, sigma, thr)
    _check(name)                                    # the next valid call is unaffected


# ------------------------------------------------------------------ marching cubes
def _grid(R):
    g = ((torch.arange(R, device=DEV, dtype=torch.float32) + 0.5) / R * 2 - 1)
    return torch.meshgrid(g, g, g, indexing='ij')


def _mc_volume(name):
    if name.startswith('prop-'):                    # a propagated volume: plateaus at +-1, exact zeros
        return run_kernel(name[5:])[0]
    kind, R = name.split('-')
    R = int(R)
    if kind in ('sphere', 'insideout'):
        X, Y, Z = _grid(R)
        v = 0.55 - torch.sqrt(X * X + Y * Y + Z * Z)
        return -v if kind == 'insideout' else v
    if kind == 'gyroid':                            # genus: a gyroid sheet cut by a ball
        X, Y, Z = _grid(R)
        f = torch.sin(9 * X) * torch.cos(9 * Y) + torch.sin(9 * Y) * torch.cos(9 * Z) + torch.sin(9 * Z) * torch.cos(9 * X)
        return torch.minimum(f, 4 * (0.8 - torch.sqrt(X * X + Y * Y + Z * Z)))
    if kind == 'noise':                             # blocks of noise: many ambiguous faces, decided both ways
        g = torch.Generator(device='cpu').manual_seed(R)
        v = torch.full((R,) * 3, -1.0)              # below every level tested
        for x, y, z in ((1, 1, 1), (100, 40, 180), (R - 49, R - 49, R - 49)):
            v[x:x + 48, y:y + 48, z:z + 48] = torch.randn((48,) * 3, generator=g)
        return v.to(DEV)
    if kind == 'ties':                              # blocks of +-0.5 checkerboards: every inner face's saddle test ties
        v = torch.full((R,) * 3, -1.0)
        i = torch.arange(6)
        cb = (((i[:, None, None] + i[None, :, None] + i[None, None, :]) % 2) * 2.0 - 1.0) * 0.5
        for x in (1, 60, 127, 200, R - 7):
            for y in (1, 100, R - 7):
                for z in (1, 33, R - 7):
                    v[x:x + 6, y:y + 6, z:z + 6] = cb
        return v.to(DEV)
    raise ValueError(name)


def _mc_counts(vol, level):
    lib = ops._lib.load()
    nv, nf = C.c_int64(), C.c_int64()
    ops.check(lib.p2s_marching_cubes_dev(ops._ptr(vol), vol.shape[0], float(level), None, 0, None, 0, C.byref(nv),
                                         C.byref(nf), ops._stream()))
    return nv.value, nf.value


MC_CASES = [('prop-' + case_name('sphere', 256, 5, 13.0), 0.0), ('prop-' + case_name('shells', 256, 5, 13.0), 0.0),
            ('prop-' + case_name('stall', 256, 5, 13.0), 0.0), ('prop-' + case_name('sphere', 256, 5, 13.0, 0.02), 0.0),
            ('noise-256', 0.0), ('noise-256', 0.3), ('noise-256', -0.7), ('ties-256', 0.0),
            ('gyroid-512', 0.0), ('insideout-512', 0.0)]


@pytest.mark.parametrize('name,level', MC_CASES)
def test_marching_cubes_matches_vectorised_oracle(name, level):
    vol = _mc_volume(name).contiguous()
    v, f = ops.marching_cubes(vol, level)
    assert _mc_counts(vol, level) == (v.shape[0], f.shape[0])
    vo, fo, flipped = mc.marching_cubes(vol.cpu().numpy(), level, return_flipped=True)
    v, f = v.cpu().numpy(), f.cpu().numpy()
    assert v.shape == vo.shape and f.shape == fo.shape, (v.shape, vo.shape, f.shape, fo.shape)
    assert np.array_equal(f, fo), int((f != fo).any(axis=1).sum())
    assert np.array_equal(v, vo), int((v != vo).any(axis=1).sum())
    assert len(f) > 1000 and mc.mesh_is_closed(f)
    # the table's triangles face the positive side, so the orientation fix flips every mesh but the inside-out one
    assert flipped != name.startswith('insideout')
    print('%s level %g: %d vertices, %d faces' % (name, level, len(v), len(f)))


def test_config5_chain_at_512():
    # sharded job: query grid -> SDF band -> sign propagation -> marching cubes for one shape at 512^3
    res, name = 512, case_name('sphere', 512, 5, 13.0)
    lin = _query('sphere', res).cpu().numpy().astype(np.int64)
    idx = orc.query_grid_indices_shifts(_cloud('sphere'), res, 3)
    assert np.array_equal(lin, (idx[:, 0] * res + idx[:, 1]) * res + idx[:, 2])
    _check(name)
    vol, _ = run_kernel(name)
    v, f = ops.marching_cubes(vol, 0.0)
    vo, fo = mc.marching_cubes(vol.cpu().numpy(), 0.0)
    assert np.array_equal(f.cpu().numpy(), fo) and np.array_equal(v.cpu().numpy(), vo)
    assert mc.mesh_is_closed(fo)
