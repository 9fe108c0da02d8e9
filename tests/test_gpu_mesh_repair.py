"""GPU tests of p2s_mesh_repair_dev (csrc/meshrepair.cu): array for array against the NumPy oracle
(oracle/mesh_repair_oracle.py) on the hand-built cases, the abc_minimal meshes and a marching-cubes torus with deleted
face sets; determinism; closed holes give a winding number of 0 or 1; far-sample distances on the repaired mesh."""
import numpy as np
import pytest
import torch

from oracle import mesh_repair_oracle as mro
from oracle import mesh_sdf_oracle as msdf
from points2surf_b200 import ops, sdf
from points2surf_b200._lib import P2SError
from helpers import load_golden
import mesh_repair_cases as mrc

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def kernel(v, f, **kw):
    vo, fo, st = ops.mesh_repair(cu(np.asarray(v, np.float32)), cu(np.asarray(f, np.int32)), **kw)
    return vo.cpu().numpy(), fo.cpu().numpy(), st


def assert_same_as_oracle(v, f, **kw):
    vk, fk, sk = kernel(v, f, **kw)
    vo, fo, so = mro.mesh_repair(v, f, **kw)
    assert sk == so, {k: (sk[k], so[k]) for k in so if sk[k] != so[k]}
    assert vk.tobytes() == vo.tobytes() and fk.tobytes() == fo.tobytes()
    return vk, fk, sk


@pytest.mark.parametrize('name', sorted(mrc.cases()))
def test_hand_cases_match_the_oracle(name):
    v, f = mrc.cases()[name]
    assert_same_as_oracle(v, f)


def test_parameters_match_the_oracle():
    v, f, _ = mrc.cube_with_holes()
    assert assert_same_as_oracle(v, f, max_hole_size=29)[2]['holes_left_open'] == 2
    assert assert_same_as_oracle(v, f, max_hole_size=0)[2]['faces_added'] == 0
    v, f = mrc.spiked_pyramid()
    assert assert_same_as_oracle(v, f, prevent_self_intersection=False)[2]['holes_closed'] == 1


def _abc(i):
    g = load_golden('mesh_sdf.npz')
    return g['verts_%d' % i].astype(np.float32), g['faces_%d' % i].astype(np.int32)


def _mc(kind, res=48):
    x = torch.linspace(-1, 1, res, device=DEV)
    X, Y, Z = torch.meshgrid(x, x, x, indexing='ij')
    if kind == 'sphere':
        vol = 0.6 - torch.sqrt(X * X + Y * Y + Z * Z)
    else:
        vol = 0.25 - torch.sqrt((torch.sqrt(X * X + Y * Y) - 0.55) ** 2 + Z * Z)
    v, f = ops.marching_cubes(vol.contiguous(), 0.0)
    v, f = v.cpu().numpy(), f.cpu().numpy()
    vo, fo, rep = ops.mesh_clean(cu(v), cu(sdf._orient_outward(v, f)))
    assert rep['watertight']
    return vo.cpu().numpy(), fo.cpu().numpy()


@pytest.mark.parametrize('mesh', ['abc0', 'abc1', 'abc2', 'torus'])
@pytest.mark.parametrize('seed', [0, 1, 2])
def test_meshes_with_deleted_faces_match_the_oracle(mesh, seed):
    v, f = _mc('torus') if mesh == 'torus' else _abc(int(mesh[-1]))
    f2 = mrc.delete_random_faces(f, seed=seed, n_sets=6, size=1 + 2 * seed)
    _, _, st = assert_same_as_oracle(v, f2)
    assert st['holes_closed'] >= 1


def test_intact_meshes_come_back_unchanged():
    for i in range(3):
        v, f = _abc(i)
        vk, fk, st = kernel(v, f)
        assert vk.tobytes() == v.tobytes() and fk.tobytes() == f.tobytes() and st['holes_left_open'] == 0


def test_bitwise_identical_across_runs():
    v, f = _mc('torus', 64)
    f2 = mrc.delete_random_faces(f, seed=5, n_sets=40, size=4)
    a = kernel(v, f2)
    for _ in range(3):
        b = kernel(v, f2)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes() and a[2] == b[2]


def test_closed_sphere_has_winding_zero_or_one():
    v, f = _mc('sphere')
    f2 = mrc.delete_random_faces(f, seed=3, n_sets=20, size=4)
    vk, fk, st = kernel(v, f2)
    assert st['holes_left_open'] == 0 and st['holes_closed'] >= 1
    q = (np.random.RandomState(0).rand(20000, 3) - 0.5) * 2.0 * np.abs(v).max() * 1.2
    _, w = ops.mesh_signed_distance(cu(vk), cu(fk), cu(q.astype(np.float32)), return_winding=True)
    w = w.cpu().numpy()
    assert (np.minimum(np.abs(w), np.abs(w - 1.0)) <= 1e-3).all()
    assert (np.abs(w - 1.0) <= 1e-3).any() and (np.abs(w) <= 1e-3).any()


@pytest.mark.parametrize('i', [0, 1, 2])
def test_far_sample_distances_on_the_repaired_mesh_match_the_oracle(i):
    v, f = _abc(i)
    vk, fk, _ = kernel(v, mrc.delete_random_faces(f, seed=i))
    q = (np.random.RandomState(i).rand(3000, 3) - 0.5).astype(np.float32)
    d = ops.mesh_signed_distance(cu(vk), cu(fk), cu(q)).cpu().numpy().astype(np.float64)
    od, _, ow = msdf.mesh_signed_distance(vk, fk, q)
    assert np.abs(np.abs(d) - np.abs(od)).max() <= 1e-6
    sure = np.abs(ow - 0.5) > 1e-3
    assert (np.sign(d[sure]) == np.sign(od[sure])).all()


def test_bad_input_raises():
    v, f = mrc.bowtie()
    with pytest.raises(P2SError):
        kernel(v, np.array([[0, 1, 99]]))
    with pytest.raises(P2SError):
        kernel(v, np.array([[0, 1, 1]]))
    with pytest.raises(P2SError):
        kernel(v, f, max_hole_size=129)
    vk, fk, st = kernel(np.zeros((0, 3)), np.zeros((0, 3)))
    assert len(vk) == 0 and len(fk) == 0 and st['faces_out'] == 0
