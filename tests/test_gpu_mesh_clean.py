"""GPU tests of p2s_mesh_clean_dev (csrc/meshclean.cu): bit-for-bit against the float64 oracle
(oracle/mesh_clean_oracle.py) on hand-built cases and corrupted meshes, repair back to the original, determinism,
errors, and make_dataset from 00_base_meshes up to one training epoch."""
import numpy as np
import pytest
import torch

from oracle import mesh_clean_oracle as mco
from points2surf_b200 import make_dataset, mesh_io, ops, sdf
from helpers import load_golden
import mesh_clean_cases as mcc
from test_mesh_clean_host import write_obj, write_stl

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def kernel(v, f):
    vo, fo, rep = ops.mesh_clean(cu(np.asarray(v, np.float32)), cu(np.asarray(f, np.int32)))
    return vo.cpu().numpy(), fo.cpu().numpy(), rep


def assert_same_as_oracle(v, f):
    vk, fk, rk = kernel(v, f)
    vo, fo, ro = mco.mesh_clean(v, f)
    assert vk.tobytes() == vo.tobytes() and fk.tobytes() == fo.tobytes()
    assert rk == ro, {k: (rk[k], ro[k]) for k in ro if rk[k] != ro[k]}
    return vk, fk, rk


@pytest.mark.parametrize('name', sorted(mcc.cases()))
def test_hand_cases_match_the_oracle(name):
    v, f, _ = mcc.cases()[name]
    assert_same_as_oracle(v, f)


def _abc(i):
    g = load_golden('mesh_sdf.npz')
    return g['verts_%d' % i].astype(np.float32), g['faces_%d' % i].astype(np.int32)


def _mc(kind, res):
    """a marching-cubes sphere or torus, cleaned once: the clean original of the corruption tests"""
    x = torch.linspace(-1, 1, res, device=DEV)
    X, Y, Z = torch.meshgrid(x, x, x, indexing='ij')
    if kind == 'sphere':
        vol = 0.6 - torch.sqrt(X * X + Y * Y + Z * Z)
    else:
        vol = 0.25 - torch.sqrt((torch.sqrt(X * X + Y * Y) - 0.55) ** 2 + Z * Z)
    v, f = ops.marching_cubes(vol.contiguous(), 0.0)
    v, f = v.cpu().numpy(), f.cpu().numpy()
    vo, fo, rep = kernel(v, sdf._orient_outward(v, f))
    assert rep['watertight'] and rep['winding_consistent'] and rep['volume'] > 0
    return vo, fo


MESHES = {'abc0': lambda: _abc(0), 'abc1': lambda: _abc(1), 'abc2': lambda: _abc(2),
          'sphere': lambda: _mc('sphere', 40), 'torus': lambda: _mc('torus', 48)}


@pytest.mark.parametrize('i', [0, 1, 2])
def test_abc_minimal_comes_back_bit_identical(i):
    v, f = _abc(i)
    vk, fk, rep = kernel(v, f)
    assert vk.tobytes() == v.tobytes() and fk.tobytes() == f.tobytes()
    assert rep['watertight'] and rep['winding_consistent'] and rep['components'] == 0


def _far_triangle_and_pair(f):
    """face 0, and two faces sharing an edge that touch no vertex of face 0's one-ring"""
    ring = set(f[np.isin(f, f[0]).any(1)].reshape(-1).tolist())
    for j in range(len(f) - 1, 0, -1):
        if ring & set(f[j].tolist()):
            continue
        nb = [k for k in np.nonzero(np.isin(f, f[j]).sum(1) == 2)[0] if not ring & set(f[k].tolist())]
        if nb:
            return j, nb[0]
    raise AssertionError('no pair found')


def corrupt(kind, v, f, rng):
    """-> (verts, faces, expected report fields)"""
    F = len(f)
    if kind == 'soup':
        return (*mcc.soup(v, f), dict(merged_vertices=3 * F - len(v)))
    if kind == 'reverse':
        rows = rng.choice(F, int(0.3 * F), replace=False)
        return v, mcc.flip(f, rows), dict(faces_reversed=len(rows))
    if kind == 'append':
        dup = f[rng.choice(F, 20, replace=False)]
        dup[::2] = dup[::2, ::-1]
        # 19 faces with a repeated index and a sliver of altitude 1e-9 on three new vertices
        sv = np.array([[10, 0, 0], [11, 0, 0], [10.5, 1e-9, 0]], np.float32)
        deg = np.concatenate([f[10:29, [0, 0, 1]], [[len(v), len(v) + 1, len(v) + 2]]])
        return (np.concatenate([v, sv]), np.concatenate([f, dup, deg]).astype(np.int32),
                dict(duplicate_faces=20, degenerate_faces=20, unreferenced_vertices=3))
    if kind == 'unreferenced':
        return np.concatenate([v, rng.rand(25, 3).astype(np.float32) + 5]), f, dict(unreferenced_vertices=25)
    if kind == 'delete':
        j, k = _far_triangle_and_pair(f)
        keep = np.ones(F, bool)
        keep[[0, j, k]] = False
        return v, f[keep], dict(holes_filled=2, faces_added=3)
    raise ValueError(kind)


@pytest.mark.parametrize('mesh', sorted(MESHES))
@pytest.mark.parametrize('kind', ['soup', 'reverse', 'append', 'unreferenced', 'delete'])
def test_corruptions_are_repaired(mesh, kind):
    v0, f0 = MESHES[mesh]()
    v, f, expect = corrupt(kind, v0, f0, np.random.RandomState(7))
    vk, fk, rep = assert_same_as_oracle(v, f)
    for k, val in expect.items():
        assert rep[k] == val, (k, rep[k], val)
    assert rep['watertight'] and rep['winding_consistent'] and rep['volume'] > 0
    assert rep['faces_out'] == len(f0) and rep['vertices_out'] == len(v0)
    if kind != 'delete':
        assert np.array_equal(vk[fk], v0[f0])                   # same faces in order, up to vertex renumbering
    else:
        got, want = mcc.canonical(vk, fk), mcc.canonical(v0, f0)
        extra = [t for t in got if t not in set(want)]
        assert len(extra) <= 2                                  # only the quad's diagonal may differ
        assert np.array_equal(vk[fk[:-3]], v0[f0][np.isin(np.arange(len(f0)), [0] + list(_far_triangle_and_pair(f0)),
                                                          invert=True)])
    assert abs(rep['volume'] - mco.mesh_clean(v0, f0)[2]['volume']) <= 1e-3 * rep['volume']


def test_deterministic_across_runs():
    v0, f0 = _mc('torus', 64)
    rng = np.random.RandomState(1)
    v, f = mcc.soup(v0, mcc.flip(f0, rng.choice(len(f0), len(f0) // 3, replace=False)))
    a, b = kernel(v, f), kernel(v, f)
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes() and a[2] == b[2]


def test_large_corrupted_case_matches_the_oracle():
    v0, f0 = _mc('torus', 300)
    assert len(f0) >= 200000
    rng = np.random.RandomState(2)
    f = mcc.flip(f0, rng.choice(len(f0), int(0.3 * len(f0)), replace=False))
    j, k = _far_triangle_and_pair(f0)
    keep = np.ones(len(f), bool)
    keep[[0, j, k]] = False
    v, f = mcc.soup(v0, np.concatenate([f[keep], f[keep][:50]]))
    _, _, rep = assert_same_as_oracle(v, f)
    assert rep['watertight'] and rep['winding_consistent'] and rep['holes_filled'] == 2 and rep['duplicate_faces'] == 50


def test_errors():
    v, f = cu(mcc.TET_V), cu(mcc.TET_F)
    for bad in (mcc.TET_F + 1, mcc.TET_F - 1):
        with pytest.raises(ops.P2SError, match='outside'):
            ops.mesh_clean(v, cu(bad))
    with pytest.raises(ops.P2SError, match='9e10'):
        ops.mesh_clean(cu(mcc.TET_V * np.float32(1e11)), f)
    lib = ops._lib.load()
    soup_v, soup_f = (cu(a) for a in mcc.soup(mcc.TET_V, mcc.TET_F[:3]))    # one hole: 4 faces out of 3 in
    vout = torch.empty((12, 3), dtype=torch.float32, device=DEV)
    fout = torch.empty((3, 3), dtype=torch.int32, device=DEV)
    rep = ops._lib.CleanReport()
    status = lib.p2s_mesh_clean_dev(ops._ptr(soup_v), 9, ops._ptr(soup_f), 3, ops._ptr(vout), 12, ops._ptr(fout), 3,
                                    ops.C.byref(rep), ops._stream())
    assert status != 0 and 'fcap' in lib.p2s_last_error().decode()
    with pytest.raises(ops.P2SError):
        ops.mesh_clean(v.cpu(), f)
    vo, fo, r = ops.mesh_clean(v, f)                            # a valid call still works; empty meshes are fine
    assert len(fo) == 4 and r['watertight']
    vo, fo, r = ops.mesh_clean(v, f[:0])
    assert len(vo) == 0 and len(fo) == 0 and r['unreferenced_vertices'] == 4


def test_chain_from_base_meshes_to_training_epoch(tmp_path):
    from points2surf_b200 import points_to_surf_train as p2s_train
    g = load_golden('mesh_sdf.npz')
    names = [str(g['name_%d' % i])[:-4] for i in range(3)]
    root = tmp_path / 'data'
    base = root / '00_base_meshes'
    (base / 'nested').mkdir(parents=True)
    v, f = _abc(0)
    write_stl(str(base / (names[0] + '.stl')), v, mcc.flip(f, np.arange(0, len(f), 4)), binary=True)
    v, f = _abc(1)
    write_obj(str(base / 'nested' / (names[1] + '.obj')), v, f.tolist())
    v, f = _abc(2)
    mesh_io.write_off(str(base / (names[2] + '.off')), v, f)
    (root / 'settings.ini').write_text('[general]\nonly_for_evaluation = 0\ngrid_resolution = 256\nepsilon = 5\n'
                                       'num_scans_per_mesh_min = 5\nnum_scans_per_mesh_max = 30\n'
                                       'scanner_noise_sigma_min = 0.0\nscanner_noise_sigma_max = 0.05\n')
    make_dataset.main([str(root), '--from_base_meshes', '--num_query_pts', '256'])
    for n in names:
        vm, _ = mesh_io.read_ply(str(root / '03_meshes' / (n + '.ply')))
        lo, hi = vm.min(0).astype(np.float64), vm.max(0).astype(np.float64)
        assert np.abs(lo + hi).max() <= 1e-6 and abs((hi - lo).max() - 1.0) <= 1e-6
        assert np.load(str(root / '04_pts' / (n + '.xyz.npy'))).shape[0] > 10000
        assert (root / '05_query_pts' / (n + '.ply.npy')).exists() and (root / '05_query_dist' / (n + '.ply.npy')).exists()
    assert sorted((root / 'testset.txt').read_text().split('\n')) == sorted(names)
    assert (root / 'valset.txt').exists() and (root / 'trainset.txt').exists()
    assert not (root / 'broken').exists()
    (root / 'trainset.txt').write_text('\n'.join(names[:2]) + '\n')
    (root / 'testset.txt').write_text(names[2] + '\n')
    opt = p2s_train.parse_arguments([
        '--name', 'chain', '--indir', str(root), '--outdir', str(tmp_path / 'models'), '--logdir', str(tmp_path / 'logs'),
        '--nepoch', '1', '--batchSize', '16', '--patches_per_shape', '32', '--points_per_patch', '300',
        '--sub_sample_size', '1000', '--patch_radius', '0.0', '--lr', '0.001', '--shared_transformer', '1',
        '--outputs', 'imp_surf_magnitude', 'imp_surf_sign', 'patch_pts_ids', 'p_index'])
    hist = p2s_train.points_to_surf_train(opt)
    assert len([h for h in hist if h[0] == 'train']) == 4 and all(np.isfinite(h[3]).all() for h in hist)
