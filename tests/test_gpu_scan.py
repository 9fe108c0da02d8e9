"""GPU tests of the scan stage: p2s_range_scan_dev against the float64 oracle (oracle/scan_oracle.py) with the reference's
own scan poses (tests/golden/scan.npz), its determinism and noise, the reference's BlenSor clouds of abc_minimal, and
make_dataset's --scan stage up to one training epoch."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import scan_oracle as so
from points2surf_b200 import make_dataset, mesh_io, ops, sdf, trafo
from helpers import load_golden

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
RES_X, RES_Y = 176, 144


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _mesh(i):
    g = load_golden('mesh_sdf.npz')
    return str(g['name_%d' % i]), g['verts_%d' % i], g['faces_%d' % i]


def _poses(i):
    g = load_golden('scan.npz')
    assert str(g['name_%d' % i]) + '.ply' == _mesh(i)[0]
    rot = np.stack([trafo.quaternion_matrix(q)[:3, :3] for q in g['rotations_%d' % i]])
    return rot, g['locations_%d' % i], float(g['sigma_%d' % i])


def _mc_mesh(kind, res):
    """closed, outward-oriented marching-cubes mesh of an analytic sphere or torus"""
    x = torch.linspace(-1, 1, res, device=DEV)
    X, Y, Z = torch.meshgrid(x, x, x, indexing='ij')
    if kind == 'sphere':
        vol = 0.6 - torch.sqrt(X * X + Y * Y + Z * Z)
    else:
        vol = 0.25 - torch.sqrt((torch.sqrt(X * X + Y * Y) - 0.55) ** 2 + Z * Z)
    v, f = ops.marching_cubes(vol.contiguous(), 0.0)
    v, f = v.cpu().numpy(), f.cpu().numpy()
    return v, sdf._orient_outward(v, f)


def _pixels(clean, R, loc):
    """pixel index of each noise-free hit (the ray through its pixel centre)"""
    p = clean.astype(np.float64) @ R.T + loc
    tw, th = math.tan(math.radians(43.6 / 2)), math.tan(math.radians(34.6 / 2))
    col = np.floor(((p[:, 2] / p[:, 1]) / tw + 1.0) / 2.0 * RES_X).astype(np.int64)
    row = np.floor((1.0 - (p[:, 0] / p[:, 1]) / th) / 2.0 * RES_Y).astype(np.int64)
    return row * RES_X + col


def _compare_with_oracle(v, f, rot, loc, scans):
    noisy, clean, face, hps = ops.range_scan(cu(v), cu(f), rot, loc)
    noisy, clean, face, hps = (t.cpu().numpy() for t in (noisy, clean, face, hps))
    assert np.array_equal(noisy, clean)   # no noise
    assert hps.sum() == len(clean)
    off = np.concatenate([[0], np.cumsum(hps)])
    ref = so.range_scan(v, f, rot[scans], loc[scans])
    checked = 0
    for s, r in zip(scans, ref):
        c, fc = clean[off[s]:off[s + 1]], face[off[s]:off[s + 1]]
        pix = _pixels(c, rot[s], loc[s])
        assert np.all(np.diff(pix) > 0)                          # (row, col) order, one hit per ray
        hit_o = np.isfinite(r['t'])
        hit_k = np.zeros(len(hit_o), bool)
        hit_k[pix] = True
        sure = r['margin'] >= 1e-6
        assert np.array_equal(hit_k[sure], hit_o[sure]), (s, np.sum(hit_k[sure] != hit_o[sure]))
        both = hit_o[pix]
        t_k = np.linalg.norm(c[both].astype(np.float64) - r['origin'], axis=1)
        t_o = r['t'][pix[both]]
        assert np.all(np.abs(t_k - t_o) <= 1e-5 * t_o)
        diff = fc[both] != r['face'][pix[both]]
        sure_b = sure[pix[both]]
        # a different face only on a tie: the oracle's t through the kernel's face equals its own
        for k in np.nonzero(diff & sure_b)[0]:
            tf, ff, _ = so.cast(v, f[[fc[both][k]]], r['origin'], r['dirs'][[pix[both][k]]])
            assert ff[0] == 0 and abs(tf[0] - t_o[k]) <= 1e-9 * t_o[k]
        checked += int(both.sum())
    return checked, hps


@pytest.mark.parametrize('i', [0, 1, 2])
def test_abc_minimal_against_oracle(i):
    _, v, f = _mesh(i)
    rot, loc, _ = _poses(i)
    checked, hps = _compare_with_oracle(v, f, rot, loc, [0, len(loc) - 1])
    assert checked > 2000 and len(hps) == len(loc)


@pytest.mark.parametrize('kind,res', [('sphere', 40), ('torus', 48)])
def test_marching_cubes_meshes_against_oracle(kind, res):
    v, f = _mc_mesh(kind, res)
    rot, loc, _ = _poses(2)
    checked, _ = _compare_with_oracle(v, f, rot[:3], loc[:3], [0, 1, 2])
    assert checked > 5000


def test_deterministic_and_independent_of_scan_batching():
    _, v, f = _mesh(1)
    rot, loc, sigma = _poses(1)
    V, F = cu(v), cu(f)
    a = [t.cpu().numpy() for t in ops.range_scan(V, F, rot, loc, noise_sigma=sigma, seed=11)]
    b = [t.cpu().numpy() for t in ops.range_scan(V, F, rot, loc, noise_sigma=sigma, seed=11)]
    parts = [[t.cpu().numpy() for t in ops.range_scan(V, F, rot[s:s + 1], loc[s:s + 1], noise_sigma=sigma, seed=11,
                                                      first_scan=s)] for s in range(len(loc))]
    for k in range(4):
        assert a[k].tobytes() == b[k].tobytes()
        assert a[k].tobytes() == np.concatenate([p[k] for p in parts]).tobytes()
    assert not np.array_equal(a[0], a[1])   # the noise is on
    c = ops.range_scan(V, F, rot, loc, noise_sigma=sigma, seed=12)
    assert np.array_equal(c[1].cpu().numpy(), a[1]) and not np.array_equal(c[0].cpu().numpy(), a[0])


def test_range_noise_is_standard_normal():
    v, f = _mc_mesh('torus', 48)
    rot, loc, _ = _poses(0)
    sigma = 0.01
    noisy, clean, _, hps = ops.range_scan(cu(v), cu(f), rot, loc, noise_sigma=sigma, seed=5)
    noisy, clean, hps = noisy.cpu().numpy().astype(np.float64), clean.cpu().numpy().astype(np.float64), hps.cpu().numpy()
    origins = np.repeat(np.stack([-(R.T @ l) for R, l in zip(rot, loc)]), hps, axis=0)
    z = (np.linalg.norm(noisy - origins, axis=1) - np.linalg.norm(clean - origins, axis=1)) / sigma
    n = len(z)
    assert n > 20000
    assert abs(z.mean()) <= 5.0 / math.sqrt(n)
    assert abs(z.std() - 1.0) <= 5.0 / math.sqrt(2 * n)
    # the noise is along the ray: the noisy point stays on the line from the scanner through the clean one
    u = (clean - origins) / np.linalg.norm(clean - origins, axis=1, keepdims=True)
    w = noisy - origins
    assert np.abs(w - (w * u).sum(1, keepdims=True) * u).max() < 1e-5


def _write_meshes(mesh_dir):
    os.makedirs(mesh_dir, exist_ok=True)
    for i in range(3):
        name, v, f = _mesh(i)
        mesh_io.write_ply(os.path.join(mesh_dir, name), v, f)


def test_sample_blensor_against_the_reference_clouds(tmp_path):
    root = tmp_path / 'abc'
    _write_meshes(str(root / '03_meshes'))
    make_dataset.sample_blensor(str(tmp_path), 'abc', None, '03_meshes', '04_pts_raw', '04_pts', '04_pts_vis', '04_pcd',
                                '04_blensor_py', '04_locations', '04_rotations', 5, 30, 8, min_pts_size=100,
                                scanner_noise_sigma_min=0.0, scanner_noise_sigma_max=0.05)
    g = load_golden('scan.npz')
    for i in range(3):
        stem = str(g['name_%d' % i])
        _, v, f = _mesh(i)
        pts = np.load(str(root / '04_pts' / (stem + '.xyz.npy')))
        hps = np.load(str(root / '04_hits_per_scan' / (stem + '.npz')))['hits_per_scan']
        assert pts.dtype == np.float32 and pts.shape[1] == 6 and hps.sum() == len(pts) and len(hps) == g['num_scans_%d' % i]
        ref_n = int(g['ref_num_pts_%d' % i])
        assert abs(len(pts) - ref_n) <= 0.01 * ref_n, (stem, len(pts), ref_n)
        d = np.abs(ops.mesh_signed_distance(cu(v), cu(f), cu(pts[:, :3])).cpu().numpy())
        q = np.quantile(d, g['quantiles'])
        ref_q = g['ref_dist_quantiles_%d' % i]
        assert np.all(np.abs(q - ref_q) <= 0.15 * ref_q), (stem, q, ref_q)
        np.testing.assert_allclose(np.linalg.norm(pts[:, 3:], axis=1), 1.0, atol=1e-6)
        assert (root / '04_pts_vis' / (stem + '.xyz')).exists()
        assert np.array_equal(np.load(str(root / '04_locations' / (stem + '.npz')))['locations'], g['locations_%d' % i])


def test_errors():
    v = cu(np.eye(3, dtype=np.float32))
    rot, loc = np.eye(3)[None], np.array([[0.0, 4.0, 0.0]])
    for bad in ([[0, 1, 3]], [[0, -1, 2]]):
        with pytest.raises(ops.P2SError):
            ops.range_scan(v, cu(np.array(bad, np.int32)), rot, loc)
    with pytest.raises(ops.P2SError):
        ops.range_scan(v.cpu(), cu(np.array([[0, 1, 2]], np.int32)), rot, loc)
    with pytest.raises(ops.P2SError):
        ops.range_scan(v, np.array([[0, 1, 2]], np.int32), rot, loc)
    with pytest.raises(ops.P2SError):
        ops.range_scan(v, cu(np.array([[0, 1, 2]], np.int32)), rot, loc, noise_sigma=-1.0)
    # a valid call still works after the errors; no scans is fine
    tri = cu(np.array([[-1, 0, -1], [1, 0, -1], [0, 0, 1]], np.float32))
    noisy, clean, face, hps = ops.range_scan(tri, cu(np.array([[0, 1, 2]], np.int32)), rot, loc)
    assert len(noisy) == int(hps[0]) > 1000 and (face == 0).all()
    assert ops.range_scan(tri, cu(np.array([[0, 1, 2]], np.int32)), rot[:0], loc[:0])[0].shape == (0, 3)


def test_chain_mesh_to_scan_to_training_epoch(tmp_path):
    from points2surf_b200 import points_to_surf_train as p2s_train
    root = tmp_path / 'data'
    _write_meshes(str(root / '03_meshes'))
    (root / 'settings.ini').write_text('[general]\nonly_for_evaluation = 0\ngrid_resolution = 256\nepsilon = 5\n'
                                       'num_scans_per_mesh_min = 5\nnum_scans_per_mesh_max = 30\n'
                                       'scanner_noise_sigma_min = 0.0\nscanner_noise_sigma_max = 0.05\n')
    make_dataset.main([str(root), '--scan', '--num_query_pts', '256'])
    names = [_mesh(i)[0][:-4] for i in range(3)]
    for n in names:
        assert np.load(str(root / '04_pts' / (n + '.xyz.npy'))).shape[0] > 10000
        assert (root / '05_query_dist' / (n + '.ply.npy')).exists()
    (root / 'trainset.txt').write_text('\n'.join(names[:2]) + '\n')
    (root / 'testset.txt').write_text(names[2] + '\n')
    opt = p2s_train.parse_arguments([
        '--name', 'chain', '--indir', str(root), '--outdir', str(tmp_path / 'models'), '--logdir', str(tmp_path / 'logs'),
        '--nepoch', '1', '--batchSize', '16', '--patches_per_shape', '32', '--points_per_patch', '300',
        '--sub_sample_size', '1000', '--patch_radius', '0.0', '--lr', '0.001', '--shared_transformer', '1',
        '--outputs', 'imp_surf_magnitude', 'imp_surf_sign', 'patch_pts_ids', 'p_index'])
    hist = p2s_train.points_to_surf_train(opt)
    assert len([h for h in hist if h[0] == 'train']) == 4 and all(np.isfinite(h[3]).all() for h in hist)
