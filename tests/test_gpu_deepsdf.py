"""GPU test of the dataset_for_deepsdf CLI on a small dataset tree made from the abc_minimal shapes: repaired meshes,
SdfSamples, SurfaceSamples and examples with the expected names, keys and counts; a second run writes nothing."""
import os

import numpy as np
import pytest

from points2surf_b200 import dataset_for_deepsdf as dsd, mesh_io
from helpers import load_golden
import mesh_repair_cases as mrc

pytestmark = pytest.mark.gpu


def _dataset(root):
    sd, g = load_golden('mesh_sdf.npz'), load_golden('deepsdf.npz')
    ds = root / 'tiny'
    names = []
    for i in range(3):
        name = str(sd['name_%d' % i])[:-4]
        names.append(name)
        f = mrc.delete_random_faces(sd['faces_%d' % i], seed=i)          # holes for the repair to close
        mesh_io.write_ply(str(ds / '03_meshes' / (name + '.ply')), sd['verts_%d' % i], f)
        mesh_io.make_dir_for_file(str(ds / '04_pts' / 'x'))
        np.save(ds / '04_pts' / (name + '.xyz.npy'), g['pts_%d' % i])
        mesh_io.make_dir_for_file(str(ds / '05_query_pts' / 'x'))
        mesh_io.make_dir_for_file(str(ds / '05_query_dist' / 'x'))
        np.save(ds / '05_query_pts' / (name + '.ply.npy'), g['query_pts_%d' % i])
        np.save(ds / '05_query_dist' / (name + '.ply.npy'), g['query_dist_%d' % i])
        mesh_io.make_dir_for_file(str(ds / '06_normals_pcpnet' / 'x'))
        (ds / '06_normals_pcpnet' / (name + '.normals')).write_text(str(g['normals_text_%d' % i]))
    (ds / 'trainset.txt').write_text('\n'.join(names[:2]) + '\n')
    (ds / 'testset.txt').write_text(names[2] + '\n')
    return ds, names, g


def _mtimes(root):
    return {os.path.join(r, n): os.path.getmtime(os.path.join(r, n)) for r, _, ns in os.walk(root) for n in ns}


def test_cli_writes_the_deepsdf_tree(tmp_path):
    ds, names, g = _dataset(tmp_path)
    out = tmp_path / 'DeepSDF'
    dsd.main([str(ds), '--out_dir', str(out)])
    assert sorted(os.listdir(ds / '05_meshes_repaired')) == sorted(n + '.ply' for n in names)
    for n in names:
        v, f = mesh_io.read_ply(str(ds / '05_meshes_repaired' / (n + '.ply')))
        v0, f0 = mesh_io.read_ply(str(ds / '03_meshes' / (n + '.ply')))
        assert len(f) > len(f0)                                         # the holes were closed
    sdf_dir = out / 'data' / 'SdfSamples' / 'tiny' / '03_meshes'
    assert sorted(os.listdir(sdf_dir)) == sorted([n + '.npz' for n in names] + [names[2] + '.npz.ply'])
    for i, n in enumerate(names[:2]):
        s = np.load(sdf_dir / (n + '.npz'))
        assert sorted(s.files) == ['neg', 'pos']
        assert s['pos'].tobytes() == g['train_pos_%d' % i].tobytes() and s['neg'].tobytes() == g['train_neg_%d' % i].tobytes()
    s = np.load(sdf_dir / (names[2] + '.npz'))
    N = len(g['pts_2'])
    assert sorted(s.files) == ['neg', 'neg_far', 'pos', 'pos_far']
    assert all(s[k].dtype == np.float32 and s[k].shape[1] == 4 for k in s.files)
    assert s['pos'].tobytes() == g['pos_2'].tobytes() and s['neg'].tobytes() == g['neg_2'].tobytes()
    assert len(s['pos_far']) + len(s['neg_far']) <= int(2 * N * 0.2) and len(s['pos_far']) > 0 and len(s['neg_far']) > 0
    assert (s['pos_far'][:, 3] > 0).all() and (s['neg_far'][:, 3] < 0).all()
    assert np.abs(s['pos_far'][:, :3]).max() <= 0.5
    assert sorted(os.listdir(out / 'data' / 'SurfaceSamples' / 'tiny' / '03_meshes')) == [names[2] + '.ply']
    v, f = mesh_io.read_ply(str(out / 'data' / 'SurfaceSamples' / 'tiny' / '03_meshes' / (names[2] + '.ply')))
    assert len(v) == N and len(f) == N
    assert sorted(os.listdir(out / 'examples' / 'splits')) == ['tiny_test.json', 'tiny_train.json']
    assert '"converted from %s."' % (ds / 'trainset.txt') in (out / 'examples' / 'tiny' / 'specs.json').read_text()

    before = _mtimes(tmp_path)
    dsd.main([str(ds), '--out_dir', str(out)])
    after = _mtimes(tmp_path)
    changed = [k for k in after if after[k] != before.get(k)]
    assert all(k.endswith('.json') for k in changed), changed         # only the example texts are rewritten
