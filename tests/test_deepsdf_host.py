"""CPU tests of the dataset_for_deepsdf mirror's host parts against the unmodified reference's output on the
abc_minimal shapes (tests/golden/deepsdf.npz, written by tests/golden/make_deepsdf_golden.py)."""
import os

import numpy as np
import pytest

from points2surf_b200 import dataset_for_deepsdf as dsd
from helpers import load_golden


@pytest.mark.parametrize('i', [0, 1, 2])
def test_close_samples_match_the_reference_bit_for_bit(i, tmp_path):
    g = load_golden('deepsdf.npz')
    (tmp_path / 'n.normals').write_text(str(g['normals_text_%d' % i]))
    normals = dsd._read_normals(str(tmp_path / 'n.normals'))
    out_p, in_p, d_out, d_in = dsd.close_samples(g['pts_%d' % i].astype(np.float32), normals)
    pos, neg = dsd._rows(in_p, d_in), dsd._rows(out_p, d_out)    # the reference's key swap
    for key, ours in (('pos', pos), ('neg', neg)):
        ref = g['%s_%d' % (key, i)]
        assert ours.dtype == ref.dtype == np.float32 and ours.shape == ref.shape
        assert ours.tobytes() == ref.tobytes()
    assert (pos[:, 3] == np.float32(0.01)).all() and (neg[:, 3] == np.float32(-0.01)).all()


@pytest.mark.parametrize('i', [0, 1, 2])
def test_far_samples_are_the_reference_stream(i, tmp_path):
    g = load_golden('deepsdf.npz')
    mesh = tmp_path / str(g['name_%d' % i])
    mesh.write_bytes(b'x')                                   # filename_to_hash needs a file; only its name counts
    far = dsd.far_samples(2 * len(g['pts_%d' % i]), str(mesh)).astype(np.float32)
    ref = np.concatenate([g['pos_far_%d' % i], g['neg_far_%d' % i]])
    assert ref.dtype == np.float32 and len(far) == int(2 * len(g['pts_%d' % i]) * 0.2) >= len(ref)
    ours = {r.tobytes() for r in far}
    assert all(r[:3].tobytes() in ours for r in ref)
    assert (g['pos_far_%d' % i][:, 3] > 0).all() and (g['neg_far_%d' % i][:, 3] < 0).all()


@pytest.mark.parametrize('i', [0, 1, 2])
def test_convert_sdf_matches_the_reference(i, tmp_path):
    g = load_golden('deepsdf.npz')
    np.save(tmp_path / 'q.npy', g['query_pts_%d' % i])
    np.save(tmp_path / 'd.npy', g['query_dist_%d' % i])
    dsd._convert_sdf(str(tmp_path / 'q.npy'), str(tmp_path / 'd.npy'), str(tmp_path / 'o.npz'))
    o = np.load(tmp_path / 'o.npz')
    assert sorted(o.files) == ['neg', 'pos']
    for k in ('pos', 'neg'):
        ref = g['train_%s_%d' % (k, i)]
        assert o[k].dtype == np.float32 and o[k].tobytes() == ref.tobytes()


def test_specs_and_split_texts_byte_for_byte(tmp_path, monkeypatch):
    g = load_golden('deepsdf.npz')
    (tmp_path / 'trainset.txt').write_text(str(g['trainset']))
    (tmp_path / 'testset.txt').write_text(str(g['testset']))
    monkeypatch.chdir(tmp_path)
    dsd.create_example('trainset.txt', 'testset.txt', str(tmp_path / 'examples'), 'abc_minimal')
    ex = tmp_path / 'examples'
    assert (ex / 'abc_minimal' / 'specs.json').read_text() == str(g['specs_json'])
    assert (ex / 'splits' / 'abc_minimal_train.json').read_text() == str(g['train_json'])
    assert (ex / 'splits' / 'abc_minimal_test.json').read_text() == str(g['test_json'])


def test_set_file_filter_uses_basename_minus_eight_characters(tmp_path):
    d = tmp_path / 'pts'
    d.mkdir()
    for n in ('a', 'b'):
        np.save(d / (n + '.xyz.npy'), np.zeros((3, 3), np.float32))
    (tmp_path / 'set.txt').write_text('a\n')
    dsd.convert_pcs(str(d), str(tmp_path / 'out'), str(tmp_path / 'set.txt'), 1)
    assert sorted(os.listdir(tmp_path / 'out')) == ['a.ply']
    from points2surf_b200 import mesh_io
    v, f = mesh_io.read_ply(str(tmp_path / 'out' / 'a.ply'))
    assert len(v) == 3 and f.tolist() == [[0, 1, 0], [0, 1, 1], [0, 1, 2]]


MLX = '<!DOCTYPE FilterScript>\n<FilterScript>\n%s</FilterScript>\n'


def test_hole_filling_filter_script(tmp_path):
    ok = tmp_path / 'ok.mlx'
    ok.write_text(MLX % (' <filter name="Repair non Manifold Edges by removing faces"/>\n'
                         ' <filter name="Repair non Manifold Edges by splitting vertices"/>\n'
                         ' <filter name="Repair non Manifold Vertices by splitting">'
                         '<Param name="VertDispRatio" value="0" type="RichFloat"/></filter>\n'
                         ' <filter name="Close Holes"><Param name="MaxHoleSize" value="12" type="RichInt"/>'
                         '<Param name="SelfIntersection" value="false" type="RichBool"/></filter>\n'
                         ' <filter name="Simplification: Quadric Edge Collapse Decimation"/>\n'))
    assert dsd.read_hole_filling_filter(str(ok)) == dict(max_hole_size=12, prevent_self_intersection=False)
    for body in (' <filter name="Screened Poisson Surface Reconstruction"/>\n',
                 ' <filter name="Close Holes"/>\n <filter name="Repair non Manifold Edges by removing faces"/>\n',
                 ' <filter name="Repair non Manifold Vertices by splitting">'
                 '<Param name="VertDispRatio" value="0.5" type="RichFloat"/></filter>\n',
                 ' <filter name="Close Holes"><Param name="Selected" value="true" type="RichBool"/></filter>\n'):
        bad = tmp_path / 'bad.mlx'
        bad.write_text(MLX % body)
        with pytest.raises(ValueError):
            dsd.read_hole_filling_filter(str(bad))
