"""CPU tests of the mesh-cleaning stages: the float64 oracle of csrc/meshclean.cu (oracle/mesh_clean_oracle.py) on
hand-built cases and on the reference's own cleaned meshes, the accept / reject decisions of _clean_mesh, the normalise
restatement, the mesh readers, and make_dataset_splits / clean_up_broken_inputs against the reference's own results
(tests/golden/dataset_stages.npz)."""
import os
import struct
import sys

import numpy as np
import pytest

from oracle import mesh_clean_oracle as mco
from points2surf_b200 import make_dataset, mesh_io
from helpers import load_golden
import mesh_clean_cases as mcc

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import make_dataset_stages_golden as stages  # noqa: E402

CASES = mcc.cases()


@pytest.mark.parametrize('name', sorted(CASES))
def test_oracle_hand_cases(name):
    v, f, expect = CASES[name]
    vo, fo, rep = mco.mesh_clean(v, f)
    for k, val in expect.items():
        if k == 'volume':
            assert rep[k] == pytest.approx(val, rel=1e-12), (k, rep[k], val)
        else:
            assert rep[k] == val, (k, rep[k], val)
    assert rep['vertices_out'] == len(vo) and rep['faces_out'] == len(fo)
    assert rep['vertices_in'] - rep['merged_vertices'] - rep['unreferenced_vertices'] == len(vo)
    assert len(np.unique(fo)) == len(vo)                       # no unreferenced vertex left


def test_oracle_repairs_back_to_the_original():
    for name, (v0, f0) in {'tet': (mcc.TET_V, mcc.TET_F), 'cube': (mcc.CUBE_V, mcc.CUBE_F)}.items():
        for case in (name, name + '_soup'):
            vo, fo, _ = mco.mesh_clean(*CASES[case][:2])
            assert np.array_equal(vo[fo], v0[f0]), case          # same faces in the same order, up to renumbering
    for case in ('cube_one_reversed', 'cube_first_reversed', 'duplicates', 'slivers', 'unreferenced_and_nan'):
        vo, fo, _ = mco.mesh_clean(*CASES[case][:2])
        assert np.array_equal(vo, mcc.CUBE_V) and np.array_equal(fo, mcc.CUBE_F), case
    vo, fo, _ = mco.mesh_clean(*CASES['tet_missing_triangle'][:2])
    assert np.array_equal(fo, mcc.TET_F)                       # the fill runs opposite to the loop: outward
    vo, fo, _ = mco.mesh_clean(*CASES['cube_missing_quad'][:2])
    assert mcc.canonical(vo, fo) == mcc.canonical(mcc.CUBE_V, mcc.CUBE_F)   # diagonal through vertex 0, as removed
    vo, fo, _ = mco.mesh_clean(*CASES['cube_inverted'][:2])
    assert np.array_equal(fo, mcc.CUBE_F[:, ::-1])             # consistent: not flipped
    v, f, _ = CASES['mobius']
    vo, fo, _ = mco.mesh_clean(v, f)
    assert np.array_equal(vo, v) and np.array_equal(fo, f)     # non-orientable: left as it came
    vo, fo, _ = mco.mesh_clean(*CASES['two_bodies_one_inverted'][:2])
    assert np.array_equal(fo[4:], mcc.CUBE_F + 4) and np.array_equal(fo[:4], mcc.TET_F)


def test_accept_decisions_of_clean_mesh():
    def accept(case, num_max_faces=None, enforce_solid=True, num_faces=None):
        _, fo, rep = mco.mesh_clean(*CASES[case][:2])
        return make_dataset._accept_cleaned(rep, len(fo) if num_faces is None else num_faces, num_max_faces,
                                            enforce_solid)
    assert accept('cube') and accept('cube_one_reversed') and accept('tet_missing_triangle')
    assert accept('cube_missing_quad') and accept('two_bodies_one_inverted')
    assert not accept('cube_inverted')                          # is_volume: negative volume
    assert not accept('missing_pentagon') and not accept('mobius') and not accept('three_face_edge')
    assert accept('missing_pentagon', enforce_solid=False) and accept('cube_inverted', enforce_solid=False)
    # the 50 000-face cap of make_dataset: strictly fewer faces are written
    assert accept('cube', 50000, num_faces=49999) and not accept('cube', 50000, num_faces=50000)
    assert accept('cube', None, num_faces=10 ** 7)


@pytest.mark.parametrize('i', [0, 1, 2])
def test_oracle_is_identity_on_the_reference_cleaned_meshes(i):
    g = load_golden('mesh_sdf.npz')
    v, f = g['verts_%d' % i], g['faces_%d' % i]
    vo, fo, rep = mco.mesh_clean(v, f)
    assert vo.tobytes() == v.astype(np.float32).tobytes() and fo.tobytes() == f.astype(np.int32).tobytes()
    assert rep['watertight'] and rep['winding_consistent'] and rep['volume'] > 0 and rep['components'] == 0


def test_oracle_errors_and_helpers():
    with pytest.raises(ValueError):
        mco.mesh_clean(mcc.TET_V, mcc.TET_F + 1)
    with pytest.raises(ValueError):
        mco.mesh_clean(mcc.TET_V * np.float32(1e11), mcc.TET_F)
    y = np.array([0.5, -0.5, 1.5, 2.4999999999999996, -2.5, 4503599627370497.0, 9e18 - 1024])
    assert mco.llround(y).tolist() == [1, -1, 2, 2, -3, 4503599627370497, int(9e18 - 1024)]
    d = np.random.RandomState(0).randn(1000)
    assert mco.fixed_sum(d) == pytest.approx(d.sum(), rel=1e-12) and mco.fixed_sum([]) == 0.0


def test_normalize_restatement(tmp_path):
    v = np.array([[1, 2, 3], [3, 2, 4], [2, 6, 3]], np.float32)
    out = make_dataset.normalized_vertices(v)
    # extents (2, 4, 1): centre (2, 4, 3.5), scale 1/4
    assert np.array_equal(out, np.array([[-0.25, -0.5, -0.125], [0.25, -0.5, 0.125], [0, 0.5, -0.125]], np.float32))
    v2 = np.array([[0.1, 0.2, 0.3], [0.7, 0.25, 0.9], [0.4, 1.0, 0.35]], np.float32)
    v64 = v2.astype(np.float64)
    t = -((v64.min(0) + v64.max(0)) * 0.5)
    s = 1.0 / (v64.max(0) - v64.min(0)).max()
    assert np.array_equal(make_dataset.normalized_vertices(v2), ((v64 + t) * s).astype(np.float32))
    assert make_dataset.normalized_vertices(np.array([[0, 0, 0], [1, 1, 0], [2, 0, 0]], np.float32)) is None
    # the file stage: a flat mesh writes nothing
    mesh_io.write_ply(str(tmp_path / 'flat.ply'), [[0, 0, 0], [1, 1, 0], [2, 0, 0]], [[0, 1, 2]])
    mesh_io.write_ply(str(tmp_path / 'ok.ply'), v, [[0, 1, 2]])
    make_dataset._normalize_mesh(str(tmp_path / 'flat.ply'), str(tmp_path / 'flat_out.ply'))
    make_dataset._normalize_mesh(str(tmp_path / 'ok.ply'), str(tmp_path / 'ok_out.ply'))
    assert not (tmp_path / 'flat_out.ply').exists()
    vo, fo = mesh_io.read_ply(str(tmp_path / 'ok_out.ply'))
    assert np.array_equal(vo, out) and fo.tolist() == [[0, 1, 2]]


# ---- mesh readers
def write_obj(path, v, polygons):
    with open(path, 'w') as fp:
        fp.write('# test\no shape\n')
        for x in v:
            fp.write('v %r %r %r\nvt 0 0\nvn 0 0 1\n' % tuple(float(c) for c in x))
        for k, p in enumerate(polygons):
            if k % 3 == 0:
                fp.write('f ' + ' '.join('%d/%d/%d' % (i + 1, i + 1, i + 1) for i in p) + '\n')
            elif k % 3 == 1:
                fp.write('f ' + ' '.join('%d//%d' % (i - len(v), i + 1) for i in p) + '\n')   # negative indices
            else:
                fp.write('f ' + ' '.join(str(i + 1) for i in p) + '\n')


def write_stl(path, v, f, binary):
    tri = np.asarray(v, np.float32)[np.asarray(f)]
    if binary:
        with open(path, 'wb') as fp:
            fp.write(b'\0' * 80 + struct.pack('<I', len(tri)))
            for t in tri:
                fp.write(struct.pack('<3f', 0, 0, 0) + t.astype('<f4').tobytes() + b'\0\0')
    else:
        with open(path, 'w') as fp:
            fp.write('solid shape\n')
            for t in tri:
                fp.write('facet normal 0 0 0\n outer loop\n' + ''.join('  vertex %r %r %r\n' % tuple(float(c) for c in x)
                                                                     for x in t) + ' endloop\nendfacet\n')
            fp.write('endsolid shape\n')


def write_off_polygons(path, v, polygons):
    with open(path, 'w') as fp:
        fp.write('OFF\n# comment\n%d %d 0\n' % (len(v), len(polygons)))
        for x in v:
            fp.write('%r %r %r\n' % tuple(float(c) for c in x))
        for p in polygons:
            fp.write('%d %s\n' % (len(p), ' '.join(map(str, p))))


def test_readers_round_trip(tmp_path):
    rng = np.random.RandomState(3)
    v = rng.rand(9, 3).astype(np.float32)
    polygons = [[0, 1, 2], [2, 3, 4, 5], [5, 6, 7, 8, 0], [1, 3, 5]]
    fan = np.array([[0, 1, 2], [2, 3, 4], [2, 4, 5], [5, 6, 7], [5, 7, 8], [5, 8, 0], [1, 3, 5]], np.int32)
    write_obj(str(tmp_path / 'a.obj'), v, polygons)
    write_off_polygons(str(tmp_path / 'a.off'), v, polygons)
    for ext in ('obj', 'off'):
        vr, fr = mesh_io.read_mesh(str(tmp_path / ('a.' + ext)))
        assert np.array_equal(vr, v) and np.array_equal(fr, fan), ext
    for binary in (True, False):
        p = str(tmp_path / ('b%d.stl' % binary))
        write_stl(p, v, fan, binary)
        vr, fr = mesh_io.read_mesh(p)
        assert np.array_equal(vr[fr], v[fan]) and len(vr) == 3 * len(fan), binary
    # a quad fans into trimesh's triangulate_quads triangles (a, b, c), (c, d, a) up to rotation
    q = mesh_io._fan([[4, 5, 6, 7]])
    assert q.tolist() == [[4, 5, 6], [4, 6, 7]]
    with pytest.raises(ValueError):
        mesh_io.read_mesh(str(tmp_path / 'a.xyz'))


def test_convert_meshes_skips_unreadable_files(tmp_path, capsys):
    src = tmp_path / '00_base_meshes'
    (src / 'sub').mkdir(parents=True)
    write_obj(str(src / 'sub' / 'good.obj'), mcc.CUBE_V, mcc.CUBE_F.tolist())
    (src / 'bad.stl').write_text('not a mesh at all')
    (src / 'ignored.txt').write_text('x')
    make_dataset.convert_meshes(str(src), str(tmp_path / '01_base_meshes_ply'), '.ply')
    assert sorted(os.listdir(str(tmp_path / '01_base_meshes_ply'))) == ['good.ply']
    vr, fr = mesh_io.read_ply(str(tmp_path / '01_base_meshes_ply' / 'good.ply'))
    assert np.array_equal(vr, mcc.CUBE_V) and np.array_equal(fr, mcc.CUBE_F)
    assert 'not an STL file' in capsys.readouterr().out


# ---- the reference's pure-Python stages
@pytest.mark.parametrize('n', stages.SIZES)
@pytest.mark.parametrize('only_test_set', [False, True])
def test_splits_and_clean_up_match_the_reference(n, only_test_set):
    g = load_golden('dataset_stages.npz')
    rec = stages.run_case(make_dataset.make_dataset_splits, make_dataset.clean_up_broken_inputs, n, only_test_set)
    for k, val in rec.items():
        assert val == str(g['%s_%d_%d' % (k, n, only_test_set)]), k
