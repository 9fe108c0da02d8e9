"""Write tests/golden/deepsdf.npz from the unmodified reference's dataset_for_deepsdf.py (_convert_sdf,
_make_sdf_samples_from_pc, create_example) on the abc_minimal meshes, the first 2000 points of their clouds
with synthetic normals and the first 4000 of their query points.

    python tests/golden/make_deepsdf_golden.py REFERENCE_ROOT

The reference runs under oracle/ref_shims.py; sdf.get_signed_distance is replaced by the float64 oracle
(oracle/mesh_sdf_oracle.py), trimesh.load by mesh_io.read_ply, the PLY visualisation is skipped, and np.random is seeded
with the file-name hash of the mesh (the stream the mirror draws its far samples from)."""
import os
import shutil
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_shims  # noqa: E402
from oracle import mesh_sdf_oracle as msdf  # noqa: E402
from points2surf_b200 import mesh_io, make_dataset  # noqa: E402


N_PTS, N_QUERY = 2000, 4000     # the first points of each cloud and query set keep the file small


def main(ref_root):
    ref_shims.REFERENCE_ROOT = ref_root
    ref_shims.install()
    import trimesh
    trimesh.load = lambda f: mesh_io.read_ply(f)
    from source import sdf as ref_sdf
    ref_sdf.get_signed_distance = lambda in_mesh, query_pts_ms, signed_distance_batch_size=1000: \
        msdf.mesh_signed_distance(in_mesh[0], in_mesh[1], query_pts_ms)[0]
    ref_sdf.visualize_query_points = lambda *a, **k: None
    import dataset_for_deepsdf as ref

    ds = os.path.join(ref_root, 'datasets', 'abc_minimal')
    tmp = tempfile.mkdtemp()
    out = {}
    rng = np.random.RandomState(7)
    for i, f in enumerate(sorted(os.listdir(os.path.join(ds, '03_meshes')))):
        base = f[:-4]
        mesh = os.path.join(ds, '03_meshes', f)
        pts = np.load(os.path.join(ds, '04_pts', base + '.xyz.npy'))[:N_PTS]
        pts_file = os.path.join(tmp, base + '.xyz.npy')
        np.save(pts_file, pts)
        q = np.load(os.path.join(ds, '05_query_pts', f + '.npy'))[:N_QUERY]
        d = np.load(os.path.join(ds, '05_query_dist', f + '.npy'))[:N_QUERY]
        np.save(os.path.join(tmp, 'q.npy'), q)
        np.save(os.path.join(tmp, 'd.npy'), d)
        normals = rng.randn(len(pts), 3) * rng.uniform(0.5, 2.0, (len(pts), 1))
        normals_file = os.path.join(tmp, base + '.normals')
        np.savetxt(normals_file, normals)
        np.random.seed(make_dataset.filename_to_hash(mesh))
        ref._make_sdf_samples_from_pc(pts_file, normals_file, mesh, os.path.join(tmp, 'samples.npz'))
        s = np.load(os.path.join(tmp, 'samples.npz'))
        ref._convert_sdf(os.path.join(tmp, 'q.npy'), os.path.join(tmp, 'd.npy'), os.path.join(tmp, 'train.npz'))
        t = np.load(os.path.join(tmp, 'train.npz'))
        out.update({'name_%d' % i: np.array(f), 'pts_%d' % i: pts, 'normals_text_%d' % i: np.array(open(normals_file).read()),
                    'query_pts_%d' % i: q, 'query_dist_%d' % i: d, 'hash_%d' % i: np.int64(make_dataset.filename_to_hash(mesh))})
        out.update({'%s_%d' % (k, i): s[k] for k in ('pos', 'neg', 'pos_far', 'neg_far')})
        out.update({'train_%s_%d' % (k, i): t[k] for k in ('pos', 'neg')})
        print(f, {k: s[k].shape for k in s.files})
    os.makedirs(os.path.join(tmp, 'splits'))     # the reference does not create it
    cwd = os.getcwd()
    os.chdir(ds)                                 # relative set-file paths: the specs text names the train set
    ref.create_example('trainset.txt', 'testset.txt', tmp, 'abc_minimal')
    os.chdir(cwd)
    for k, p in (('specs_json', 'abc_minimal/specs.json'), ('train_json', 'splits/abc_minimal_train.json'),
                 ('test_json', 'splits/abc_minimal_test.json')):
        out[k] = np.array(open(os.path.join(tmp, p)).read())
    out['trainset'] = np.array(open(os.path.join(ds, 'trainset.txt')).read())
    out['testset'] = np.array(open(os.path.join(ds, 'testset.txt')).read())
    shutil.rmtree(tmp)
    path = os.path.join(ROOT, 'tests', 'golden', 'deepsdf.npz')
    np.savez_compressed(path, **out)
    print('written', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main(sys.argv[1])
