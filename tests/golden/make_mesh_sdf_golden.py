"""Write tests/golden/mesh_sdf.npz: the three abc_minimal meshes with the reference's own training targets for them
(05_query_pts / 05_query_dist, written by make_dataset.py through trimesh), the reference's file-name hashes (the seeds
of the query-point streams) and the float64 oracle's distances, closest faces and winding numbers.

    python tests/golden/make_mesh_sdf_golden.py REFERENCE_ROOT

The oracle is checked against the reference's distances before anything is written."""
import importlib.util
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import mesh_sdf_oracle as msdf  # noqa: E402
from points2surf_b200 import mesh_io  # noqa: E402


def main(ref_root):
    spec = importlib.util.spec_from_file_location('ref_file_utils', os.path.join(ref_root, 'source', 'base', 'file_utils.py'))
    ref_file_utils = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref_file_utils)
    ds = os.path.join(ref_root, 'datasets', 'abc_minimal')
    out = {'patch_radius': np.float64((1.0 + 5) / 256), 'far_query_pts_ratio': np.float64(0.5)}   # settings.ini
    for i, f in enumerate(sorted(os.listdir(os.path.join(ds, '03_meshes')))):
        mesh_file = os.path.join(ds, '03_meshes', f)
        v, fc = mesh_io.read_ply(mesh_file)
        q = np.load(os.path.join(ds, '05_query_pts', f + '.npy'))
        d = np.load(os.path.join(ds, '05_query_dist', f + '.npy'))
        od, of, ow = msdf.mesh_signed_distance(v, fc, q)
        err = np.abs(np.abs(od) - np.abs(d)).max()
        mism = int((np.sign(od) != np.sign(d)).sum())
        print(f, 'V', len(v), 'F', len(fc), 'max | |d| - |d_ref| | %.2e' % err, 'sign mismatches', mism)
        assert err <= 1e-5 and mism == 0
        out.update({'name_%d' % i: np.array(f), 'verts_%d' % i: v.astype(np.float32), 'faces_%d' % i: fc.astype(np.int32),
                    'ref_query_pts_%d' % i: q, 'ref_query_dist_%d' % i: d,
                    'hash_%d' % i: np.int64(ref_file_utils.filename_to_hash(mesh_file)),
                    'oracle_dist_%d' % i: od, 'oracle_face_%d' % i: of.astype(np.int32), 'oracle_wind_%d' % i: ow})
    path = os.path.join(ROOT, 'tests', 'golden', 'mesh_sdf.npz')
    np.savez_compressed(path, **out)
    print('written', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main(sys.argv[1])
