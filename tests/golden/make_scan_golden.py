"""Write tests/golden/scan.npz: the scan poses that the reference's own make_dataset.sample_blensor draws for the three
abc_minimal meshes, and statistics of the point clouds its BlenSor scans produced (04_pts).

    python tests/golden/make_scan_golden.py REFERENCE_ROOT

The unmodified sample_blensor runs on a temporary copy of the meshes through oracle/ref_shims.py, with trimesh stubbed
and trimesh.transformations given the restated quaternion helpers of points2surf_b200/trafo.py.  The process pool is
intercepted, so Blender and the pcd merge never run.  Recorded per mesh: the number of scans, the noise sigma (from
the generated Blender script), the locations and rotations (from the 04_locations / 04_rotations files it writes), the
number of points in the reference's 04_pts cloud and quantiles of their distance to the mesh (float64 oracle on a
seeded sample of 10 000 points)."""
import ast
import os
import shutil
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import mesh_sdf_oracle as msdf  # noqa: E402
from oracle import ref_shims  # noqa: E402
from points2surf_b200 import mesh_io, trafo  # noqa: E402

QUANTILES = np.array([0.1, 0.25, 0.5, 0.75, 0.9])


def main(ref_root):
    ref_shims.REFERENCE_ROOT = ref_root
    ref_shims.install()
    tt = sys.modules['trimesh'].transformations
    tt.random_quaternion = trafo.random_quaternion
    tt.quaternion_matrix = trafo.quaternion_matrix
    tt.quaternion_conjugate = trafo.quaternion_conjugate
    for m in [m for m in sys.modules if m == 'source' or m.startswith('source.')]:
        del sys.modules[m]          # this repository's source/ shim package must not shadow the reference's
    sys.path.remove(ROOT)
    sys.path.insert(0, ref_root)
    import make_dataset as ref_md
    from source.base import utils_mp
    assert os.path.dirname(os.path.abspath(ref_md.__file__)) == os.path.abspath(ref_root)

    pools = []
    utils_mp.start_process_pool = lambda fn, params, num_processes, timeout=None: pools.append((fn, list(params)))
    ds = os.path.join(ref_root, 'datasets', 'abc_minimal')
    out = {'quantiles': QUANTILES}
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        shutil.copytree(os.path.join(ds, '03_meshes'), os.path.join(tmp, 'abc', '03_meshes'))
        os.chdir(ref_root)          # sample_blensor reads blensor_script_template.py from the working directory
        try:
            ref_md.sample_blensor(base_dir=tmp, dataset_dir='abc', blensor_bin='blender', dir_in='03_meshes',
                                  dir_out_raw='04_pts_raw', dir_out='04_pts', dir_out_vis='04_pts_vis',
                                  dir_out_pcd='04_pcd', dir_out_blensor_scripts='04_blensor_py',
                                  dir_out_locations='04_locations', dir_out_rotations='04_rotations',
                                  num_scans_per_mesh_min=5, num_scans_per_mesh_max=30, num_processes=1,
                                  min_pts_size=100, scanner_noise_sigma_min=0.0, scanner_noise_sigma_max=0.05)
        finally:
            os.chdir(cwd)
        assert pools[0][1] and not pools[1][1], 'expected Blender calls and no pcd merge'
        for i, f in enumerate(sorted(os.listdir(os.path.join(ds, '03_meshes')))):
            stem = f[:-4]
            loc = np.load(os.path.join(tmp, 'abc', '04_locations', stem + '.npz'))['locations']
            rot = np.load(os.path.join(tmp, 'abc', '04_rotations', stem + '.npz'))['rotations']
            script = open(os.path.join(tmp, 'abc', '04_blensor_py', stem + '.py')).read()
            line = [ln for ln in script.split('\n') if ln.startswith('scan_sigmas = ')][0]
            sigmas = ast.literal_eval(line[len('scan_sigmas = '):])
            assert len(set(sigmas)) == 1 and len(sigmas) == len(loc) == len(rot)
            v, fc = mesh_io.read_ply(os.path.join(ds, '03_meshes', f))
            pts = np.load(os.path.join(ds, '04_pts', stem + '.xyz.npy'))
            sample = pts[np.random.RandomState(i).choice(len(pts), 10000, replace=False), :3]
            d = np.abs(msdf.mesh_signed_distance(v, fc, sample)[0])
            q = np.quantile(d, QUANTILES)
            print(stem, 'faces', len(fc), 'scans', len(loc), 'sigma %.5f' % sigmas[0], 'ref points', len(pts),
                  'dist quantiles', np.round(q, 5))
            out.update({'name_%d' % i: np.array(stem), 'num_scans_%d' % i: np.int64(len(loc)),
                        'sigma_%d' % i: np.float64(sigmas[0]), 'locations_%d' % i: loc, 'rotations_%d' % i: rot,
                        'ref_num_pts_%d' % i: np.int64(len(pts)), 'ref_dist_quantiles_%d' % i: q})
    path = os.path.join(ROOT, 'tests', 'golden', 'scan.npz')
    np.savez_compressed(path, **out)
    print('written', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main(sys.argv[1])
