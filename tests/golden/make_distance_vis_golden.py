"""Write tests/golden/distance_vis.npz: what the reference's own distance_vis.get_normalization_target,
distance_vis.visualize_mesh_with_distances (the _stats.txt text) and point_cloud.write_xyz produce on seeded inputs.

    python tests/golden/make_distance_vis_golden.py REFERENCE_ROOT

The unmodified functions run through oracle/ref_shims.py; trimesh.Trimesh is replaced by a stand-in whose export() does
nothing, so visualize_mesh_with_distances writes only its statistics file.  The inputs are stored next to the outputs.
tests/test_closest_point_host.py runs this repository's mirrors on the same inputs."""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
CUTS = (0.9, 0.5, 0.0, 0.999, 1.0, None)


class _Trimesh:
    vertices = faces = None

    def __init__(self, *a, **k):
        pass

    def export(self, *a, **k):
        pass


def main(ref_root):
    sys.path.insert(0, ROOT)
    from oracle import ref_shims
    ref_shims.REFERENCE_ROOT = ref_root
    ref_shims.install()
    for m in [m for m in sys.modules if m == 'source' or m.startswith('source.')]:
        del sys.modules[m]          # this repository's source/ shim package must not shadow the reference's
    sys.path.remove(ROOT)
    sys.path.insert(0, ref_root)
    sys.modules['trimesh'].Trimesh = _Trimesh
    from source.figure import distance_vis as ref_dv
    from source.base import point_cloud as ref_pc
    assert os.path.abspath(ref_dv.__file__).startswith(os.path.abspath(ref_root))
    rng = np.random.RandomState(1234)
    out = {}
    # distances as the mirror returns them: fp32 values widened to float64, one list of three reconstructions
    dists = [rng.exponential(0.01, n).astype(np.float32).astype(np.float64) for n in (7, 100, 1001)]
    for i, d in enumerate(dists):
        out['dist_%d' % i] = d
    for k, cut in enumerate(CUTS):
        out['target_%d' % k] = np.float64(ref_dv.get_normalization_target(dists, cut_percentil=cut))
        out['target_single_%d' % k] = np.float64(ref_dv.get_normalization_target(dists[1:2], cut_percentil=cut))
    with tempfile.TemporaryDirectory() as tmp:
        for i, d in enumerate(dists):
            f = os.path.join(tmp, 'rec%d.ply' % i)
            ref_dv.visualize_mesh_with_distances(f, _Trimesh(), d, out['target_0'], cut_percentil=0.9)
            out['stats_%d' % i] = np.array(open(f + '_stats.txt').read())
        pts32 = (rng.rand(50, 3) * 2 - 1).astype(np.float32)
        nrm64 = rng.normal(size=(50, 3))
        nrm64 /= np.linalg.norm(nrm64, axis=1, keepdims=True)
        pts64 = rng.rand(5, 3) * 1e-3
        pts2d = rng.rand(4, 2).astype(np.float32)
        ptsT = rng.rand(3, 6).astype(np.float32)
        out.update(xyz_pts32=pts32, xyz_nrm64=nrm64, xyz_pts64=pts64, xyz_pts2d=pts2d, xyz_ptsT=ptsT)
        cases = {'pts32_normals': (pts32, nrm64), 'pts32': (pts32, None), 'pts64_normals': (pts64, nrm64[:5]),
                 'pts2d': (pts2d, None), 'ptsT': (ptsT, None)}
        for name, (p, n) in cases.items():
            f = os.path.join(tmp, name + '.xyz')
            ref_pc.write_xyz(f, p, normals=n)
            out['xyz_text_' + name] = np.array(open(f).read())
    path = os.path.join(ROOT, 'tests', 'golden', 'distance_vis.npz')
    np.savez_compressed(path, **out)
    print('written', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main(sys.argv[1])
