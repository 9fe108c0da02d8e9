"""The ground-truth point normals of the reference's eval_dataset.py (utils.get_pts_normals, source/base/utils.py:109-164),
which the "SPSR + GT normals" baseline reconstructs from, with the point-to-mesh work on the GPU:
  device surface samples with their face ids (p2s_mesh_sample_dev) -> nearest sample of every cloud point
  (p2s_nn_distance_dev, cKDTree's semantics) -> the oriented unit normal of that sample's face.

    python -m points2surf_b200.eval_dataset DATASET_DIR

writes DATASET_DIR/06_normals/<name>.xyz.npy and 06_normals/pts/<name>.xyz from 04_pts and 03_meshes with 100 000 samples
per mesh, like eval_dataset.py:143-146.  The Screened-Poisson stages of eval_dataset.py need meshlabserver and are not
run."""
import argparse
import os
import sys

import numpy as np
import torch

from . import make_dataset
from . import mesh_io
from . import ops
from . import point_cloud
from . import sdf


def _face_normals_dev(verts, faces):
    """Unit normals [F,3] float64 of the faces, on the device (zero for zero-area faces, like make_dataset.face_normals)."""
    v = verts.double()
    f = faces.long()
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    n = torch.linalg.cross(b - a, c - a)
    norm = torch.linalg.norm(n, dim=1, keepdim=True)
    return torch.where(norm > 0, n / torch.where(norm > 0, norm, torch.ones_like(norm)), torch.zeros_like(n))


def pts_normals(pts, verts, faces, samples_per_model, seed):
    """Ground-truth normals [N,3] float64 of the points pts [N,3]: the oriented unit face normal of the nearest of
    `samples_per_model` area-weighted surface samples (ties -> lowest sample index).  Of trimesh's fix_normals only the
    global flip is applied: every face is reversed when the mesh's signed volume is negative."""
    dev = sdf._device()
    v = torch.from_numpy(np.ascontiguousarray(verts, np.float32)).to(dev)
    f = torch.from_numpy(np.ascontiguousarray(faces, np.int32)).to(dev)
    samples, face_ids = ops.mesh_sample(v, f, samples_per_model, seed, return_face_ids=True)
    oriented = torch.from_numpy(sdf._orient_outward(np.asarray(verts, np.float32), np.asarray(faces, np.int32))).to(dev)
    p = torch.from_numpy(np.ascontiguousarray(pts[:, :3], np.float32)).to(dev)
    _, sample_ids = ops.nn_distance(p, samples)
    face_for_pts = face_ids[sample_ids.long()]
    return _face_normals_dev(v, oriented[face_for_pts]).cpu().numpy()


def _get_pts_normals_single_file(pts_file_in, mesh_file_in, normals_file_out, pts_normals_file_out,
                                 samples_per_model=10000):
    """source/base/utils.py:109-131 for one shape.  04_pts may be [N,3] or [N,6] (points and scan normals); the points are
    columns 0:3.  The samples are seeded by the mesh's file name (the reference's are unseeded)."""
    pts = np.load(pts_file_in)[:, :3]
    verts, faces = mesh_io.read_mesh(mesh_file_in)
    normals = pts_normals(pts, verts, faces, samples_per_model, make_dataset.filename_to_hash(mesh_file_in))
    np.save(normals_file_out, normals)
    point_cloud.write_xyz(pts_normals_file_out, pts, normals=normals)


def get_pts_normals(base_dir, dataset_dir, dir_in_pointcloud, dir_in_meshes, dir_out_normals, samples_per_model=10000,
                    num_processes=1):
    """source/base/utils.py:134-164: for every <name>.xyz.npy in dir_in_pointcloud with the mesh <name>.ply in
    dir_in_meshes, write dir_out_normals/<name>.xyz.npy and dir_out_normals/pts/<name>.xyz, unless both exist and are
    newer than the inputs.  `num_processes` is accepted and ignored: the shapes run one after the other on the GPU."""
    dir_in_pts_abs = os.path.join(base_dir, dataset_dir, dir_in_pointcloud)
    dir_in_meshes_abs = os.path.join(base_dir, dataset_dir, dir_in_meshes)
    dir_out_normals_abs = os.path.join(base_dir, dataset_dir, dir_out_normals)
    dir_out_pts_normals_abs = os.path.join(base_dir, dataset_dir, dir_out_normals, 'pts')
    os.makedirs(dir_out_normals_abs, exist_ok=True)
    os.makedirs(dir_out_pts_normals_abs, exist_ok=True)
    pts_files = sorted(f for f in os.listdir(dir_in_pts_abs)
                       if os.path.isfile(os.path.join(dir_in_pts_abs, f)) and f[-4:] == '.npy')
    for f in pts_files:
        pts_in = os.path.join(dir_in_pts_abs, f)
        mesh_in = os.path.join(dir_in_meshes_abs, f[:-8] + '.ply')
        normals_out = os.path.join(dir_out_normals_abs, f)
        pts_normals_out = os.path.join(dir_out_pts_normals_abs, f[:-8] + '.xyz')
        if not os.path.isfile(mesh_in):
            print('WARNING: Input file are missing: {}'.format([mesh_in]))
            continue
        if sdf._call_necessary([pts_in, mesh_in], [normals_out, pts_normals_out]):
            _get_pts_normals_single_file(pts_in, mesh_in, normals_out, pts_normals_out, samples_per_model)


def main(argv=None):
    parser = argparse.ArgumentParser(description='Ground-truth point normals (06_normals) for the point clouds in '
                                                 'DATASET_DIR/04_pts from the meshes in DATASET_DIR/03_meshes.')
    parser.add_argument('dataset_dir', help='dataset directory containing 03_meshes and 04_pts')
    args = parser.parse_args(argv)
    dataset = os.path.abspath(args.dataset_dir)
    print('### Screened-Poisson reconstructions (06_poisson_rec*) need meshlabserver: skipped')
    print('### get ground truth normals for point cloud')
    get_pts_normals(base_dir=os.path.dirname(dataset), dataset_dir=os.path.basename(dataset),
                    dir_in_pointcloud='04_pts', dir_in_meshes='03_meshes', dir_out_normals='06_normals',
                    samples_per_model=100000)


if __name__ == '__main__':
    main(sys.argv[1:])
