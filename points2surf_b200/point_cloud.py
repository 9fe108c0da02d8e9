"""Point-cloud helpers of source/base/point_cloud.py that the evaluation needs:
  get_closest_distance_batched  point_cloud.py:195-218  trimesh.proximity.closest_point in batches -> one device pass
                                                        (p2s_mesh_closest_point_dev)
  write_xyz                     point_cloud.py:63-103   the reference's text format: one 'x y z [nx ny nz] [r g b] ' line
                                                        per point, every value as str() of its NumPy scalar
"""
import numpy as np
import torch

from . import mesh_io
from . import ops
from . import sdf


def get_closest_distance_batched(query_pts, mesh, batch_size=1000, workers=0):
    """source/base/point_cloud.py:195-218 -> (closest points [Q,3] float64, distances [Q] float64, face ids [Q] int64),
    NumPy like the reference.  `mesh`: anything with .vertices / .faces, or a (vertices, faces) pair.  `batch_size` and
    `workers` are accepted and ignored: one device call covers all queries.  The mesh and the queries are rounded to
    float32 and the results are the kernel's fp32 values (rules in include/p2s_b200.h); ties go to the lowest face
    index."""
    verts, faces = sdf._mesh_arrays(mesh)
    dev = sdf._device()
    q = torch.from_numpy(np.ascontiguousarray(np.asarray(query_pts).reshape(-1, 3), dtype=np.float32)).to(dev)
    closest, dist, face = ops.mesh_closest_point(torch.from_numpy(verts).to(dev), torch.from_numpy(faces).to(dev), q)
    return (closest.cpu().numpy().astype(np.float64), dist.cpu().numpy().astype(np.float64),
            face.cpu().numpy().astype(np.int64))


def write_xyz(file_path, points, normals=None, colors=None):
    """source/base/point_cloud.py:63-103: text point cloud, values formatted exactly like the reference's."""
    mesh_io.make_dir_for_file(file_path)
    if points.shape == (3,):
        points = np.expand_dims(points, axis=0)
    if points.shape[0] == 3 and points.shape[1] != 3:
        points = points.transpose([1, 0])
    if colors is not None and colors.shape[0] == 3 and colors.shape[1] != 3:
        colors = colors.transpose([1, 0])
    if normals is not None and normals.shape[0] == 3 and normals.shape[1] != 3:
        normals = normals.transpose([1, 0])
    if points.shape[1] == 2:
        points = np.concatenate([points, np.zeros((points.shape[0], 1))], axis=1)
    with open(file_path, 'w') as fp:
        for vi, v in enumerate(points):
            line = str(v[0]) + ' ' + str(v[1]) + ' ' + str(v[2]) + ' '
            if normals is not None:
                line += str(normals[vi][0]) + ' ' + str(normals[vi][1]) + ' ' + str(normals[vi][2]) + ' '
            if colors is not None:
                line += str(colors[vi][0]) + ' ' + str(colors[vi][1]) + ' ' + str(colors[vi][2]) + ' '
            fp.write(line + '\n')
