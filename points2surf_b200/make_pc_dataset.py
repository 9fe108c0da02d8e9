"""The reference's make_pc_dataset.py: turn bare point clouds into a dataset the evaluation stages can use.

    python -m points2surf_b200.make_pc_dataset DATASET_DIR [--target_num_points 50000]

reads DATASET_DIR/00_base_pc/*.{off,ply,obj,stl,xyz} (the vertices of a mesh file, faces ignored; .xyz is plain text
x y z [...]), moves every cloud into the unit cube, sub-samples it to at most `target_num_points` points and writes
04_pts/<name>.xyz.npy (float32 [N,3]), 04_pts_vis/<name>.xyz, testset.txt and valset.txt (no trainset.txt: such a dataset
is for evaluation only).  This is host code: it produces the mesh-less 04_pts that eval_dataset --spsr_estimated_normals
and full_eval reconstruct from.

Deviations from the reference: the sub-sample is seeded by the file name (RandomState(filename_to_hash(file)), the
reference's is unseeded); a cloud with a zero extent is skipped with a warning (the reference crashes on it); .xyz text is
accepted in addition."""
import argparse
import os
import sys

import numpy as np

from . import make_dataset
from . import mesh_io
from . import point_cloud
from . import sdf

ALLOWED_TYPES = ['.off', '.ply', '.obj', '.stl', '.xyz']


def _to_unit_cube(vertices):
    """make_pc_dataset.py:20-36 on the vertices [N,3]: centre of the bounding box to the origin, longest extent to 1.
    -> float64 [N,3], or None when an extent is zero."""
    v = np.asarray(vertices, np.float64)[:, :3]
    lo, hi = v.min(axis=0), v.max(axis=0)
    extents = hi - lo
    if extents.min() == 0.0:
        return None
    return (v - (lo + hi) * 0.5) * (1.0 / extents.max())


def _read_points(in_pc):
    if in_pc[-4:].lower() == '.xyz':
        return np.loadtxt(in_pc, dtype=np.float64, ndmin=2)[:, :3]
    return mesh_io.read_mesh(in_pc)[0]


def _convert_point_cloud(in_pc, out_pc_xyz, out_pc_npy, target_num_points=150000):
    """make_pc_dataset.py:39-67 for one file."""
    vertices = _read_points(in_pc)
    points = _to_unit_cube(vertices) if vertices is not None and len(vertices) else None
    if points is None:
        print('WARNING: {} has no points or a zero extent: skipped'.format(in_pc))
        return
    points = points.astype(np.float32)
    if target_num_points is not None and 0 < target_num_points < points.shape[0]:
        rng = np.random.RandomState(make_dataset.filename_to_hash(in_pc))
        points = points[rng.choice(points.shape[0], target_num_points, replace=False)]
    mesh_io.make_dir_for_file(out_pc_npy)
    mesh_io.make_dir_for_file(out_pc_xyz)
    np.save(out_pc_npy, points)
    point_cloud.write_xyz(out_pc_xyz, points)


def convert_point_clouds(in_dir_abs, out_dir_abs, out_dir_npy_abs, target_file_type: str,
                         target_num_points=150000, num_processes=8):
    """make_pc_dataset.py:70-101: every cloud under in_dir_abs -> out_dir_abs/<name><type> and
    out_dir_npy_abs/<name><type>.npy, unless both are newer than the input.  `num_processes` is accepted and ignored."""
    os.makedirs(out_dir_abs, exist_ok=True)
    files = sorted(os.path.join(root, name) for root, _, names in os.walk(in_dir_abs, topdown=True) for name in names)
    for f in files:
        if f[-4:].lower() not in ALLOWED_TYPES:
            continue
        base = os.path.basename(f)[:-4]
        file_out = os.path.join(out_dir_abs, base + target_file_type)
        file_out_npy = os.path.join(out_dir_npy_abs, base + target_file_type + '.npy')
        if sdf._call_necessary([f], [file_out, file_out_npy]):
            _convert_point_cloud(f, file_out, file_out_npy, target_num_points)


def main(argv=None):
    parser = argparse.ArgumentParser(description='Make an evaluation-only dataset (04_pts, 04_pts_vis, testset.txt, '
                                                 'valset.txt) from the point clouds in DATASET_DIR/00_base_pc.')
    parser.add_argument('dataset_dir', help='dataset directory containing 00_base_pc')
    parser.add_argument('--target_num_points', type=int, default=50000,
                        help='sub-sample larger clouds to this many points (0: keep all)')
    args = parser.parse_args(argv)
    dataset = os.path.abspath(args.dataset_dir)
    base_dir, dataset_dir = os.path.dirname(dataset), os.path.basename(dataset)
    print('Processing dataset: ' + dataset)
    print('### convert base point clouds to xyz')
    convert_point_clouds(in_dir_abs=os.path.join(dataset, '00_base_pc'), out_dir_abs=os.path.join(dataset, '04_pts_vis'),
                         out_dir_npy_abs=os.path.join(dataset, '04_pts'), target_file_type='.xyz',
                         target_num_points=args.target_num_points)
    make_dataset.make_dataset_splits(base_dir=base_dir, dataset_dir=dataset_dir, final_out_dir='04_pts', seed=42,
                                     only_test_set=True, testset_ratio=0.1)


if __name__ == '__main__':
    main(sys.argv[1:])
