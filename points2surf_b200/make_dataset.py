"""The query-point stage of the reference's make_dataset.py (make_dataset.py:447-538): training targets
05_query_pts / 05_query_dist (and optionally 05_query_vis) for every mesh in 03_meshes, with the signed distances
computed on the GPU.  Cleaning, BlenSor scans and dataset splits are not part of this module.

    python -m points2surf_b200.make_dataset DATASET_DIR [--num_query_pts 2000] [--far_query_pts_ratio 0.5] [--debug]

patch_radius is (1 + epsilon) / grid_resolution from DATASET_DIR/settings.ini, like make_dataset.py:760."""
import argparse
import configparser
import hashlib
import os
import sys

import numpy as np

from . import mesh_io
from . import sdf


def filename_to_hash(file_path):
    """source/base/file_utils.py:6-12: seed of a shape's query-point stream, the MD5 of the file name up to its first
    dot, modulo 2^32 - 1."""
    if not os.path.isfile(file_path):
        raise ValueError('Path does not point to a file: {}'.format(file_path))
    stem = os.path.basename(file_path).split('.')[0]
    return int(hashlib.md5(stem.encode()).hexdigest(), 16) % (2 ** 32 - 1)


def _get_and_save_query_pts(file_in_mesh, file_out_query_pts, file_out_query_dist, file_out_query_vis, num_query_pts,
                            patch_radius, far_query_pts_ratio=0.1, signed_distance_batch_size=1000, debug=False):
    """make_dataset.py:447-478 for one mesh: float32 query points and distances (NaN -> 0, Inf -> 1, clamped to [-1, 1])."""
    rng = np.random.RandomState(filename_to_hash(file_in_mesh))
    mesh = mesh_io.read_ply(file_in_mesh)
    query_pts_ms = sdf.get_query_pts_for_mesh(mesh, num_query_pts, patch_radius, far_query_pts_ratio, rng)
    np.save(file_out_query_pts, query_pts_ms.astype(np.float32))
    query_dist_ms = sdf.get_signed_distance(mesh, query_pts_ms, signed_distance_batch_size)
    query_dist_ms[np.isnan(query_dist_ms)] = 0.0
    query_dist_ms[np.isinf(query_dist_ms)] = 1.0
    query_dist_ms = np.clip(query_dist_ms, -1.0, 1.0)
    np.save(file_out_query_dist, query_dist_ms.astype(np.float32))
    if debug and file_out_query_vis is not None:
        sdf.visualize_query_points(query_pts_ms, query_dist_ms, file_out_query_vis)


def get_query_pts_dist_ms(base_dir, dataset_dir, dir_in_mesh, dir_out_query_pts_ms, dir_out_query_dist_ms,
                          dir_out_query_vis, patch_radius, num_query_pts=2000, far_query_pts_ratio=0.1,
                          signed_distance_batch_size=1000, num_processes=8, debug=False):
    """make_dataset.py:481-538: every .ply in dir_in_mesh whose outputs are missing or older than the mesh.
    `num_processes` is accepted and ignored: the shapes run one after the other on the GPU."""
    root = os.path.join(base_dir, dataset_dir)
    dir_mesh = os.path.join(root, dir_in_mesh)
    dir_pts = os.path.join(root, dir_out_query_pts_ms)
    dir_dist = os.path.join(root, dir_out_query_dist_ms)
    dir_vis = os.path.join(root, dir_out_query_vis)
    os.makedirs(dir_pts, exist_ok=True)
    os.makedirs(dir_dist, exist_ok=True)
    if debug:
        os.makedirs(dir_vis, exist_ok=True)
    print('### get query points')
    files_mesh = sorted(f for f in os.listdir(dir_mesh) if os.path.isfile(os.path.join(dir_mesh, f)) and f[-4:] == '.ply')
    for f in files_mesh:
        file_in_mesh = os.path.join(dir_mesh, f)
        file_out_query_pts = os.path.join(dir_pts, f + '.npy')
        file_out_query_dist = os.path.join(dir_dist, f + '.npy')
        file_out_query_vis = os.path.join(dir_vis, f + '.ply')
        if sdf._call_necessary([file_in_mesh], [file_out_query_pts, file_out_query_dist]):
            _get_and_save_query_pts(file_in_mesh, file_out_query_pts, file_out_query_dist, file_out_query_vis,
                                    num_query_pts, patch_radius, far_query_pts_ratio, signed_distance_batch_size, debug)


def main(argv=None):
    parser = argparse.ArgumentParser(description='Query points and ground-truth signed distances (05_query_pts, '
                                                 '05_query_dist) for the meshes in DATASET_DIR/03_meshes.')
    parser.add_argument('dataset_dir', help='dataset directory containing settings.ini and 03_meshes')
    parser.add_argument('--num_query_pts', type=int, default=2000)
    parser.add_argument('--far_query_pts_ratio', type=float, default=0.5)
    parser.add_argument('--debug', action='store_true', help='also write coloured query points to 05_query_vis')
    args = parser.parse_args(argv)
    dataset = os.path.abspath(args.dataset_dir)
    config_file = os.path.join(dataset, 'settings.ini')
    if not os.path.isfile(config_file):
        raise SystemExit('no settings.ini in %s (needs [general] grid_resolution and epsilon)' % dataset)
    config = configparser.ConfigParser()
    config.read(config_file)
    patch_radius = (1.0 + int(config['general']['epsilon'])) / int(config['general']['grid_resolution'])
    get_query_pts_dist_ms(os.path.dirname(dataset), os.path.basename(dataset), '03_meshes', '05_query_pts', '05_query_dist',
                          '05_query_vis', patch_radius, num_query_pts=args.num_query_pts,
                          far_query_pts_ratio=args.far_query_pts_ratio, debug=args.debug)


if __name__ == '__main__':
    main(sys.argv[1:])
