"""Two stages of the reference's make_dataset.py for every mesh in 03_meshes, on the GPU:
  - with --scan, the input point clouds 04_pts (sample_blensor, make_dataset.py:242-380): simulated time-of-flight scans
    (csrc/scan.cu) instead of Blender / BlenSor, with the reference's scan poses and noise levels;
  - the training targets 05_query_pts / 05_query_dist (and optionally 05_query_vis) of the query-point stage
    (make_dataset.py:447-538), with the signed distances of csrc/meshsdf.cu.
Cleaning, normalisation and dataset splits are not part of this module.

    python -m points2surf_b200.make_dataset DATASET_DIR [--scan] [--num_query_pts 2000] [--far_query_pts_ratio 0.5] [--debug]

From DATASET_DIR/settings.ini: patch_radius = (1 + epsilon) / grid_resolution (make_dataset.py:760); with --scan also
num_scans_per_mesh_min/max, scanner_noise_sigma_min/max and only_for_evaluation (make_dataset.py:809-815)."""
import argparse
import configparser
import hashlib
import os
import sys

import numpy as np
import torch

from . import mesh_io
from . import ops
from . import sdf
from . import trafo


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


def get_scan_poses(file_in_mesh, num_scans_per_mesh_min, num_scans_per_mesh_max, scanner_noise_sigma_min=0.0,
                   scanner_noise_sigma_max=0.05):
    """The scan stream of make_dataset.py:303-321 for one mesh -> (noise sigma, locations [S,3], rotations [S,4] as
    [w, x, y, z] quaternions).  Scan s places the model point p at quaternion_matrix(rotations[s]) p + locations[s] in the
    scanner frame of ops.range_scan."""
    rnd = np.random.RandomState(filename_to_hash(file_in_mesh))
    num_scans = rnd.randint(num_scans_per_mesh_min, num_scans_per_mesh_max + 1)
    noise_sigma = rnd.rand() * (scanner_noise_sigma_max - scanner_noise_sigma_min) + scanner_noise_sigma_min
    locations, rotations = [], []
    for _ in range(num_scans):
        obj_location = (rnd.rand(3) * 2.0 - 1.0) * np.array([0.1, 1.0, 0.1])
        obj_location[1] += 4.0  # offset in the scanner's view direction
        locations.append(obj_location)
        rotations.append(trafo.random_quaternion(rnd.rand(3)))
    return noise_sigma, np.array(locations).reshape(-1, 3), np.array(rotations).reshape(-1, 4)


def face_normals(verts, faces):
    """Unit normals [F,3] float64 of the faces (trimesh's Trimesh.face_normals); zero for zero-area faces."""
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)
    n = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    norm = np.linalg.norm(n, axis=1, keepdims=True)
    return np.divide(n, norm, out=np.zeros_like(n), where=norm > 0)


def _scan_and_save_pts(file_in_mesh, file_out_pts, file_out_vis, file_out_hits_per_scan, noise_sigma, locations,
                       rotations, min_pts_size=0):
    """Scan one mesh and merge the scans like _pcd_files_to_pts (make_dataset.py:147-239): 04_pts float32 [N, 6] = the
    noisy points and the unit normal of the face each noise-free point lies on; 04_pts_vis text (points only) when
    N > min_pts_size; 04_hits_per_scan.  Nothing but a message when no ray hits the mesh, like the reference."""
    verts, faces = mesh_io.read_ply(file_in_mesh)
    dev = sdf._device()
    rot = np.stack([trafo.quaternion_matrix(q)[:3, :3] for q in rotations]) if len(rotations) else np.zeros((0, 3, 3))
    noisy, _, face_ids, hits_per_scan = ops.range_scan(
        torch.from_numpy(np.ascontiguousarray(verts, np.float32)).to(dev),
        torch.from_numpy(np.ascontiguousarray(faces, np.int32)).to(dev), rot, locations, noise_sigma=noise_sigma,
        seed=filename_to_hash(file_in_mesh))
    noisy, face_ids, hits_per_scan = noisy.cpu().numpy(), face_ids.cpu().numpy(), hits_per_scan.cpu().numpy()
    if len(noisy) == 0:
        print('No scanner hits for object {} in {} scans'.format(os.path.basename(file_in_mesh), len(locations)))
        return
    pts = np.concatenate([noisy, face_normals(verts, faces)[face_ids]], axis=1).astype(np.float32)
    np.save(file_out_pts, pts)
    if pts.shape[0] > min_pts_size:
        np.savetxt(file_out_vis, pts[:, :3], fmt='%.9g')
    np.savez_compressed(file_out_hits_per_scan, hits_per_scan=hits_per_scan.astype(np.int32))


def sample_blensor(base_dir, dataset_dir, blensor_bin, dir_in, dir_out_raw, dir_out, dir_out_vis, dir_out_pcd,
                   dir_out_blensor_scripts, dir_out_locations, dir_out_rotations, num_scans_per_mesh_min,
                   num_scans_per_mesh_max, num_processes, min_pts_size=0, scanner_noise_sigma_min=0.0,
                   scanner_noise_sigma_max=0.05):
    """make_dataset.py:242-380 with the BlenSor time-of-flight scans simulated on the GPU (ops.range_scan): for every
    .ply in dir_in whose outputs are missing or older than the mesh, the reference's scan poses and noise sigma
    (get_scan_poses) -> dir_out_locations/<name>.npz (locations), dir_out_rotations/<name>.npz (rotations),
    04_hits_per_scan/<name>.npz (hits_per_scan), dir_out/<name>.xyz.npy and dir_out_vis/<name>.xyz.

    `blensor_bin`, `dir_out_raw`, `dir_out_pcd`, `dir_out_blensor_scripts` and `num_processes` are accepted and
    ignored: no Blender process, script or BlenSor file (04_pts_raw, 04_pcd) is involved, and the meshes run one after
    the other on the GPU.  The point clouds are named <name>.xyz.npy, the name both training loops and the reconstruction
    read; the reference's own merge step writes <name>.ply.npy."""
    root = os.path.join(base_dir, dataset_dir)
    dir_mesh = os.path.join(root, dir_in)
    dir_pts = os.path.join(root, dir_out)
    dir_vis = os.path.join(root, dir_out_vis)
    dir_loc = os.path.join(root, dir_out_locations)
    dir_rot = os.path.join(root, dir_out_rotations)
    dir_hits = os.path.join(root, '04_hits_per_scan')
    for d in (dir_pts, dir_vis, dir_loc, dir_rot, dir_hits):
        os.makedirs(d, exist_ok=True)
    print('### scan meshes')
    files_mesh = sorted(f for f in os.listdir(dir_mesh) if os.path.isfile(os.path.join(dir_mesh, f)) and f[-4:] == '.ply')
    for f in files_mesh:
        stem = f[:-4]
        file_in_mesh = os.path.join(dir_mesh, f)
        file_pts = os.path.join(dir_pts, stem + '.xyz.npy')
        file_vis = os.path.join(dir_vis, stem + '.xyz')
        file_loc = os.path.join(dir_loc, stem + '.npz')
        file_rot = os.path.join(dir_rot, stem + '.npz')
        file_hits = os.path.join(dir_hits, stem + '.npz')
        if not sdf._call_necessary([file_in_mesh], [file_pts, file_loc, file_rot, file_hits]):
            continue
        noise_sigma, locations, rotations = get_scan_poses(file_in_mesh, num_scans_per_mesh_min, num_scans_per_mesh_max,
                                                           scanner_noise_sigma_min, scanner_noise_sigma_max)
        np.savez_compressed(file_loc, locations=locations)
        np.savez_compressed(file_rot, rotations=rotations)
        _scan_and_save_pts(file_in_mesh, file_pts, file_vis, file_hits, noise_sigma, locations, rotations, min_pts_size)


def main(argv=None):
    parser = argparse.ArgumentParser(description='Query points and ground-truth signed distances (05_query_pts, '
                                                 '05_query_dist) for the meshes in DATASET_DIR/03_meshes, and with '
                                                 '--scan first their input point clouds (04_pts).')
    parser.add_argument('dataset_dir', help='dataset directory containing settings.ini and 03_meshes')
    parser.add_argument('--num_query_pts', type=int, default=2000)
    parser.add_argument('--far_query_pts_ratio', type=float, default=0.5)
    parser.add_argument('--debug', action='store_true', help='also write coloured query points to 05_query_vis')
    parser.add_argument('--scan', action='store_true',
                        help='first scan the meshes into the input point clouds 04_pts (simulated time-of-flight scans)')
    args = parser.parse_args(argv)
    dataset = os.path.abspath(args.dataset_dir)
    config_file = os.path.join(dataset, 'settings.ini')
    if not os.path.isfile(config_file):
        raise SystemExit('no settings.ini in %s (needs [general] grid_resolution and epsilon)' % dataset)
    config = configparser.ConfigParser()
    config.read(config_file)
    general = config['general']
    patch_radius = (1.0 + int(general['epsilon'])) / int(general['grid_resolution'])
    if args.scan:
        sample_blensor(os.path.dirname(dataset), os.path.basename(dataset), None, '03_meshes', '04_pts_raw', '04_pts',
                       '04_pts_vis', '04_pcd', '04_blensor_py', '04_locations', '04_rotations',
                       int(general['num_scans_per_mesh_min']), int(general['num_scans_per_mesh_max']), 1,
                       min_pts_size=0 if int(general.get('only_for_evaluation', '0')) else 100,
                       scanner_noise_sigma_min=float(general['scanner_noise_sigma_min']),
                       scanner_noise_sigma_max=float(general['scanner_noise_sigma_max']))
    get_query_pts_dist_ms(os.path.dirname(dataset), os.path.basename(dataset), '03_meshes', '05_query_pts', '05_query_dist',
                          '05_query_vis', patch_radius, num_query_pts=args.num_query_pts,
                          far_query_pts_ratio=args.far_query_pts_ratio, debug=args.debug)


if __name__ == '__main__':
    main(sys.argv[1:])
