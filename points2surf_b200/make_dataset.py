"""The reference's make_dataset.py, with its mesh work on the GPU:
  - convert_meshes, clean_meshes (csrc/meshclean.cu), normalize_meshes: 00_base_meshes -> 01_base_meshes_ply ->
    02_meshes_cleaned -> 03_meshes;
  - with --scan, the input point clouds 04_pts (sample_blensor, make_dataset.py:242-380): simulated time-of-flight scans
    (csrc/scan.cu) instead of Blender / BlenSor, with the reference's scan poses and noise levels;
  - the training targets 05_query_pts / 05_query_dist (and optionally 05_query_vis) of the query-point stage
    (make_dataset.py:447-538), with the signed distances of csrc/meshsdf.cu;
  - clean_up_broken_inputs, make_dataset_splits and make_dataset, which runs all of it (--from_base_meshes);
  - with --gt_recon, reconstruct_gt (make_dataset.py:649-712) in model space: the grid targets 05_query_pts_grid /
    05_query_dist_grid, meshes from them through sign propagation (06_mc_gt_recon) and with the exact inside/outside sign
    of every voxel (06_mc_gt_exact_sign, csrc/inside.cu), and their Chamfer reports.

    python -m points2surf_b200.make_dataset DATASET_DIR [--scan] [--num_query_pts 2000] [--far_query_pts_ratio 0.5] [--debug]
    python -m points2surf_b200.make_dataset DATASET_DIR --from_base_meshes [--num_query_pts 2000]
    python -m points2surf_b200.make_dataset DATASET_DIR --gt_recon [--grid_resolution 256] [--epsilon 3] [--sigma 5]
                                                                 [--certainty_threshold 13] [--dataset testset.txt]

From DATASET_DIR/settings.ini: patch_radius = (1 + epsilon) / grid_resolution (make_dataset.py:760); with --scan also
num_scans_per_mesh_min/max, scanner_noise_sigma_min/max and only_for_evaluation (make_dataset.py:809-815)."""
import argparse
import configparser
import hashlib
import os
import random
import shutil
import sys

import numpy as np
import torch

from . import evaluation
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


def _signed_distance_target(mesh, query_pts_ms, signed_distance_batch_size=1000):
    """The signed-distance target of make_dataset.py:464-474: sdf.get_signed_distance with NaN -> 0, Inf -> 1, clamped to
    [-1, 1] (float64; the files store it as float32)."""
    query_dist_ms = sdf.get_signed_distance(mesh, query_pts_ms, signed_distance_batch_size)
    query_dist_ms[np.isnan(query_dist_ms)] = 0.0
    query_dist_ms[np.isinf(query_dist_ms)] = 1.0
    return np.clip(query_dist_ms, -1.0, 1.0)


def _get_and_save_query_pts(file_in_mesh, file_out_query_pts, file_out_query_dist, file_out_query_vis, num_query_pts,
                            patch_radius, far_query_pts_ratio=0.1, signed_distance_batch_size=1000, debug=False):
    """make_dataset.py:447-478 for one mesh: float32 query points and distances (NaN -> 0, Inf -> 1, clamped to [-1, 1])."""
    rng = np.random.RandomState(filename_to_hash(file_in_mesh))
    mesh = mesh_io.read_ply(file_in_mesh)
    query_pts_ms = sdf.get_query_pts_for_mesh(mesh, num_query_pts, patch_radius, far_query_pts_ratio, rng)
    np.save(file_out_query_pts, query_pts_ms.astype(np.float32))
    query_dist_ms = _signed_distance_target(mesh, query_pts_ms, signed_distance_batch_size)
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


def get_query_pts_dist_grid(base_dir, dataset_dir, dir_in_pts, dir_in_mesh, dir_out_query_pts, dir_out_query_dist,
                            grid_resolution, epsilon):
    """The grid targets that the reference's reconstruct_gt reads, in model space: for every <name>.xyz.npy in dir_in_pts
    with a dir_in_mesh/<name>.ply whose outputs are missing or older than either input,
      dir_out_query_pts/<name>.xyz.npy  float32 [Q, 3] = sdf.get_voxel_centers_grid_smaller_pc(points, grid_resolution,
                                        epsilon), the query points of the reconstruction at that resolution and epsilon;
      dir_out_query_dist/<name>.xyz.npy float32 [Q] = the mesh's signed distances there, cleaned up like 05_query_dist.
    Columns 0:3 of the point cloud are the points.  No 05_patch_ids_grid: model-space points need no patch centre."""
    root = os.path.join(base_dir, dataset_dir)
    dir_pts, dir_mesh = os.path.join(root, dir_in_pts), os.path.join(root, dir_in_mesh)
    dir_q, dir_d = os.path.join(root, dir_out_query_pts), os.path.join(root, dir_out_query_dist)
    os.makedirs(dir_q, exist_ok=True)
    os.makedirs(dir_d, exist_ok=True)
    for f in sorted(f for f in os.listdir(dir_pts) if os.path.isfile(os.path.join(dir_pts, f)) and f[-8:] == '.xyz.npy'):
        file_pts, file_mesh = os.path.join(dir_pts, f), os.path.join(dir_mesh, f[:-8] + '.ply')
        file_q, file_d = os.path.join(dir_q, f), os.path.join(dir_d, f)
        if not os.path.isfile(file_mesh) or not sdf._call_necessary([file_pts, file_mesh], [file_q, file_d]):
            continue
        query_pts_ms = sdf.get_voxel_centers_grid_smaller_pc(np.load(file_pts)[:, :3], grid_resolution, epsilon)
        np.save(file_q, query_pts_ms.astype(np.float32))
        query_dist_ms = _signed_distance_target(mesh_io.read_ply(file_mesh), query_pts_ms)
        np.save(file_d, query_dist_ms.astype(np.float32))


def reconstruct_gt(base_dir, dataset_dir, pts_dir, query_dist_dir, query_pts_dir, gt_reconstruction_dir,
                   grid_resolution, sigma, certainty_threshold, num_processes=1):
    """make_dataset.py:662-712, the reconstruction from ground-truth signed distances, on model-space grid files (the
    reference's patch-space call cannot run: it omits patch_space_to_model_space's patch radius), so the signature has no
    p_ids_grid_dir.  For every <name>.xyz.npy in query_dist_dir whose outputs are missing or older than an input:
    sdf.implicit_surface_to_mesh -> gt_reconstruction_dir/<name>.ply and gt_reconstruction_dir/vol/<name>.xyz.off.
    `num_processes` is accepted and ignored."""
    root = os.path.join(base_dir, dataset_dir)
    dir_mesh = os.path.join(root, gt_reconstruction_dir)
    dir_vol = os.path.join(dir_mesh, 'vol')
    os.makedirs(dir_vol, exist_ok=True)
    dir_d = os.path.join(root, query_dist_dir)
    for f in sorted(f for f in os.listdir(dir_d) if os.path.isfile(os.path.join(dir_d, f)) and f[-8:] == '.xyz.npy'):
        file_pts, file_d, file_q = (os.path.join(root, d, f) for d in (pts_dir, query_dist_dir, query_pts_dir))
        file_vol, file_rec = os.path.join(dir_vol, f[:-4] + '.off'), os.path.join(dir_mesh, f[:-8] + '.ply')
        if sdf._call_necessary([file_pts, file_d, file_q], [file_rec, file_vol]):
            sdf.implicit_surface_to_mesh_file(file_d, file_q, file_vol, file_rec, grid_resolution, sigma,
                                              certainty_threshold)


def mesh_is_closed(faces):
    """True iff every edge is shared by exactly two faces that run it in opposite directions (the condition under which
    the parity of ops.mesh_inside_grid is an inside/outside sign)."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    if len(f) == 0:
        return False
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    if (e[:, 0] == e[:, 1]).any():
        return False
    n = int(e.max()) + 1
    fwd, cnt = np.unique(e[:, 0] * n + e[:, 1], return_counts=True)
    # each directed edge once (not in two faces the same way, not in three or more faces) and its reverse present
    return bool((cnt == 1).all() and np.isin(e[:, 1] * n + e[:, 0], fwd).all())


def exact_sign_volume(inside, lin_idx, dist):
    """The volume [res, res, res] fp32 of the exact-sign reconstruction: the signed distances dist at the voxels lin_idx,
    clamped to [-1, 1] like ops.sdf_to_volume, and +1 inside / -1 outside (inside [res, res, res] bool) everywhere else."""
    vol = torch.where(inside, 1.0, -1.0)
    vol.view(-1)[lin_idx.long()] = dist.clamp(-1.0, 1.0)
    return vol


def reconstruct_gt_exact_sign(base_dir, dataset_dir, mesh_dir, query_dist_dir, query_pts_dir, out_dir, grid_resolution,
                              sigma, certainty_threshold):
    """Marching cubes on exact_sign_volume for every <name>.xyz.npy in query_dist_dir with a closed mesh_dir/<name>.ply
    whose output out_dir/<name>.ply is missing or older than an input; the inside flags come from ops.mesh_inside_grid.
    Prints per shape Q and the number of voxels whose sign after sign propagation (ops.sdf_to_volume on the same distances
    with sigma and certainty_threshold; a voxel left at 0 counts as outside) differs from the exact sign.  A mesh that is
    not closed gets one line and no output."""
    root = os.path.join(base_dir, dataset_dir)
    dir_out = os.path.join(root, out_dir)
    os.makedirs(dir_out, exist_ok=True)
    dir_d = os.path.join(root, query_dist_dir)
    dev = sdf._device()
    for f in sorted(f for f in os.listdir(dir_d) if os.path.isfile(os.path.join(dir_d, f)) and f[-8:] == '.xyz.npy'):
        name = f[:-8]
        file_mesh = os.path.join(root, mesh_dir, name + '.ply')
        file_d, file_q = os.path.join(dir_d, f), os.path.join(root, query_pts_dir, f)
        file_rec = os.path.join(dir_out, name + '.ply')
        if not os.path.isfile(file_mesh) or not sdf._call_necessary([file_mesh, file_d, file_q], [file_rec]):
            continue
        verts, faces = mesh_io.read_ply(file_mesh)
        if not mesh_is_closed(faces):
            print('{}: mesh is not closed (an edge not shared by exactly two opposite faces), no exact-sign '
                  'reconstruction'.format(name))
            continue
        inside = ops.mesh_inside_grid(torch.from_numpy(np.ascontiguousarray(verts, np.float32)).to(dev),
                                      torch.from_numpy(np.ascontiguousarray(faces, np.int32)).to(dev), grid_resolution)
        lin = sdf.volume_lin_idx(np.load(file_q), grid_resolution)
        dist = torch.from_numpy(np.ascontiguousarray(np.load(file_d), np.float32)).to(dev)
        vol = exact_sign_volume(inside, lin, dist)
        prop, _ = ops.sdf_to_volume(lin, dist, grid_resolution, sigma, certainty_threshold)
        print('{}: {} grid queries, {} voxels with a propagated sign other than the exact sign'.format(
            name, len(dist), int(((prop > 0.0) != (vol > 0.0)).sum())))
        v, fc = ops.marching_cubes(vol, 0.0)
        if len(fc) == 0:
            print('Warning: marching cubes gives no result for {}'.format(name))
            continue
        mesh_io.write_ply(file_rec, v.cpu().numpy(), fc.cpu().numpy())


def gt_recon(dataset, grid_resolution=256, epsilon=3, sigma=5, certainty_threshold=13, dataset_file='testset.txt'):
    """Where the reconstruction error comes from: 05_query_pts_grid / 05_query_dist_grid, then meshes from the
    ground-truth distances through sign propagation (06_mc_gt_recon) and with every voxel's exact sign
    (06_mc_gt_exact_sign), then their Hausdorff / Chamfer reports against 03_meshes for the shapes in dataset_file
    (comp_mc_gt_recon.csv, comp_mc_gt_exact_sign.csv)."""
    base_dir, dataset_dir = os.path.dirname(dataset), os.path.basename(dataset)
    print('### grid query points, signed distances')
    get_query_pts_dist_grid(base_dir, dataset_dir, '04_pts', '03_meshes', '05_query_pts_grid', '05_query_dist_grid',
                            grid_resolution, epsilon)
    print('### reconstruct from ground-truth signed distances')
    reconstruct_gt(base_dir, dataset_dir, '04_pts', '05_query_dist_grid', '05_query_pts_grid', '06_mc_gt_recon',
                   grid_resolution, sigma, certainty_threshold)
    print('### reconstruct from ground-truth signed distances with exact signs')
    reconstruct_gt_exact_sign(base_dir, dataset_dir, '03_meshes', '05_query_dist_grid', '05_query_pts_grid',
                              '06_mc_gt_exact_sign', grid_resolution, sigma, certainty_threshold)
    for rec_dir, report in (('06_mc_gt_recon', 'comp_mc_gt_recon.csv'), ('06_mc_gt_exact_sign', 'comp_mc_gt_exact_sign.csv')):
        rec_dir_abs = os.path.join(dataset, rec_dir)
        if not any(f[-4:] == '.ply' for f in os.listdir(rec_dir_abs)):
            print('### {}: no meshes to compare'.format(rec_dir))
            continue
        print('### {} - hausdorff distance'.format(rec_dir))
        evaluation.mesh_comparison(new_meshes_dir_abs=rec_dir_abs, ref_meshes_dir_abs=os.path.join(dataset, '03_meshes'),
                                   num_processes=1, report_name=os.path.join(dataset, report), samples_per_model=10000,
                                   dataset_file_abs=os.path.join(dataset, dataset_file))


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


def convert_meshes(in_dir_abs, out_dir_abs, target_file_type: str, num_processes=8):
    """make_dataset.py:21-68: every .off / .ply / .obj / .stl under in_dir_abs (recursively) whose output is missing or
    older -> out_dir_abs/<name><target_file_type> as binary PLY (mesh_io.read_mesh; polygons fan-triangulated).  The
    faces are written as read, without welding: an STL stays a triangle soup until the clean stage welds it.  Files
    that fail to parse are reported and skipped, like the reference's except branches.  `num_processes` is accepted
    and ignored."""
    if target_file_type != '.ply':
        raise ValueError('only .ply output is supported, got %s' % target_file_type)
    os.makedirs(out_dir_abs, exist_ok=True)
    mesh_files = []
    for root, dirs, files in os.walk(in_dir_abs, topdown=True):
        for name in files:
            mesh_files.append(os.path.join(root, name))
    mesh_files = [f for f in mesh_files if f[-4:] in ('.off', '.ply', '.obj', '.stl')]
    for f in mesh_files:
        file_out = os.path.join(out_dir_abs, os.path.basename(f)[:-4] + target_file_type)
        if not sdf._call_necessary([f], [file_out]):
            continue
        try:
            verts, faces = mesh_io.read_mesh(f)
        except (AttributeError, IndexError, ValueError, NameError, UnicodeDecodeError, AssertionError) as e:
            print(e)
            continue
        mesh_io.write_ply(file_out, verts, faces)


def _accept_cleaned(report, num_faces, num_max_faces=None, enforce_solid=True):
    """The decisions of _clean_mesh (make_dataset.py:395-413) on a p2s_mesh_clean report, in the reference's order:
    with enforce_solid reject if not watertight, if the winding is still inconsistent, or unless is_volume (watertight,
    consistent, finite, volume > 0); then write only if num_faces < num_max_faces."""
    if enforce_solid and not report['watertight']:
        return False
    if enforce_solid and not report['winding_consistent']:
        return False
    if enforce_solid and not (report['watertight'] and report['winding_consistent'] and np.isfinite(report['volume'])
                              and report['volume'] > 0.0):
        return False
    return num_max_faces is None or num_faces < num_max_faces


def _clean_mesh(file_in, file_out, num_max_faces=None, enforce_solid=True):
    """make_dataset.py:383-413: repair the mesh on the GPU (ops.mesh_clean), then write it as binary PLY if
    _accept_cleaned accepts the report."""
    verts, faces = mesh_io.read_mesh(file_in)
    dev = sdf._device()
    v, f, report = ops.mesh_clean(torch.from_numpy(np.ascontiguousarray(verts, np.float32)).to(dev),
                                  torch.from_numpy(np.ascontiguousarray(faces, np.int32)).to(dev))
    if _accept_cleaned(report, len(f), num_max_faces, enforce_solid):
        mesh_io.write_ply(file_out, v.cpu().numpy(), f.cpu().numpy())


def clean_meshes(base_dir, dataset_dir, dir_in_meshes, dir_out, num_processes, num_max_faces=None, enforce_solid=True):
    """make_dataset.py:416-444: _clean_mesh for every file in dir_in_meshes whose output is missing or older.
    `num_processes` is accepted and ignored."""
    dir_in_abs = os.path.join(base_dir, dataset_dir, dir_in_meshes)
    dir_out_abs = os.path.join(base_dir, dataset_dir, dir_out)
    os.makedirs(dir_out_abs, exist_ok=True)
    for f in [f for f in os.listdir(dir_in_abs) if os.path.isfile(os.path.join(dir_in_abs, f))]:
        file_in, file_out = os.path.join(dir_in_abs, f), os.path.join(dir_out_abs, f)
        if sdf._call_necessary([file_in], [file_out]):
            _clean_mesh(file_in, file_out, num_max_faces, enforce_solid)


def normalized_vertices(verts):
    """make_dataset.py:71-88 on the vertices: None when an extent is 0, else float32((v + t) s) with
    t = -(min + max) / 2 and s = 1 / max extent, in float64 -- what trimesh's two apply_transform calls compute."""
    v = np.asarray(verts, np.float64)
    if len(v) == 0:
        return None
    lo, hi = v.min(0), v.max(0)
    ext = hi - lo
    if ext.min() == 0.0:
        return None
    t = -((lo + hi) * 0.5)
    s = 1.0 / ext.max()
    return ((v + t) * s).astype(np.float32)


def _normalize_mesh(file_in, file_out):
    """make_dataset.py:71-88: translate to the origin and scale to the unit cube; nothing is written when the mesh has
    zero extent along an axis."""
    verts, faces = mesh_io.read_ply(file_in)
    v = normalized_vertices(verts if verts is not None else np.zeros((0, 3)))
    if v is not None:
        mesh_io.write_ply(file_out, v, faces)


def normalize_meshes(base_dir, in_dir, out_dir, dataset_dir, num_processes=1):
    """make_dataset.py:91-121.  `num_processes` is accepted and ignored."""
    in_dir_abs = os.path.join(base_dir, dataset_dir, in_dir)
    out_dir_abs = os.path.join(base_dir, dataset_dir, out_dir)
    os.makedirs(out_dir_abs, exist_ok=True)
    for f in [f for f in os.listdir(in_dir_abs) if os.path.isfile(os.path.join(in_dir_abs, f))]:
        file_in, file_out = os.path.join(in_dir_abs, f), os.path.join(out_dir_abs, f)
        if sdf._call_necessary([file_in], [file_out]):
            _normalize_mesh(file_in, file_out)


def make_dataset_splits(base_dir, dataset_dir, final_out_dir, seed=42, only_test_set=False, testset_ratio=0.1):
    """make_dataset.py:541-577, restated exactly: trainset.txt, testset.txt and valset.txt (= the test set) from the .npy
    files of final_out_dir in os.listdir order, the test set drawn by random.Random(seed).sample."""
    rnd = random.Random(seed)
    final_out_dir_abs = os.path.join(base_dir, dataset_dir, final_out_dir)
    final_output_files = [f for f in os.listdir(final_out_dir_abs)
                          if os.path.isfile(os.path.join(final_out_dir_abs, f)) and f[-4:] == '.npy']
    files_dataset = [f[:-8] for f in final_output_files]
    if len(files_dataset) == 0:
        raise ValueError('Dataset is empty! {}'.format(final_out_dir_abs))
    if only_test_set:
        files_test = files_dataset
    else:
        files_test = rnd.sample(files_dataset, max(3, min(int(testset_ratio * len(files_dataset)), 100)))
    files_train = list(set(files_dataset).difference(set(files_test)))
    files_test.sort()
    files_train.sort()
    file_train_set = os.path.join(base_dir, dataset_dir, 'trainset.txt')
    file_test_set = os.path.join(base_dir, dataset_dir, 'testset.txt')
    file_val_set = os.path.join(base_dir, dataset_dir, 'valset.txt')
    mesh_io.make_dir_for_file(file_test_set)
    with open(file_test_set, 'w') as text_file:
        text_file.write('\n'.join(files_test))
    if not only_test_set:
        with open(file_train_set, 'w') as text_file:
            text_file.write('\n'.join(files_train))
    with open(file_val_set, 'w') as text_file:
        text_file.write('\n'.join(files_test))   # the test set doubles as the validation set


def clean_up_broken_inputs(base_dir, dataset_dir, final_out_dir, final_out_extension, clean_up_dirs,
                           broken_dir='broken'):
    """make_dataset.py:580-617, restated exactly: move every file of clean_up_dirs whose stem (the name up to its first
    '.') has no file in final_out_dir (with final_out_extension, None = any) to broken_dir/<dir>/."""
    final_out_dir_abs = os.path.join(base_dir, dataset_dir, final_out_dir)
    final_output_files = [f for f in os.listdir(final_out_dir_abs)
                          if os.path.isfile(os.path.join(final_out_dir_abs, f)) and
                          (final_out_extension is None or f[-len(final_out_extension):] == final_out_extension)]
    if len(final_output_files) == 0:
        print('Warning: Output dir "{}" is empty'.format(final_out_dir_abs))
        return
    final_output_file_stems = set(f.split('.', 1)[0] for f in final_output_files)
    for clean_up_dir in clean_up_dirs:
        dir_abs = os.path.join(base_dir, dataset_dir, clean_up_dir)
        if not os.path.isdir(dir_abs):
            continue
        dir_files = [f for f in os.listdir(dir_abs) if os.path.isfile(os.path.join(dir_abs, f))]
        dir_files_without_final_output = [f for f in dir_files if f.split('.', 1)[0] not in final_output_file_stems]
        broken_dir_abs = os.path.join(base_dir, dataset_dir, broken_dir, clean_up_dir)
        for f in dir_files_without_final_output:
            os.makedirs(broken_dir_abs, exist_ok=True)
            shutil.move(os.path.join(dir_abs, f), os.path.join(broken_dir_abs, f))


DIRS_TO_CLEAN = ['00_base_meshes', '01_base_meshes_ply', '02_meshes_cleaned', '03_meshes',
                 '04_pts', '04_pts_raw', '04_pts_vis', '04_blensor_py', '04_locations', '04_rotations',
                 '05_patch_dists', '05_patch_ids', '05_query_dist', '05_query_pts',
                 '05_patch_ids_grid', '05_query_pts_grid', '05_query_dist_grid',
                 '06_poisson_rec', '06_mc_gt_recon', '06_poisson_rec_gt_normals',
                 '06_normals', '06_normals/pts', '06_dist_from_p_normals']


def make_dataset(dataset_name: str, blensor_bin: str, base_dir: str, num_processes=7, seed=42,
                 num_query_points_per_shape=2000):
    """make_dataset.py:731-850: 00_base_meshes -> 01_base_meshes_ply -> 02_meshes_cleaned -> 03_meshes -> 04_pts ->
    05_query_pts / 05_query_dist -> trainset / testset / valset.txt, with the reference's stage order, settings,
    clean-ups and splits.  `blensor_bin` and `num_processes` are accepted and ignored (the scans are simulated on the
    GPU, and the shapes run one after the other)."""
    dataset_dir = dataset_name
    config_file = os.path.join(base_dir, dataset_dir, 'settings.ini')
    if not os.path.isfile(config_file):
        raise ValueError('no settings.ini in %s' % os.path.join(base_dir, dataset_dir))
    config = configparser.ConfigParser()
    config.read(config_file)
    print('Processing dataset: ' + config_file)
    general = config['general']
    only_for_evaluation = bool(int(general['only_for_evaluation']))
    patch_radius = (1.0 + int(general['epsilon'])) / int(general['grid_resolution'])

    def clean_up(final_out_dir, ext):
        clean_up_broken_inputs(base_dir, dataset_dir, final_out_dir, ext, DIRS_TO_CLEAN, 'broken')

    clean_up('00_base_meshes', None)
    print('### convert base meshes to ply')
    convert_meshes(os.path.join(base_dir, dataset_dir, '00_base_meshes'),
                   os.path.join(base_dir, dataset_dir, '01_base_meshes_ply'), '.ply', num_processes)
    clean_up('01_base_meshes_ply', '.ply')
    print('### clean mesh')
    clean_meshes(base_dir, dataset_dir, '01_base_meshes_ply', '02_meshes_cleaned', num_processes,
                 num_max_faces=None if only_for_evaluation else 50000, enforce_solid=not only_for_evaluation)
    clean_up('02_meshes_cleaned', '.ply')
    print('### scale and translate mesh')
    normalize_meshes(base_dir, '02_meshes_cleaned', '03_meshes', dataset_dir, num_processes)
    print('### sample with Blensor')
    sample_blensor(base_dir, dataset_dir, blensor_bin, '03_meshes', '04_pts_raw', '04_pts', '04_pts_vis', '04_pcd',
                   '04_blensor_py', '04_locations', '04_rotations', int(general['num_scans_per_mesh_min']),
                   int(general['num_scans_per_mesh_max']), num_processes,
                   min_pts_size=0 if only_for_evaluation else 100,
                   scanner_noise_sigma_min=float(general['scanner_noise_sigma_min']),
                   scanner_noise_sigma_max=float(general['scanner_noise_sigma_max']))
    clean_up('04_pts', '.xyz.npy')
    if not only_for_evaluation:
        print('### make query points, calculate signed distances')
        get_query_pts_dist_ms(base_dir, dataset_dir, '03_meshes', '05_query_pts', '05_query_dist', '05_query_vis',
                              patch_radius, num_query_pts=num_query_points_per_shape, far_query_pts_ratio=0.5,
                              signed_distance_batch_size=500, num_processes=num_processes, debug=True)
        print('### statistics and clean up')
        clean_up('05_query_dist', '.npy')
    make_dataset_splits(base_dir, dataset_dir, '04_pts' if only_for_evaluation else '05_query_pts', seed=seed,
                        only_test_set=only_for_evaluation, testset_ratio=0.1)


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
    parser.add_argument('--from_base_meshes', action='store_true',
                        help='run the whole make_dataset from DATASET_DIR/00_base_meshes (convert, clean, normalise, '
                             'scan, query points, splits); --scan, --debug and --far_query_pts_ratio do not apply')
    parser.add_argument('--gt_recon', action='store_true',
                        help='instead of the query stage, reconstruct from ground-truth signed distances on the '
                             'reconstruction grid of 04_pts: 05_query_pts_grid, 05_query_dist_grid, 06_mc_gt_recon (sign '
                             'propagation), 06_mc_gt_exact_sign (exact signs, closed meshes only) and their reports '
                             'comp_mc_gt_recon.csv, comp_mc_gt_exact_sign.csv')
    parser.add_argument('--grid_resolution', type=int, default=256, help='--gt_recon: the reconstruction grid resolution')
    parser.add_argument('--epsilon', type=int, default=3,
                        help='--gt_recon: voxels around the points that get a query (not settings.ini\'s epsilon)')
    parser.add_argument('--sigma', type=int, default=5, help='--gt_recon: sign propagation window')
    parser.add_argument('--certainty_threshold', type=float, default=13, help='--gt_recon: sign propagation threshold')
    parser.add_argument('--dataset', default='testset.txt', help='--gt_recon: the shapes to compare with 03_meshes')
    args = parser.parse_args(argv)
    dataset = os.path.abspath(args.dataset_dir)
    if args.gt_recon:
        gt_recon(dataset, args.grid_resolution, args.epsilon, args.sigma, args.certainty_threshold, args.dataset)
        return
    if args.from_base_meshes:
        make_dataset(os.path.basename(dataset), None, os.path.dirname(dataset),
                     num_query_points_per_shape=args.num_query_pts)
        return
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
