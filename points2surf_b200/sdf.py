"""Drop-in for the hot-path functions of source/sdf.py, on the CUDA kernels."""
import os
import time

import numpy as np
import torch

from . import ops
from . import mesh_io


def _device():
    if not torch.cuda.is_available():
        raise ops.P2SError('CUDA is not available: points2surf_b200 has no CPU fallback')
    return torch.device('cuda', torch.cuda.current_device())


def get_voxel_centers_grid_smaller_pc(pts, grid_resolution, distance_threshold_vs=10):
    """source/sdf.py:46-70 -> float32 [Q,3] (NumPy, like the reference)."""
    p = torch.from_numpy(np.ascontiguousarray(pts[:, :3], dtype=np.float32)).to(_device())
    lin = ops.query_grid(p, grid_resolution, distance_threshold_vs)
    return ops.query_points(lin, grid_resolution).cpu().numpy()


def model_space_to_volume_space(pts_ms, vol_res):
    """source/sdf.py:73-75 (float32 arithmetic for float32 input)."""
    return np.floor(((pts_ms + 1.0) / 2.0) * vol_res).astype(int)


def implicit_surface_to_mesh(query_dist_ms, query_pts_ms, volume_out_file, mc_out_file, grid_res, sigma,
                             certainty_threshold=26):
    """source/sdf.py:181-230: scatter -> sign propagation -> clamp -> marching cubes -> PLY.
    Prints the same warnings and writes nothing in the same situations as the reference."""
    query_dist_ms = np.asarray(query_dist_ms)
    if query_dist_ms.max() == 0.0 and query_dist_ms.min() == 0.0:
        print('WARNING: implicit surface for {} contains only zeros'.format(volume_out_file))
        return
    dev = _device()
    idx = model_space_to_volume_space(np.asarray(query_pts_ms), grid_res)
    if idx.size and (idx.min() < 0 or idx.max() >= grid_res):
        # the reference raises IndexError for an index >= grid_res and silently wraps a negative one
        # (sdf.py:95-111, SURVEY section 10 "Precondition"); both are rejected here, nothing is written out of bounds
        raise IndexError('query points outside [-1, 1)^3: voxel index out of range for grid resolution %d' % grid_res)
    lin = torch.from_numpy(((idx[:, 0] * grid_res + idx[:, 1]) * grid_res + idx[:, 2]).astype(np.int32)).to(dev)
    sdf = torch.from_numpy(np.ascontiguousarray(query_dist_ms, dtype=np.float32)).to(dev)
    start = time.time()
    vol, _ = ops.sdf_to_volume(lin, sdf, grid_res, sigma, certainty_threshold)
    torch.cuda.synchronize()
    print('Sign propagation took: {}'.format(time.time() - start))

    # green = inside; red = outside  (sdf.py:204-209)
    norm = query_dist_ms / np.max(np.abs(query_dist_ms))
    color = np.zeros((norm.shape[0], 3))
    color[norm < 0.0, 0] = np.abs(norm[norm < 0.0]) + 1.0 / 2.0
    color[norm > 0.0, 1] = norm[norm > 0.0] + 1.0 / 2.0
    mesh_io.write_off(volume_out_file, query_pts_ms, np.array([]), colors_vertex=color)

    vmin, vmax = float(vol.min()), float(vol.max())
    if vmin < 0.0 and vmax > 0.0:
        start = time.time()
        v, f = ops.marching_cubes(vol, 0.0)
        torch.cuda.synchronize()
        print('Marching Cubes took: {}'.format(time.time() - start))
        if v.shape[0] == 0 and f.shape[0] == 0:
            print('Warning: marching cubes gives no result!')
        else:
            mesh_io.write_ply(mc_out_file, v.cpu().numpy(), f.cpu().numpy())
    else:
        print('Warning: volume for marching cubes contains no 0-level set!')


def implicit_surface_to_mesh_file(query_dist_ms_file, query_pts_ms_file, volume_out_file, mc_out_file, grid_res, sigma,
                                  certainty_threshold):
    implicit_surface_to_mesh(np.load(query_dist_ms_file), np.load(query_pts_ms_file), volume_out_file, mc_out_file,
                             grid_res, sigma, certainty_threshold)


def _call_necessary(files_in, files_out):
    """mtime rule of source/base/file_utils.py:194-247: run when an output is missing/empty or older than an input."""
    for f in files_out:
        if not os.path.isfile(f) or os.path.getsize(f) == 0:
            return True
    newest_in = max(os.path.getmtime(f) for f in files_in)
    return any(os.path.getmtime(f) < newest_in for f in files_out)


def implicit_surface_to_mesh_directory(imp_surf_dist_ms_dir, query_pts_ms_dir, vol_out_dir, mesh_out_dir, grid_res, sigma,
                                       certainty_threshold, num_processes=1):
    """source/sdf.py:241-266.  `num_processes` is accepted and ignored: shapes run back to back on the GPU."""
    os.makedirs(vol_out_dir, exist_ok=True)
    os.makedirs(mesh_out_dir, exist_ok=True)
    files = [f for f in os.listdir(imp_surf_dist_ms_dir)
             if os.path.isfile(os.path.join(imp_surf_dist_ms_dir, f)) and f[-8:] == '.xyz.npy']
    for f in files:
        d_in, q_in = os.path.join(imp_surf_dist_ms_dir, f), os.path.join(query_pts_ms_dir, f)
        v_out, m_out = os.path.join(vol_out_dir, f[:-8] + '.off'), os.path.join(mesh_out_dir, f[:-8] + '.ply')
        if _call_necessary([d_in, q_in], [v_out, m_out]):
            implicit_surface_to_mesh_file(d_in, q_in, v_out, m_out, grid_res, sigma, certainty_threshold)


def visualize_query_points(query_pts_ms, query_dist_ms, file_out_off):
    """source/sdf.py:269-285: coloured point cloud (red = negative/outside, green = positive/inside)."""
    a = np.abs(query_dist_ms)
    an = a / a.max()
    col = np.zeros((query_dist_ms.shape[0], 3))
    neg, pos = query_dist_ms < 0.0, query_dist_ms > 0.0
    col[neg, 0] = 0.5 + 0.5 * an[neg]
    col[pos, 1] = 0.5 + 0.5 * an[pos]
    mesh_io.write_ply(file_out_off, query_pts_ms, None, colors=col)
