"""Drop-in for the hot-path functions of source/sdf.py, on the CUDA kernels."""
import hashlib
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


def volume_lin_idx(query_pts_ms, grid_res):
    """The voxels of the query points (model_space_to_volume_space) as int32 linear indices (ix * res + iy) * res + iz on
    the device, the scatter order of ops.sdf_to_volume."""
    idx = model_space_to_volume_space(np.asarray(query_pts_ms), grid_res)
    if idx.size and (idx.min() < 0 or idx.max() >= grid_res):
        # the reference raises IndexError for an index >= grid_res and silently wraps a negative one
        # (sdf.py:95-111, SURVEY section 10 "Precondition"); both are rejected here, nothing is written out of bounds
        raise IndexError('query points outside [-1, 1)^3: voxel index out of range for grid resolution %d' % grid_res)
    return torch.from_numpy(((idx[:, 0] * grid_res + idx[:, 1]) * grid_res + idx[:, 2]).astype(np.int32)).to(_device())


def implicit_surface_to_mesh(query_dist_ms, query_pts_ms, volume_out_file, mc_out_file, grid_res, sigma,
                             certainty_threshold=26):
    """source/sdf.py:181-230: scatter -> sign propagation -> clamp -> marching cubes -> PLY.
    Prints the same warnings and writes nothing in the same situations as the reference."""
    query_dist_ms = np.asarray(query_dist_ms)
    if query_dist_ms.max() == 0.0 and query_dist_ms.min() == 0.0:
        print('WARNING: implicit surface for {} contains only zeros'.format(volume_out_file))
        return
    dev = _device()
    lin = volume_lin_idx(query_pts_ms, grid_res)
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


def _mesh_arrays(in_mesh):
    """(vertices [V,3] float32, faces [F,3] int32) of an object with .vertices / .faces or of a (vertices, faces) pair."""
    v, f = (in_mesh.vertices, in_mesh.faces) if hasattr(in_mesh, 'vertices') else in_mesh
    v = np.ascontiguousarray(v, dtype=np.float32).reshape(-1, 3)
    f = np.ascontiguousarray(f, dtype=np.int32).reshape(-1, 3)
    if len(f) == 0 or f.min() < 0 or f.max() >= len(v):
        raise ops.P2SError('mesh has no faces or a face index outside [0, V)')
    return v, f


def _orient_outward(verts, faces):
    """The global part of trimesh's fix_normals (called at source/sdf.py:307): reverse every face when the mesh's signed
    volume is negative.  Faces oriented inconsistently with their neighbours are not repaired."""
    v = verts.astype(np.float64)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    if np.einsum('ij,ij->', a, np.cross(b, c)) < 0.0:
        return np.ascontiguousarray(faces[:, ::-1])
    return faces


def _query_pts_rng_draws(rng, num_query_pts, patch_radius, far_query_pts_ratio):
    """What source/sdf.py:295,304-311 draws from the caller's stream, in its order: the close points' offsets along the
    normal in [-patch_radius, patch_radius), then the far points in [-0.5, 0.5)^3.  -> (offsets [num_close], far [num_far,3])"""
    num_far = int(num_query_pts * far_query_pts_ratio)
    num_close = num_query_pts - num_far
    offset = (rng.random(size=(num_close,)) - 0.5) * 2.0 * patch_radius
    far = rng.random(size=(num_far, 3)) - 0.5
    return offset, far


def _sampler_seed(rng):
    """Seed of the surface sampler, read from the caller's stream without drawing from it (so that the draws of
    _query_pts_rng_draws stay the reference's): different streams and positions give different samples."""
    _, key, pos = rng.get_state()[:3]
    return int.from_bytes(hashlib.blake2b(key.tobytes() + int(pos).to_bytes(4, 'little'), digest_size=8).digest(), 'little')


def _query_pts_and_faces(in_mesh, num_query_pts, patch_radius, far_query_pts_ratio, rng):
    verts, faces = _mesh_arrays(in_mesh)
    faces = _orient_outward(verts, faces)
    seed = _sampler_seed(rng)
    offset, far = _query_pts_rng_draws(rng, num_query_pts, patch_radius, far_query_pts_ratio)
    dev = _device()
    samples, face_id = ops.mesh_sample(torch.from_numpy(verts).to(dev), torch.from_numpy(faces).to(dev), len(offset), seed,
                                       return_face_ids=True)
    samples, face_id = samples.cpu().numpy().astype(np.float64), face_id.cpu().numpy()
    v = verts.astype(np.float64)
    f = faces[face_id]
    n = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    n /= np.linalg.norm(n, axis=1, keepdims=True)                      # trimesh's unit face normals
    n /= np.sqrt(np.linalg.norm(n, axis=1, keepdims=True))             # the reference's extra step (source/sdf.py:297-299)
    close = samples + offset[:, None] * n
    return np.concatenate((far, close), axis=0), face_id


def get_query_pts_for_mesh(in_mesh, num_query_pts, patch_radius, far_query_pts_ratio=0.1, rng=None):
    """source/sdf.py:288-315 -> float64 [num_query_pts, 3]: int(num_query_pts * far_query_pts_ratio) uniform points in
    [-0.5, 0.5)^3, then points near the surface (area-weighted surface samples moved along their face normal by a uniform
    offset in [-patch_radius, patch_radius)).  The offsets and the far points come from `rng` in the reference's order, so
    the far half is bit-identical to the reference's for the same stream.  The surface samples come from the device
    sampler (p2s_mesh_sample_dev, seeded from rng's state without drawing from it); the reference's are unseeded.
    Of `in_mesh.fix_normals()` only the global flip is applied (faces reversed when the signed volume is negative), and
    `in_mesh` is not modified.  `in_mesh`: anything with .vertices / .faces, or a (vertices, faces) pair."""
    rng = np.random.RandomState() if rng is None else rng
    return _query_pts_and_faces(in_mesh, num_query_pts, patch_radius, far_query_pts_ratio, rng)[0]


def get_signed_distance(in_mesh, query_pts_ms, signed_distance_batch_size=1000):
    """source/sdf.py:318-348 -> float64 [Q]: distance to the mesh, positive inside and on the surface (trimesh's
    convention), on the device in one exhaustive pass (p2s_mesh_signed_distance_dev).  `signed_distance_batch_size` is
    accepted and ignored: there is no memory blow-up to batch around.  The query points are rounded to float32 (what
    05_query_pts stores).  The mesh is oriented outward like get_query_pts_for_mesh does (the sign comes from the
    winding number, which depends on orientation; trimesh's ray test does not)."""
    verts, faces = _mesh_arrays(in_mesh)
    faces = _orient_outward(verts, faces)
    dev = _device()
    q = torch.from_numpy(np.ascontiguousarray(np.asarray(query_pts_ms).reshape(-1, 3), dtype=np.float32)).to(dev)
    d = ops.mesh_signed_distance(torch.from_numpy(verts).to(dev), torch.from_numpy(faces).to(dev), q)
    dists_ms = d.cpu().numpy().astype(np.float64)
    num_nans, num_infs = int(np.isnan(dists_ms).sum()), int(np.isinf(dists_ms).sum())
    if num_nans > 0 or num_infs > 0:
        print('Error: Encountered {} NaN and {} Inf values in signed distance of {}.'.format(num_nans, num_infs, query_pts_ms))
    return dists_ms


def visualize_query_points(query_pts_ms, query_dist_ms, file_out_off):
    """source/sdf.py:269-285: coloured point cloud (red = negative/outside, green = positive/inside)."""
    a = np.abs(query_dist_ms)
    an = a / a.max()
    col = np.zeros((query_dist_ms.shape[0], 3))
    neg, pos = query_dist_ms < 0.0, query_dist_ms > 0.0
    col[neg, 0] = 0.5 + 0.5 * an[neg]
    col[pos, 1] = 0.5 + 0.5 * an[pos]
    mesh_io.write_ply(file_out_off, query_pts_ms, None, colors=col)
