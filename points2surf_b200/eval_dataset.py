"""The ground-truth point normals of the reference's eval_dataset.py (utils.get_pts_normals, source/base/utils.py:109-164),
which the "SPSR + GT normals" baseline reconstructs from, with the point-to-mesh work on the GPU:
  device surface samples with their face ids (p2s_mesh_sample_dev) -> nearest sample of every cloud point
  (p2s_nn_distance_dev, cKDTree's semantics) -> the oriented unit normal of that sample's face.

    python -m points2surf_b200.eval_dataset DATASET_DIR

writes DATASET_DIR/06_normals/<name>.xyz.npy and 06_normals/pts/<name>.xyz from 04_pts and 03_meshes with 100 000 samples
per mesh, like eval_dataset.py:143-146.  The Screened-Poisson stages of eval_dataset.py need meshlabserver and are not
run; with --spsr

    python -m points2surf_b200.eval_dataset DATASET_DIR --spsr

the "SPSR + GT normals" stage of eval_dataset.py:143-158 runs instead, with the reconstruction on the GPU
(apply_meshlab_filter, points2surf_b200/poisson.py): 06_normals, then 06_poisson_rec_gt_normals/<name>.ply, then
comp_poisson_rec_gt_normals.csv against 03_meshes for the shapes in valset.txt.  With --spsr_estimated_normals

    python -m points2surf_b200.eval_dataset DATASET_DIR --spsr_estimated_normals

the stage of the reference's normals_poisson.mlx (eval_dataset.py:160-172) runs without meshlab and without meshes: oriented
normals estimated from 04_pts alone (ops.point_normals) into 06_normals_est, Screened Poisson from them into 06_poisson_rec,
and comp_poisson_rec_ml_normals.csv when 03_meshes and valset.txt exist."""
import argparse
import os
import sys
import xml.etree.ElementTree as ET

import numpy as np
import torch

from . import evaluation
from . import make_dataset
from . import mesh_io
from . import ops
from . import point_cloud
from . import poisson
from . import sdf

# the Screened Poisson parameters of the reference's poisson.mlx that this reconstruction uses
POISSON_MLX_DEFAULTS = dict(depth=8, point_weight=4.0, scale=1.1, iters=8)
# the "Compute normals for point sets" parameters of the reference's normals_poisson.mlx
NORMALS_MLX_DEFAULTS = dict(k=10, smooth_iter=0, flip_flag=False, view_pos=(0.0, 0.0, 0.0))
_MLX_PARAMS = dict(depth=('depth', int), pointWeight=('point_weight', float), scale=('scale', float),
                   iters=('iters', int))


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


def read_poisson_filter(filter_file):
    """depth / point_weight / scale / iters of the Screened Poisson filter in a meshlab filter script (.mlx), the
    poisson.mlx defaults for a parameter it does not set.  Raises ValueError when the script holds any other filter."""
    params = dict(POISSON_MLX_DEFAULTS)
    filters = [e for e in ET.parse(filter_file).getroot() if e.tag in ('filter', 'xmlfilter')]
    names = [e.get('name', '') for e in filters]
    if len(filters) != 1 or 'screened poisson' not in names[0].lower():
        raise ValueError('{}: only a single Screened Poisson filter is supported, found {}'.format(filter_file, names))
    for p in filters[0]:
        if p.get('name') in _MLX_PARAMS:
            key, conv = _MLX_PARAMS[p.get('name')]
            params[key] = conv(p.get('value'))
    return params


def apply_meshlab_filter(base_dir, dataset_dir, pts_dir, recon_mesh_dir, num_processes, filter_file, meshlabserver_bin):
    """eval_dataset.py:50-67 without meshlab: Screened Poisson reconstruction (points2surf_b200/poisson.py) of every
    <pts_dir>/<name>.xyz (text x y z nx ny nz, as point_cloud.write_xyz writes it) into <recon_mesh_dir>/<name>.ply,
    unless that is newer than its input.  The parameters come from `filter_file` when it exists (read_poisson_filter),
    else from poisson.mlx (POISSON_MLX_DEFAULTS).  `num_processes` and `meshlabserver_bin` are accepted and ignored."""
    params = read_poisson_filter(filter_file) if filter_file and os.path.isfile(filter_file) \
        else dict(POISSON_MLX_DEFAULTS)
    _poisson_reconstruct_dir(base_dir, dataset_dir, pts_dir, recon_mesh_dir, params)


def _poisson_reconstruct_dir(base_dir, dataset_dir, pts_dir, recon_mesh_dir, params):
    """The per-file loop of apply_meshlab_filter with the Screened Poisson parameters given."""
    pts_dir_abs = os.path.join(base_dir, dataset_dir, pts_dir)
    recon_mesh_dir_abs = os.path.join(base_dir, dataset_dir, recon_mesh_dir)
    os.makedirs(recon_mesh_dir_abs, exist_ok=True)
    pts_files = sorted(f for f in os.listdir(pts_dir_abs)
                       if os.path.isfile(os.path.join(pts_dir_abs, f)) and f[-4:] == '.xyz')
    for pts_file in pts_files:
        pts_file_abs = os.path.join(pts_dir_abs, pts_file)
        mesh_abs = os.path.join(recon_mesh_dir_abs, pts_file[:-4] + '.ply')
        if not sdf._call_necessary([pts_file_abs], [mesh_abs]):
            continue
        xyz = np.loadtxt(pts_file_abs, dtype=np.float64, ndmin=2)
        if xyz.shape[1] < 6:
            raise ValueError('{}: Screened Poisson needs points with normals (x y z nx ny nz)'.format(pts_file_abs))
        verts, faces, _ = poisson.reconstruct(xyz[:, :3], xyz[:, 3:6], **params)
        mesh_io.write_ply(mesh_abs, verts, faces)


def read_normals_poisson_filter(filter_file):
    """A meshlab filter script of the shape of the reference's normals_poisson.mlx: "Compute normals for point sets", then
    Screened Poisson ("Delete Current Mesh" filters are ignored).
    -> (dict(k, smooth_iter, flip_flag, view_pos), Screened Poisson parameters like read_poisson_filter's).
    Raises ValueError for any other script, and for smoothIter != 0 (normal smoothing is not built)."""
    normals = dict(NORMALS_MLX_DEFAULTS)
    params = dict(POISSON_MLX_DEFAULTS)
    filters = [e for e in ET.parse(filter_file).getroot() if e.tag in ('filter', 'xmlfilter')
               and 'delete current mesh' not in e.get('name', '').lower()]
    names = [e.get('name', '') for e in filters]
    if len(filters) != 2 or 'compute normals for point sets' not in names[0].lower() \
            or 'screened poisson' not in names[1].lower():
        raise ValueError('{}: expected "Compute normals for point sets" followed by Screened Poisson, found {}'.format(
            filter_file, names))
    for p in filters[0]:
        name = p.get('name')
        if name == 'K':
            normals['k'] = int(p.get('value'))
        elif name == 'smoothIter':
            normals['smooth_iter'] = int(p.get('value'))
        elif name == 'flipFlag':
            normals['flip_flag'] = p.get('value', '').lower() == 'true'
        elif name == 'viewPos':
            normals['view_pos'] = tuple(float(p.get(a)) for a in ('x', 'y', 'z'))
    if normals['smooth_iter'] != 0:
        raise ValueError('{}: smoothIter = {} (normal smoothing is not built)'.format(filter_file, normals['smooth_iter']))
    for p in filters[1]:
        if p.get('name') in _MLX_PARAMS:
            key, conv = _MLX_PARAMS[p.get('name')]
            params[key] = conv(p.get('value'))
    return normals, params


def estimate_pts_normals(base_dir, dataset_dir, dir_in_pointcloud, dir_out_normals, k=10, flip_flag=False,
                         view_pos=(0.0, 0.0, 0.0)):
    """For every <name>.xyz.npy in dir_in_pointcloud ([N,3] or [N,6]; the points are columns 0:3) write the estimated
    oriented normals dir_out_normals/<name>.xyz.npy (float64 [N,3], like 06_normals) and dir_out_normals/pts/<name>.xyz,
    unless both are newer than the input.  ops.point_normals over k neighbours; flip_flag: every normal faces view_pos
    (meshlab's flipFlag / viewPos), else the signs are propagated over the cloud."""
    dir_in_abs = os.path.join(base_dir, dataset_dir, dir_in_pointcloud)
    dir_out_abs = os.path.join(base_dir, dataset_dir, dir_out_normals)
    dir_out_pts_abs = os.path.join(dir_out_abs, 'pts')
    os.makedirs(dir_out_pts_abs, exist_ok=True)
    dev = sdf._device()
    for f in sorted(f for f in os.listdir(dir_in_abs) if os.path.isfile(os.path.join(dir_in_abs, f)) and f[-4:] == '.npy'):
        pts_in = os.path.join(dir_in_abs, f)
        normals_out = os.path.join(dir_out_abs, f)
        pts_normals_out = os.path.join(dir_out_pts_abs, f[:-8] + '.xyz')
        if not sdf._call_necessary([pts_in], [normals_out, pts_normals_out]):
            continue
        pts = np.load(pts_in)[:, :3]
        p = torch.from_numpy(np.ascontiguousarray(pts, np.float32)).to(dev)
        normals = ops.point_normals(p, k=k, mode='viewpoint' if flip_flag else 'propagate',
                                    viewpoint=view_pos if flip_flag else None).cpu().numpy().astype(np.float64)
        np.save(normals_out, normals)
        point_cloud.write_xyz(pts_normals_out, pts, normals=normals)


def _spsr_estimated_normals(dataset, base_dir, dataset_dir):
    """The normals_poisson.mlx stage of eval_dataset.py:160-172 without meshlab: 06_normals_est, 06_poisson_rec and, when
    03_meshes and valset.txt exist, comp_poisson_rec_ml_normals.csv."""
    filter_file = 'normals_poisson.mlx'
    normals, params = read_normals_poisson_filter(filter_file) if os.path.isfile(filter_file) \
        else (dict(NORMALS_MLX_DEFAULTS), dict(POISSON_MLX_DEFAULTS))
    print('### normal estimation for point cloud')
    estimate_pts_normals(base_dir=base_dir, dataset_dir=dataset_dir, dir_in_pointcloud='04_pts',
                         dir_out_normals='06_normals_est', k=normals['k'], flip_flag=normals['flip_flag'],
                         view_pos=normals['view_pos'])
    print('### poisson reconstruction from estimated normals')
    _poisson_reconstruct_dir(base_dir, dataset_dir, '06_normals_est/pts', '06_poisson_rec', params)
    if os.path.isdir(os.path.join(dataset, '03_meshes')) and os.path.isfile(os.path.join(dataset, 'valset.txt')):
        print('### normal estimation and poisson reconstruction - hausdorff distance')
        evaluation.mesh_comparison(new_meshes_dir_abs=os.path.join(dataset, '06_poisson_rec'),
                                   ref_meshes_dir_abs=os.path.join(dataset, '03_meshes'), num_processes=1,
                                   report_name=os.path.join(dataset, 'comp_poisson_rec_ml_normals.csv'),
                                   samples_per_model=10000, dataset_file_abs=os.path.join(dataset, 'valset.txt'))


def main(argv=None):
    parser = argparse.ArgumentParser(description='Ground-truth point normals (06_normals) for the point clouds in '
                                                 'DATASET_DIR/04_pts from the meshes in DATASET_DIR/03_meshes.')
    parser.add_argument('dataset_dir', help='dataset directory containing 03_meshes and 04_pts')
    parser.add_argument('--spsr', action='store_true',
                        help='also reconstruct Screened Poisson surfaces from the ground-truth normals on the GPU '
                             '(06_poisson_rec_gt_normals) and compare them with 03_meshes for the shapes in valset.txt '
                             '(comp_poisson_rec_gt_normals.csv)')
    parser.add_argument('--spsr_estimated_normals', action='store_true',
                        help='estimate oriented normals from 04_pts alone on the GPU (06_normals_est), reconstruct Screened '
                             'Poisson surfaces from them (06_poisson_rec) and, when 03_meshes and valset.txt exist, compare '
                             '(comp_poisson_rec_ml_normals.csv); needs neither 03_meshes nor 06_normals')
    args = parser.parse_args(argv)
    dataset = os.path.abspath(args.dataset_dir)
    base_dir, dataset_dir = os.path.dirname(dataset), os.path.basename(dataset)
    if args.spsr_estimated_normals:
        _spsr_estimated_normals(dataset, base_dir, dataset_dir)
        if not args.spsr:
            return
    if args.spsr:
        print('### Screened-Poisson reconstruction from PCPNet normals (06_poisson_rec_pcpnet_normals) needs '
              'PCPNet\'s normals: skipped')
    else:
        print('### Screened-Poisson reconstructions (06_poisson_rec*) need meshlabserver: skipped')
    print('### get ground truth normals for point cloud')
    get_pts_normals(base_dir=base_dir, dataset_dir=dataset_dir,
                    dir_in_pointcloud='04_pts', dir_in_meshes='03_meshes', dir_out_normals='06_normals',
                    samples_per_model=100000)
    if not args.spsr:
        return
    print('### poisson reconstruction from gt normals')
    apply_meshlab_filter(base_dir=base_dir, dataset_dir=dataset_dir, pts_dir='06_normals/pts',
                         recon_mesh_dir='06_poisson_rec_gt_normals', num_processes=1,
                         filter_file='poisson.mlx', meshlabserver_bin=None)
    print('### normal estimation and poisson reconstruction gt normals - hausdorff distance')
    evaluation.mesh_comparison(new_meshes_dir_abs=os.path.join(dataset, '06_poisson_rec_gt_normals'),
                               ref_meshes_dir_abs=os.path.join(dataset, '03_meshes'), num_processes=1,
                               report_name=os.path.join(dataset, 'comp_poisson_rec_gt_normals.csv'),
                               samples_per_model=10000, dataset_file_abs=os.path.join(dataset, 'valset.txt'))


if __name__ == '__main__':
    main(sys.argv[1:])
