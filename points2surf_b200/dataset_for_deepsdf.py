"""The reference's dataset_for_deepsdf.py: turn a Points2Surf dataset into the inputs of the DeepSDF baseline.

    python -m points2surf_b200.dataset_for_deepsdf DATASET_DIR --out_dir DIR [--normals_dir 06_normals_pcpnet]

runs the body of the reference's main() for one dataset:
  1. 03_meshes -> 05_meshes_repaired: the hole filling of hole_filling_mesh_simp.mlx on the GPU (ops.mesh_repair)
  2. 04_pts of testset.txt -> DIR/data/SurfaceSamples/<dataset>/03_meshes/<name>.ply (DeepSDF's Chamfer samples)
  3. 05_query_pts / 05_query_dist of trainset.txt -> DIR/data/SdfSamples/<dataset>/03_meshes/<name>.npz
  4. 04_pts, normals and 05_meshes_repaired of testset.txt -> the same SdfSamples tree: samples eta = 0.01 off the surface
     along the normals, and 20 % far samples in [-0.5, 0.5)^3 with their signed distance to the repaired mesh, computed
     on the GPU (ops.mesh_signed_distance)
  5. DIR/examples/<dataset>/specs.json and DIR/examples/splits/<dataset>_{train,test}.json
Normals are <name>.normals text (PCPNet's output, what the reference reads) or <name>.xyz.npy (this project's 06_normals
or 06_normals_est).

Deviations from the reference: the far samples are drawn from RandomState(filename_to_hash(mesh)) (the reference's are
unseeded); the SurfaceSamples PLY is written by mesh_io with the reference's dummy faces and without merging vertices
(trimesh's exporter is not available to pin); the repaired meshes are not decimated to 100 000 faces (they only serve as
the far samples' signed-distance target, which the GPU computes on the full mesh); a second run skips every output that
is newer than its inputs, for the SDF samples too."""
import argparse
import os
import sys
import xml.etree.ElementTree as ET

import numpy as np
import torch

from . import make_dataset
from . import mesh_io
from . import ops
from . import sdf

# the Close Holes parameters of the reference's hole_filling_mesh_simp.mlx
HOLE_FILLING_MLX_DEFAULTS = dict(max_hole_size=30, prevent_self_intersection=True)
DECIMATION_TARGET_FACES = 100000
_MLX_FILTERS = ('repair non manifold edges by removing faces', 'repair non manifold edges by splitting vertices',
                'repair non manifold vertices by splitting', 'close holes',
                'simplification: quadric edge collapse decimation')


def read_hole_filling_filter(filter_file):
    """The Close Holes parameters of a meshlab script made of hole_filling_mesh_simp.mlx's filters (any subset, in its
    order).  The decimation filter is accepted and skipped.  Raises ValueError for any other filter or for parameters
    this repair does not implement (VertDispRatio != 0, Selected = true)."""
    params = dict(HOLE_FILLING_MLX_DEFAULTS)
    filters = [e for e in ET.parse(filter_file).getroot() if e.tag in ('filter', 'xmlfilter')]
    names = [e.get('name', '').lower() for e in filters]
    pos = [(_MLX_FILTERS.index(n) if n in _MLX_FILTERS else -1) for n in names]
    if not filters or -1 in pos or pos != sorted(set(pos)):
        raise ValueError('{}: only the filters of hole_filling_mesh_simp.mlx, in its order, are supported, found {}'.format(
            filter_file, [e.get('name') for e in filters]))
    for e in filters:
        for p in e:
            name, value = p.get('name'), p.get('value', '')
            if name == 'VertDispRatio' and float(value) != 0.0:
                raise ValueError('{}: VertDispRatio {} is not supported (only 0)'.format(filter_file, value))
            if e.get('name').lower() == 'close holes':
                if name == 'MaxHoleSize':
                    params['max_hole_size'] = int(value)
                elif name == 'SelfIntersection':
                    params['prevent_self_intersection'] = value.lower() == 'true'
                elif name == 'Selected' and value.lower() == 'true':
                    raise ValueError('{}: closing only selected holes is not supported'.format(filter_file))
    return params


def _device():
    if not torch.cuda.is_available():
        raise RuntimeError('dataset_for_deepsdf needs a CUDA device (the repair and the distances run on the GPU)')
    return torch.device('cuda', torch.cuda.current_device())


def repair_mesh(verts, faces, max_hole_size=30, prevent_self_intersection=True):
    """-> (verts, faces, stats) of ops.mesh_repair, as NumPy arrays"""
    dev = _device()
    v, f, stats = ops.mesh_repair(torch.from_numpy(np.ascontiguousarray(verts, np.float32)).to(dev),
                                  torch.from_numpy(np.ascontiguousarray(faces, np.int32)).to(dev),
                                  max_hole_size, prevent_self_intersection)
    return v.cpu().numpy(), f.cpu().numpy(), stats


def _set_names(file_set):
    with open(file_set) as fp:
        return set(f.replace('\n', '') for f in fp.readlines())


def _files(in_dir, ext='.npy'):
    return sorted(os.path.join(root, name) for root, _, names in os.walk(in_dir, topdown=True) for name in names
                  if name[-4:] == ext)


def _convert_pc(in_pc, out_pc):
    """dataset_for_deepsdf.py:15-40: a point cloud .npy -> PLY with dummy faces (0, 1, i), which keep every vertex."""
    pc = np.load(in_pc).astype(np.float64)
    faces = np.zeros((pc.shape[0], 3), dtype=np.int32)
    faces[:, 1] = 1
    faces[:, 2] = np.arange(pc.shape[0])
    mesh_io.write_ply(out_pc, pc, faces)


def convert_pcs(in_dir_abs, out_dir_abs, file_set, num_processes):
    """dataset_for_deepsdf.py:43-72: every <name>.xyz.npy of `file_set` -> out_dir_abs/<name>.ply, unless newer than
    its input.  `num_processes` is accepted and ignored."""
    os.makedirs(out_dir_abs, exist_ok=True)
    names = _set_names(file_set)
    for f in _files(in_dir_abs):
        base = os.path.basename(f)[:-8]
        if base not in names:
            continue
        file_out = os.path.join(out_dir_abs, base + '.ply')
        if sdf._call_necessary([f], [file_out]):
            _convert_pc(f, file_out)


def _convert_sdf(file_in_query_pts, file_in_sdf, out_pc):
    """dataset_for_deepsdf.py:75-99: query points and distances -> npz with 'pos' (d > 0) and 'neg' (d < 0) [n,4]
    float32 rows (x, y, z, d); points at d == 0 are dropped."""
    pts = np.load(file_in_query_pts).astype(np.float32)
    dist = np.load(file_in_sdf).astype(np.float32)
    out = {}
    for key, sel in (('pos', dist > 0.0), ('neg', dist < 0.0)):
        rows = np.zeros((int(sel.sum()), 4), dtype=np.float32)
        rows[:, 0:3] = pts[sel]
        rows[:, 3] = dist[sel]
        out[key] = rows
    np.savez(out_pc, pos=out['pos'], neg=out['neg'])


def convert_sdfs(in_dir_query_pts, in_dir_query_sdf, out_dir_sdf, file_set, num_processes):
    """dataset_for_deepsdf.py:167-194 for the shapes of `file_set`, skipping outputs newer than their inputs."""
    if not os.path.isfile(file_set):
        print('WARNING: dataset is missing a set file: {}'.format(file_set))
        return
    os.makedirs(out_dir_sdf, exist_ok=True)
    names = _set_names(file_set)
    for f in _files(in_dir_query_pts):
        base = os.path.basename(f)[:-8]
        if base not in names:
            continue
        file_out = os.path.join(out_dir_sdf, base + '.npz')
        file_sdf = os.path.join(in_dir_query_sdf, base + '.ply.npy')
        if sdf._call_necessary([f, file_sdf], [file_out]):
            _convert_sdf(f, file_sdf, file_out)


def _read_normals(file_in_normal):
    if file_in_normal.endswith('.npy'):
        return np.load(file_in_normal).astype(np.float64)[:, :3]
    return np.loadtxt(file_in_normal)


def _rows(pts, dist):
    rows = np.zeros((pts.shape[0], 4), dtype=np.float32)
    rows[:, 0:3] = pts
    rows[:, 3] = dist
    return rows


def close_samples(pts, normals, eta=0.01):
    """The near-surface samples of _make_sdf_samples_from_pc, float64 on the host: pts +- eta n / |n|.
    -> (outside points, inside points, their values -eta / +eta)"""
    n = normals / np.linalg.norm(normals, axis=1)[:, None]
    return pts + eta * n, pts - eta * n, np.full((pts.shape[0],), -eta), np.full((pts.shape[0],), eta)


def far_samples(num_close, file_in_mesh):
    """int(num_close * 0.2) uniform points in [-0.5, 0.5)^3 from RandomState(filename_to_hash(file_in_mesh))"""
    rng = np.random.RandomState(make_dataset.filename_to_hash(file_in_mesh))
    return rng.rand(int(num_close * 0.2), 3) - 0.5


def _make_sdf_samples_from_pc(file_in_pts, file_in_normal, file_in_mesh, out_pc):
    """dataset_for_deepsdf.py:102-164 for one shape.  Close samples on the host in float64 (close_samples), stored
    with the reference's key swap ('pos' holds the inside points pts - eta n with value +eta, 'neg' the outside points
    with -eta).  Far samples (far_samples): signed distance to the mesh on the GPU, positive inside (trimesh's sign),
    split into 'pos_far' (> 0) and 'neg_far' (< 0).  Also writes the coloured point cloud out_pc + '.ply'."""
    pts = np.load(file_in_pts).astype(np.float32)
    query_pts_pos, query_pts_neg, signed_dist_pos, signed_dist_neg = close_samples(pts, _read_normals(file_in_normal))
    far = far_samples(query_pts_pos.shape[0] + query_pts_neg.shape[0], file_in_mesh)
    verts, faces = mesh_io.read_mesh(file_in_mesh)
    far_sd = sdf.get_signed_distance(in_mesh=(verts, faces), query_pts_ms=far)
    far_pos, far_neg = far_sd > 0.0, far_sd < 0.0

    np.savez(out_pc, pos=_rows(query_pts_neg, signed_dist_neg), neg=_rows(query_pts_pos, signed_dist_pos),
             pos_far=_rows(far[far_pos], far_sd[far_pos]), neg_far=_rows(far[far_neg], far_sd[far_neg]))

    file_out_query_vis = out_pc + '.ply'
    sdf.visualize_query_points(np.concatenate((query_pts_pos, query_pts_neg, far[far_pos], far[far_neg])),
                               np.concatenate((signed_dist_pos, signed_dist_neg, far_sd[far_pos], far_sd[far_neg])),
                               file_out_query_vis)
    print('wrote vis to {}'.format(file_out_query_vis))


def _normals_file(in_dir_normals, base):
    txt = os.path.join(in_dir_normals, base + '.normals')
    npy = os.path.join(in_dir_normals, base + '.xyz.npy')
    return npy if not os.path.isfile(txt) and os.path.isfile(npy) else txt


def make_sdf_samples(in_dir_pts, in_dir_normals, in_dir_meshes, out_dir_sdf, file_set, num_processes):
    """dataset_for_deepsdf.py:197-225 for the shapes of `file_set`, skipping outputs newer than their inputs."""
    if not os.path.isfile(file_set):
        print('WARNING: dataset is missing a set file: {}'.format(file_set))
        return
    os.makedirs(out_dir_sdf, exist_ok=True)
    names = _set_names(file_set)
    for f in _files(in_dir_pts):
        base = os.path.basename(f)[:-8]
        if base not in names:
            continue
        file_out = os.path.join(out_dir_sdf, base + '.npz')
        file_normal = _normals_file(in_dir_normals, base)
        file_mesh = os.path.join(in_dir_meshes, base + '.ply')
        if sdf._call_necessary([f, file_normal, file_mesh], [file_out, file_out + '.ply']):
            _make_sdf_samples_from_pc(f, file_normal, file_mesh, file_out)


# DeepSDF's default experiment settings as the reference writes them (without code_bound)
_SPECS_JSON = '''
{
  "Description" : [ "converted from @ORIGIN@." ],
  "DataSource" : "data/",
  "TrainSplit" : "examples/splits/@DATASET@_train.json",
  "TestSplit" : "examples/splits/@DATASET@_test.json",
  "NetworkArch" : "deep_sdf_decoder",
  "NetworkSpecs" : {
    "dims" : [ 512, 512, 512, 512, 512, 512, 512, 512 ],
    "dropout" : [0, 1, 2, 3, 4, 5, 6, 7],
    "dropout_prob" : 0.2,
    "norm_layers" : [0, 1, 2, 3, 4, 5, 6, 7],
    "latent_in" : [4],
    "xyz_in_all" : false,
    "use_tanh" : false,
    "latent_dropout" : false,
    "weight_norm" : true
    },
  "CodeLength" : 256,
  "NumEpochs" : 1001,
  "SnapshotFrequency" : 100,
  "AdditionalSnapshots" : [ 100, 200, 500 ],
  "LearningRateSchedule" : [
    {
      "Type" : "Step",
      "Initial" : 0.0005,
      "Interval" : 500,
      "Factor" : 0.5
    },
    {
      "Type" : "Step",
      "Initial" : 0.001,
      "Interval" : 500,
      "Factor" : 0.5
    }],
  "SamplesPerScene" : 16384,
  "ScenesPerBatch" : 64,
  "DataLoaderThreads" : 16,
  "ClampingDistance" : 0.1,
  "CodeRegularization" : true,
  "CodeRegularizationLambda" : 1e-4
}
    '''


def _split_json(dataset, set_file):
    with open(set_file) as fp:
        lines = ['\t\t\t"{}",'.format(f.replace('\n', '')) for f in fp.readlines()]
    lines[-1] = lines[-1][:-1]
    return '\n{\n  "%s": {\n    "03_meshes": [\n' % dataset + '\n'.join(lines) + '\n    ]\n  }\n}\n'


def create_example(train_set, test_set, out_dir_examples, dataset):
    """dataset_for_deepsdf.py:228-316: out_dir_examples/<dataset>/specs.json and, for each set file that exists,
    out_dir_examples/splits/<dataset>_{train,test}.json, byte for byte as the reference writes them."""
    out_dir_example = os.path.join(out_dir_examples, dataset)
    os.makedirs(out_dir_example, exist_ok=True)
    with open(os.path.join(out_dir_example, 'specs.json'), 'w') as fp:
        fp.write(_SPECS_JSON.replace('@ORIGIN@', train_set).replace('@DATASET@', dataset))
    out_dir_splits = os.path.join(out_dir_examples, 'splits')
    os.makedirs(out_dir_splits, exist_ok=True)
    for set_file, kind in ((train_set, 'train'), (test_set, 'test')):
        if os.path.isfile(set_file):
            with open(os.path.join(out_dir_splits, '{}_{}.json'.format(dataset, kind)), 'w') as fp:
                fp.write(_split_json(dataset, set_file))


def apply_meshlab_filter(base_dir, dataset_dir, in_dir, out_dir, num_processes, filter_file, meshlabserver_bin):
    """dataset_for_deepsdf.py:319-336 without meshlab: every mesh of <in_dir> repaired on the GPU (ops.mesh_repair) into
    <out_dir>/<same name> as PLY, unless that is newer than its input.  The parameters come from `filter_file` when it
    exists (read_hole_filling_filter), else from hole_filling_mesh_simp.mlx (HOLE_FILLING_MLX_DEFAULTS).  The decimation
    is not done; a repaired mesh above 100 000 faces is reported.  `num_processes` and `meshlabserver_bin` are accepted
    and ignored."""
    params = read_hole_filling_filter(filter_file) if filter_file and os.path.isfile(filter_file) \
        else dict(HOLE_FILLING_MLX_DEFAULTS)
    in_dir_abs = os.path.join(base_dir, dataset_dir, in_dir)
    out_dir_abs = os.path.join(base_dir, dataset_dir, out_dir)
    os.makedirs(out_dir_abs, exist_ok=True)
    for name in sorted(os.listdir(in_dir_abs)):
        file_in = os.path.join(in_dir_abs, name)
        file_out = os.path.join(out_dir_abs, name)
        if not os.path.isfile(file_in) or not sdf._call_necessary([file_in], [file_out]):
            continue
        v, f = mesh_io.read_mesh(file_in)
        v, f, stats = repair_mesh(v, f, **params)
        if len(f) > DECIMATION_TARGET_FACES:
            print('{}: {} faces, not decimated to {}'.format(file_out, len(f), DECIMATION_TARGET_FACES))
        mesh_io.write_ply(file_out, v, f)


def main(argv=None):
    parser = argparse.ArgumentParser(description='Write the DeepSDF baseline inputs (SdfSamples, SurfaceSamples, '
                                                 'examples) of a Points2Surf dataset.')
    parser.add_argument('dataset_dir', help='dataset directory containing 03_meshes, 04_pts, 05_query_pts, ...')
    parser.add_argument('--out_dir', required=True, help='DeepSDF root: data/ and examples/ are written under it')
    parser.add_argument('--normals_dir', default='06_normals_pcpnet',
                        help='normals of 04_pts inside the dataset (<name>.normals text or <name>.xyz.npy)')
    parser.add_argument('--filter_file', default='hole_filling_mesh_simp.mlx',
                        help='meshlab script with the repair parameters (defaults of the reference\'s when missing)')
    args = parser.parse_args(argv)
    dataset = os.path.abspath(args.dataset_dir)
    base_dir, name = os.path.dirname(dataset), os.path.basename(dataset)
    out_dir = os.path.abspath(args.out_dir)
    print('Processing {}'.format(name))
    test_set = os.path.join(dataset, 'testset.txt')
    train_set = os.path.join(dataset, 'trainset.txt')
    apply_meshlab_filter(base_dir=base_dir, dataset_dir=name, in_dir='03_meshes', out_dir='05_meshes_repaired',
                         num_processes=1, filter_file=args.filter_file, meshlabserver_bin=None)
    convert_pcs(os.path.join(dataset, '04_pts'), os.path.join(out_dir, 'data', 'SurfaceSamples', name, '03_meshes'),
                test_set, 1)
    out_dir_sdf = os.path.join(out_dir, 'data', 'SdfSamples', name, '03_meshes')
    convert_sdfs(in_dir_query_pts=os.path.join(dataset, '05_query_pts'), in_dir_query_sdf=os.path.join(dataset, '05_query_dist'),
                 out_dir_sdf=out_dir_sdf, file_set=train_set, num_processes=1)
    make_sdf_samples(in_dir_pts=os.path.join(dataset, '04_pts'), in_dir_normals=os.path.join(dataset, args.normals_dir),
                     in_dir_meshes=os.path.join(dataset, '05_meshes_repaired'), out_dir_sdf=out_dir_sdf,
                     file_set=test_set, num_processes=1)
    create_example(train_set=train_set, test_set=test_set, out_dir_examples=os.path.join(out_dir, 'examples'),
                   dataset=name)


if __name__ == '__main__':
    main(sys.argv[1:])
