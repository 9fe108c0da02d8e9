"""Mirror of the reference's `source.points_to_surf_train` (SURVEY.md section 8f-4): `parse_arguments` with the same
flags and defaults, `points_to_surf_train(opt)` with the same epoch / batch / test-interleaving structure, learning-rate
schedule, printed progress lines and output files (`<outdir>/<name>_params.pth`, `_model.pth`, `_model_<epoch>.pth`,
`_description.txt`; state dicts carry the `module.` prefix of the DataParallel wrapper the reference saves, so
`points2surf_b200.eval` and the reference's own evaluation load them).

What runs where: the per-sample work of the reference's DataLoader workers (kNN patch, sub-sample, rotation augmentation,
source/data_loader.py:322-421) is done per batch on the GPU through `points2surf_b200.ops` (the same call sequence as the
evaluation pass), the network iteration through `points2surf_b200.train.TrainStep`.  Random streams differ from the
reference's NumPy / per-worker streams (same sampling laws); the index samplers and the parameter initialisation reproduce
the reference bit for bit (`tests/golden/samplers.npz`, `tests/golden/train_init.npz`).

Status: the host logic is exercised on the CPU with the test primitives (tests/test_train_loop.py); the GPU assembly branch
has not been run on hardware yet (no GPU budget was left when it was written) -- see DESIGN.md section 7.

Supported configuration: the subset of points2surf_b200.train (`max` pooling; magnitude + sign outputs, or the regression
output `imp_surf` with `patch_pts_ids` and `p_index`, the output lists points2surf_b200.eval accepts).
"""
import argparse
import math
import os
import random
import shutil

import numpy as np
import torch

from . import arch, samplers
from .train import TrainStep


def parse_arguments(args=None):
    """The reference's training flags (source/points_to_surf_train.py:28-137), same names, types and defaults."""
    p = argparse.ArgumentParser()
    p.add_argument('--name', type=str, default='debug', help='training run name')
    p.add_argument('--desc', type=str, default='My training run for single-scale normal estimation.', help='description')
    p.add_argument('--indir', type=str, default='datasets/abc_minimal', help='input folder (meshes)')
    p.add_argument('--outdir', type=str, default='models', help='output folder (trained models)')
    p.add_argument('--logdir', type=str, default='logs', help='training log folder')
    p.add_argument('--trainset', type=str, default='trainset.txt', help='training set file name')
    p.add_argument('--testset', type=str, default='testset.txt', help='test set file name')
    p.add_argument('--save_interval', type=int, default='10', help='save model each n epochs')
    p.add_argument('--debug_interval', type=int, default='1', help='print logging info each n epochs')
    p.add_argument('--refine', type=str, default='', help='refine model at this path')
    p.add_argument('--gpu_idx', type=int, default=[0], nargs='+', help='GPU indices (this implementation needs >= 0)')
    p.add_argument('--patch_radius', type=float, default=0.05, help='Neighborhood of points that is queried per patch. Fixed radius ball query if r > 0.0, k-NN query if r <= 0.0')
    p.add_argument('--net_size', type=int, default=1024, help='number of neurons in the largest fully connected layer')
    p.add_argument('--nepoch', type=int, default=2, help='number of epochs to train for')
    p.add_argument('--batchSize', type=int, default=2, help='input batch size')
    p.add_argument('--patch_center', type=str, default='point', help='center patch at point / mean')
    p.add_argument('--patch_point_count_std', type=float, default=0, help='standard deviation of the number of points in a patch')
    p.add_argument('--patches_per_shape', type=int, default=1000, help='number of patches sampled from each shape in an epoch')
    p.add_argument('--sub_sample_size', type=int, default=500, help='number of points of the point cloud that are trained with each patch')
    p.add_argument('--workers', type=int, default=8, help='accepted for compatibility (batches are assembled on the GPU)')
    p.add_argument('--cache_capacity', type=int, default=100, help='max. number of shapes held at the same time')
    p.add_argument('--seed', type=int, default=3627473, help='manual seed')
    p.add_argument('--single_transformer', type=int, default=0, help='0: two transformers, 1: unsupported here')
    p.add_argument('--uniform_subsample', type=int, default=0, help='1: uniform global sub-sample, 0: distance-dependent')
    p.add_argument('--fixed_subsample', type=int, default=0, help='1: same fixed sub-sample for all patches (with --uniform_subsample 1 only)')
    p.add_argument('--shared_transformer', type=int, default=0, help='single shared QSTN for the local and global point sets')
    p.add_argument('--training_order', type=str, default='random', help='random | random_shape_consecutive')
    p.add_argument('--identical_epochs', type=int, default=False, help='use same patches in each epoch, mainly for debugging')
    p.add_argument('--lr', type=float, default=0.001, help='learning rate')
    p.add_argument('--scheduler_steps', type=int, nargs='+', default=[75, 125], help='the lr is multiplied with 0.1 at these epochs')
    p.add_argument('--momentum', type=float, default=0.9, help='gradient descent momentum')
    p.add_argument('--normal_loss', type=str, default='ms_euclidean', help='unused (kept for compatibility)')
    p.add_argument('--outputs', type=str, nargs='+', default=['imp_surf', 'imp_surf_magnitude', 'imp_surf_sign', 'patch_pts_ids', 'p_index'],
                   help='outputs of the network')
    p.add_argument('--use_point_stn', type=int, default=True, help='use point spatial transformer')
    p.add_argument('--use_feat_stn', type=int, default=True, help='use feature spatial transformer')
    p.add_argument('--sym_op', type=str, default='max', help='symmetry operation')
    p.add_argument('--points_per_patch', type=int, default=50, help='max. number of points per patch')
    p.add_argument('--debug', type=int, default=0, help='set to 1 of you want debug outputs to validate the model')
    return p.parse_args(args=args)


def initial_state_dict(use_point_stn, shared_transformer, net_size=1024, output_dim=2):
    """Parameters initialised exactly like `PointsToSurfModel(...)` under the current torch seed: the reference's module
    constructors create their Conv1d / Linear layers in the order of `arch.layer_specs`, and torch's default initialisers
    draw from the global generator in construction order (source/points_to_surf_model.py:12-36,72-99,134-167,237-294)."""
    sd = {}
    for name, kind, cout, cin in arch.layer_specs(bool(use_point_stn), bool(shared_transformer), net_size, output_dim):
        if kind == 'conv':
            m = torch.nn.Conv1d(cin, cout, 1)
        elif kind == 'fc':
            m = torch.nn.Linear(cin, cout)
        else:
            m = torch.nn.BatchNorm1d(cout)
        for k, v in m.state_dict().items():
            sd[name + '.' + k] = v.detach().clone()
    return sd


def _check_supported(opt):
    outs = list(opt.outputs)
    for o in outs:
        if o not in ('imp_surf', 'imp_surf_magnitude', 'imp_surf_sign', 'p_index', 'patch_pts_ids'):
            raise ValueError('Unknown output: %s' % o)
    arch.head_output_dim(outs)          # the rule of points2surf_b200.eval: every checkpoint written can be evaluated
    if opt.sym_op != 'max':
        raise ValueError('Unsupported symmetric operation: %s' % opt.sym_op)
    if opt.single_transformer:
        raise ValueError('Unsupported option: single_transformer=1')
    if not opt.use_feat_stn:
        raise ValueError('Unsupported option: use_feat_stn=0')
    if opt.fixed_subsample and not opt.uniform_subsample:
        raise ValueError('Unsupported option: fixed_subsample=1 with the distance-weighted sub-sample (only with uniform_subsample=1)')
    if opt.training_order not in ('random', 'random_shape_consecutive'):
        raise ValueError('Unknown training order: %s' % opt.training_order)
    if opt.use_point_stn and not (opt.shared_transformer in (0, 1, False, True)):
        raise ValueError('bad shared_transformer')


class _ShapeSet:
    """Shape names, per-shape query counts and lazily loaded arrays (cloud, query points, signed distances) of one
    `<set>.txt`; the part of PointcloudPatchDataset.__init__ / load_shape the samplers and the batch assembly need
    (source/data_loader.py:16-68,262-318)."""

    def __init__(self, root, list_file, cache_capacity):
        self.root = root
        with open(os.path.join(root, list_file)) as f:
            self.shape_names = list(filter(None, (x.strip() for x in f.readlines())))
        print('getting information for {} shapes'.format(len(self.shape_names)))
        self.shape_patch_count = [int(np.load(os.path.join(root, '05_query_pts', n + '.ply.npy'), mmap_mode='r').shape[0])
                                  for n in self.shape_names]
        self.offsets = np.concatenate([[0], np.cumsum(self.shape_patch_count)])
        self.capacity = max(1, int(cache_capacity))
        self._cache, self._used, self._tick = {}, {}, 0

    def shape_index(self, index):
        si = int(np.searchsorted(self.offsets, index, side='right') - 1)
        return si, int(index - self.offsets[si])

    def get(self, si):
        if si not in self._cache:
            if len(self._cache) >= self.capacity:
                old = min(self._used, key=self._used.get)
                del self._cache[old], self._used[old]
            name = self.shape_names[si]
            pts = np.load(os.path.join(self.root, '04_pts', name + '.xyz.npy'))
            if pts.shape[1] > 3:
                pts = pts[:, 0:3]
            q = np.load(os.path.join(self.root, '05_query_pts', name + '.ply.npy'))
            d = np.load(os.path.join(self.root, '05_query_dist', name + '.ply.npy'))
            self._cache[si] = (np.ascontiguousarray(pts, dtype=np.float32), np.ascontiguousarray(q, dtype=np.float32),
                               np.ascontiguousarray(d, dtype=np.float32).reshape(-1))
        self._used[si] = self._tick
        self._tick += 1
        return self._cache[si]


class GpuAssembler:
    """kNN patch + radius + patch-space normalisation and the global sub-sample of a group of query points of one shape,
    on the device (the call sequence of points2surf_b200.eval._eval_given_queries)."""

    def __init__(self, device, points_per_patch, sub_sample_size, uniform_subsample, seed, patch_radius=0.0, fixed_subsample=False):
        from . import ops
        self.ops, self.device = ops, device
        self.P, self.S, self.uniform, self.seed = points_per_patch, sub_sample_size, bool(uniform_subsample), int(seed)
        self.patch_radius = float(patch_radius)          # > 0: ball-query patches of a fixed radius (radius ablations)
        self.fixed = bool(fixed_subsample)               # --fixed_subsample 1: the same uniform ids for every query of a shape
        self._clouds = {}
        self.calls = 0

    def cloud(self, key, pts):
        if key not in self._clouds:
            if len(self._clouds) > 64:
                self._clouds.clear()
            self._clouds[key] = torch.from_numpy(pts).to(self.device)
        return self._clouds[key]

    def assemble(self, key, pts, query_pts):
        """-> patch [n,P,3] (patch space), radius [n], sub-sample [n,S,3] (model space), query [n,3] device tensors."""
        pts_dev = self.cloud(key, pts)
        q = torch.from_numpy(np.ascontiguousarray(query_pts, dtype=np.float32)).to(self.device)
        self.calls += 1
        if self.patch_radius > 0.0:
            _, patch, radius, _ = self.ops.ball_patch(pts_dev, q, self.P, self.patch_radius, self.seed + self.calls)
        else:
            _, patch, radius = self.ops.knn_patch(pts_dev, q, self.P)
        if self.fixed:
            from .samplers import fixed_uniform_subsample_ids
            ids = torch.from_numpy(fixed_uniform_subsample_ids(pts_dev.shape[0], self.S).astype(np.int64)).to(self.device)
            return patch, radius, pts_dev.index_select(0, ids).unsqueeze(0).expand(q.shape[0], -1, -1).contiguous(), q
        ids = self.ops.subsample(pts_dev, q, self.S, self.uniform, self.seed + self.calls)   # a fresh Philox stream per call
        return patch, radius, self.ops.gather_points(pts_dev, ids), q


def _random_rotations(rng, n):
    from .eval import _random_rotations as rr     # trimesh.transformations.random_rotation_matrix(rng.rand(3)), restated once
    return rr(rng, n)


def _assemble_batch(dataset, indices, assembler, rng, device, dtype=torch.float32):
    """The batch dict PointcloudPatchDataset.__getitem__ + the default collate produce for these global patch indices
    (source/data_loader.py:352-421): keys patch_pts_ps, patch_radius_ms, pts_sub_sample_ms, imp_surf_query_point_ms,
    imp_surf_magnitude_ms, imp_surf_dist_sign_ms, imp_surf_ms, with the per-sample random rotation applied to patch, sub-sample, query."""
    n = len(indices)
    per_shape = {}
    for pos, gi in enumerate(indices):
        si, pi = dataset.shape_index(int(gi))
        per_shape.setdefault(si, []).append((pos, pi))
    order, parts, dist = [], [], np.empty(n, dtype=np.float32)
    for si, items in per_shape.items():
        pts, qpts, qdist = dataset.get(si)
        pis = np.array([pi for _, pi in items], dtype=np.int64)
        parts.append(assembler.assemble((dataset.root, dataset.shape_names[si]), pts, qpts[pis]))
        order.extend(pos for pos, _ in items)
        dist[[pos for pos, _ in items]] = qdist[pis]
    inv = torch.from_numpy(np.argsort(np.asarray(order))).to(device)
    patch = torch.cat([p[0] for p in parts]).index_select(0, inv)
    radius = torch.cat([p[1] for p in parts]).index_select(0, inv)
    sub = torch.cat([p[2] for p in parts]).index_select(0, inv)
    q = torch.cat([p[3] for p in parts]).index_select(0, inv)
    R = torch.from_numpy(_random_rotations(rng, n)).to(device=device, dtype=patch.dtype)      # data_loader.py:381-393
    Rt = R.transpose(1, 2)
    d = torch.from_numpy(dist).to(device)
    batch = {
        'patch_pts_ps': torch.matmul(patch, Rt).contiguous(),
        'patch_radius_ms': radius.contiguous(),
        'pts_sub_sample_ms': torch.matmul(sub, Rt).contiguous(),
        'imp_surf_query_point_ms': torch.matmul(q.unsqueeze(1), Rt).squeeze(1).contiguous(),
        'imp_surf_magnitude_ms': d.abs().contiguous(),
        'imp_surf_dist_sign_ms': (d >= 0).to(patch.dtype).contiguous(),        # 0.0 if sign < 0 else 1.0  (data_loader.py:367-368)
        'imp_surf_ms': d.contiguous(),                                          # the signed distance (data_loader.py:369,402)
    }
    return {k: v.to(dtype) for k, v in batch.items()}


def calc_metrics(pred, batch, fixed_radius=False):
    """abs_dist_rms and the sign-classification scores of source/points_to_surf_train.py:566-598, for the two-output head
    (pred [B,2]: magnitude + sign) and the regression head (pred [B,1]: signed distance).
    The reference's compute_loss divides batch_data['imp_surf_magnitude_ms'] / ['imp_surf_ms'] by the patch radius IN
    PLACE (points_to_surf_train.py:544-555) before calc_metrics reads it, so the logged rmse is against the normalised
    target; for the regression head it also sets the logits to -1 / +1 in place before classifying them (:589-591), which
    gives +1 where pred >= 0 (-0.0 included) and -1 elsewhere (NaN included).  This mirror mutates neither the batch nor
    the logits and applies both rules here."""
    from . import evaluation
    key = 'imp_surf_ms' if pred.shape[1] == 1 else 'imp_surf_magnitude_ms'
    abs_dist = torch.tanh(pred[:, 0]).pow(2)
    target = batch[key] if fixed_radius else batch[key] / batch['patch_radius_ms']
    rms = torch.sqrt(torch.mean((abs_dist.abs() - target.abs()) ** 2))
    inside = torch.where(pred[:, -1] >= 0.0, torch.ones_like(abs_dist), -torch.ones_like(abs_dist))
    out = evaluation.compare_predictions_binary_tensors(ground_truth=batch['imp_surf_dist_sign_ms'], predicted=inside,
                                                        prediction_name='training_metrics')
    out['abs_dist_rms'] = float(rms)
    return out


def _log_line(opt, epoch, batchind, num_batch, prefix, losses, metrics):
    if batchind % opt.debug_interval == 0:
        print('[{name} {epoch}: {batch}/{n_batches}] {prefix} loss: {loss:+.2f}, rmse: {rmse:+.2f}, f1: {f1:+.2f}'.format(
            name=opt.name, epoch=epoch, batch=batchind, n_batches=num_batch - 1, prefix=prefix, loss=sum(float(l) for l in losses),
            rmse=metrics['abs_dist_rms'], f1=metrics['f1_score']))


def _make_sampler(opt, dataset):
    if opt.training_order == 'random':
        return samplers.RandomPointcloudPatchSampler(dataset, patches_per_shape=opt.patches_per_shape, seed=opt.seed,
                                                     identical_epochs=opt.identical_epochs)
    return samplers.SequentialShapeRandomPointcloudPatchSampler(dataset, patches_per_shape=opt.patches_per_shape, seed=opt.seed,
                                                                identical_epochs=opt.identical_epochs)


def _batches(sampler, batch_size):
    idx = list(iter(sampler))
    return [idx[i:i + batch_size] for i in range(0, len(idx), batch_size)]      # DataLoader default: keep the last partial batch


def _prefixed(sd):
    return {'module.' + k: v.detach().cpu() for k, v in sd.items()}


def points_to_surf_train(opt, prims=None, assembler=None, device=None, dtype=torch.float32):
    """Train like source/points_to_surf_train.py:165-535.  `prims` / `assembler` / `device` / `dtype` exist for the
    CPU tests of the host logic; the product path leaves them at their defaults (CUDA primitives, GPU assembly)."""
    _check_supported(opt)
    # data parallelism: one process per GPU (torchrun); each rank trains on its slice of every batch, gradients are
    # averaged by TrainStep's all_reduce, BatchNorm statistics stay per rank like the reference's nn.DataParallel replicas
    # (points_to_surf_train.py:412-413).  Rank 0 alone prompts, logs and writes files.
    rank, world = 0, 1
    if torch.distributed.is_available() and torch.distributed.is_initialized():
        rank, world = torch.distributed.get_rank(), torch.distributed.get_world_size()
    if device is None:
        if not torch.cuda.is_available() or opt.gpu_idx[0] < 0:
            raise RuntimeError('points2surf_b200 needs a CUDA device (--gpu_idx >= 0): there is no CPU fallback')
        if world > 1:
            device = torch.device('cuda', int(os.environ.get('LOCAL_RANK', 0)))
        else:
            if len(opt.gpu_idx) > 1:
                raise ValueError('--gpu_idx lists %d devices: multi-GPU training runs one process per GPU here '
                                 '(python -m torch.distributed.run --nproc-per-node N ...), not nn.DataParallel threads' % len(opt.gpu_idx))
            device = torch.device('cuda', opt.gpu_idx[0])
        torch.cuda.set_device(device)
    is_main = rank == 0
    print('Training on %d devices:\n  %s' % (world, str(device)))

    log_dirname = os.path.join(opt.logdir, opt.name)
    params_filename = os.path.join(opt.outdir, '%s_params.pth' % opt.name)
    model_filename = os.path.join(opt.outdir, '%s_model.pth' % opt.name)
    desc_filename = os.path.join(opt.outdir, '%s_description.txt' % opt.name)
    if is_main and (os.path.exists(log_dirname) or os.path.exists(model_filename)):
        if opt.name != 'test':
            response = input('A training run named "{}" already exists, overwrite? (y/n) '.format(opt.name))
            if response != 'y':
                return
        if os.path.exists(log_dirname):
            try:
                shutil.rmtree(log_dirname)
            except OSError:
                print("Can't delete " + log_dirname)

    output_dim = arch.head_output_dim(opt.outputs)       # points_to_surf_train.py:200-240: pred_dim and the loss weights
    output_names = [o for o in opt.outputs if o in ('imp_surf', 'imp_surf_magnitude', 'imp_surf_sign')]
    output_loss_weights = {o: 1.0 for o in output_names}

    if opt.seed < 0:
        opt.seed = random.randint(1, 10000)
    print('Random Seed: %d' % opt.seed)
    random.seed(opt.seed)
    torch.manual_seed(opt.seed)

    start_epoch = 0
    if opt.refine != '':
        print(f'Refining weights from {opt.refine}')
        from .weights import strip_module_prefix
        state = strip_module_prefix(torch.load(opt.refine, map_location='cpu'))
        try:    # a file name like 'vanilla_model_50.pth'
            start_epoch = int(str(opt.refine)[str(opt.refine).rfind('_') + 1:str(opt.refine).rfind('.')]) + 1
            print(f'Continuing training from epoch {start_epoch}')
        except ValueError:
            print(f'Warning: {opt.refine} has no epoch in the name. The log will continue at epoch 0 and might be messed up!')
    else:
        state = initial_state_dict(opt.use_point_stn, opt.shared_transformer, opt.net_size, output_dim)

    train_set = _ShapeSet(opt.indir, opt.trainset, opt.cache_capacity)
    test_set = _ShapeSet(opt.indir, opt.testset, opt.cache_capacity)
    train_sampler, test_sampler = _make_sampler(opt, train_set), _make_sampler(opt, test_set)
    opt.train_shapes, opt.test_shapes = train_set.shape_names, test_set.shape_names
    n_train_batches = math.ceil(len(train_sampler) / opt.batchSize)
    n_test_batches = math.ceil(len(test_sampler) / opt.batchSize)
    print('Training set: {} patches (in {} batches) | Test set: {} patches (in {} batches)'.format(
        len(train_sampler), n_train_batches, len(test_sampler), n_test_batches))
    os.makedirs(opt.outdir, exist_ok=True)

    writer = None
    if is_main:
        try:
            from torch.utils.tensorboard import SummaryWriter
            writer = SummaryWriter(log_dirname, comment=opt.name)
            writer.add_scalar('LR', opt.lr, 0)
        except Exception:       # tensorboard is optional here
            writer = None

    ts = TrainStep({k: v.to(device) for k, v in state.items()}, opt.use_point_stn, opt.shared_transformer,
                   points_per_patch=opt.points_per_patch, sub_sample_size=opt.sub_sample_size, net_size=opt.net_size, lr=opt.lr,
                   momentum=opt.momentum, device=device, prims=prims, outputs=tuple(output_names),
                   output_loss_weights=output_loss_weights, fixed_radius=opt.patch_radius > 0.0, dtype=dtype)
    if assembler is None:
        assembler = GpuAssembler(device, opt.points_per_patch, opt.sub_sample_size, opt.uniform_subsample, opt.seed + rank,
                                 patch_radius=opt.patch_radius, fixed_subsample=opt.fixed_subsample)
    rng_aug = np.random.RandomState(opt.seed + rank)            # augmentation / sub-sample streams differ per rank

    if is_main:
        torch.save(opt, params_filename)
        with open(desc_filename, 'w+') as text_file:
            print(opt.desc, file=text_file)

    green = lambda x: '\033[92m' + x + '\033[0m'
    blue = lambda x: '\033[94m' + x + '\033[0m'
    # the reference builds a fresh MultiStepLR after a --refine resume (points_to_surf_train.py:406-410): milestones count
    # scheduler steps since the (re)start, the first epoch always runs at opt.lr
    lr = opt.lr
    history = []
    for epoch in range(start_epoch, opt.nepoch):
        # every rank draws the same index sequence (same sampler seed) and takes its slice of each batch
        train_batches = [b[rank::world] for b in _batches(train_sampler, opt.batchSize)]
        test_batches = [b[rank::world] for b in _batches(test_sampler, opt.batchSize)]
        if world > 1 and any(len(b) == 0 for b in train_batches + test_batches):
            raise ValueError('batchSize %d leaves a rank without queries in the last batch: use a batch size that is a '
                             'multiple of the world size %d' % (opt.batchSize, world))
        test_batchind, test_fraction_done = -1, 0.0
        for train_batchind, indices in enumerate(train_batches):
            batch = _assemble_batch(train_set, indices, assembler, rng_aug, device, dtype)
            ts.lr = lr
            losses = ts.step(batch)                                   # train(): zero_grad, forward, loss, backward, SGD
            train_fraction_done = (train_batchind + 1) / len(train_batches)
            metrics = calc_metrics(ts.last_logits, batch, fixed_radius=opt.patch_radius > 0.0)
            _log_line(opt, epoch, train_batchind, len(train_batches), green('train'), losses, metrics)
            step = (epoch + train_fraction_done) * len(train_batches) * opt.batchSize
            if writer is not None:
                writer.add_scalar('loss/train/total', sum(float(l) for l in losses), step)
            history.append(('train', epoch, train_batchind, [float(l) for l in losses]))
            while test_fraction_done <= train_fraction_done and test_batchind + 1 < len(test_batches):
                test_batchind += 1
                tb = _assemble_batch(test_set, test_batches[test_batchind], assembler, rng_aug, device, dtype)
                pred, tl = ts.evaluate(tb)                            # eval(): running statistics, no gradients
                tm = calc_metrics(pred, tb, fixed_radius=opt.patch_radius > 0.0)
                test_fraction_done = (test_batchind + 1) / len(test_batches)
                _log_line(opt, epoch, test_batchind, len(train_batches), blue('test'), tl, tm)
                if writer is not None:
                    writer.add_scalar('loss/eval/total', sum(float(l) for l in tl), step)
                history.append(('test', epoch, test_batchind, [float(l) for l in tl]))

        if is_main and (epoch % opt.save_interval == 0 or epoch == opt.nepoch - 1):
            torch.save(_prefixed(ts.state_dict()), model_filename)
        if is_main and (epoch % (5 * 10 ** math.floor(math.log10(max(2, epoch - 1)))) == 0 or epoch % 100 == 0 or epoch == opt.nepoch - 1):
            torch.save(_prefixed(ts.state_dict()), os.path.join(opt.outdir, '%s_model_%d.pth' % (opt.name, epoch)))

        # MultiStepLR(milestones=scheduler_steps, gamma=0.1), stepped once per epoch (points_to_surf_train.py:519-529)
        new_lr = opt.lr * (0.1 ** sum(1 for m in opt.scheduler_steps if epoch - start_epoch + 1 >= m))
        if new_lr != lr:
            print('LR changed from {} to {} in epoch {}'.format(lr, new_lr, epoch))
        lr = new_lr
        if writer is not None:
            writer.add_scalar('LR', lr, (epoch + 1) * len(train_batches) * opt.batchSize - 1)
            writer.flush()
    if writer is not None:
        writer.close()
    return history


if __name__ == '__main__':
    points_to_surf_train(parse_arguments())
