"""Synthetic inputs for tests and benchmarks: point clouds of the sizes BASELINE.json
names and rand-init-but-non-trivial checkpoints (there is no network, so the
pre-trained weights of models/download_models_*.py are unavailable).

The checkpoint factory is deliberately *not* PyTorch-default init: SURVEY.md section 4
shows that default init gives input-independent logits and identity BatchNorm,
which would make every parity test vacuous.  Weights are He-scaled and the BN
affine parameters / running statistics are randomised, all from a NumPy legacy
RandomState so that the same seed gives the same checkpoint on any box.
"""
import argparse
import json
import os
from collections import OrderedDict

import numpy as np

VARIANTS = {
    # (use_point_stn, shared_transformer, uniform_subsample)  -- experiments/train_p2s_*.sh
    'vanilla': dict(use_point_stn=1, shared_transformer=1, uniform_subsample=0),
    'max': dict(use_point_stn=0, shared_transformer=0, uniform_subsample=1),
    'uniform': dict(use_point_stn=1, shared_transformer=0, uniform_subsample=1),
    # experiments/train_p2s_regression.sh: the per-branch QSTN network with the distance-weighted sub-sample and the
    # regression head (outputs imp_surf patch_pts_ids p_index: fc4 128 -> 1)
    'regression': dict(use_point_stn=1, shared_transformer=0, uniform_subsample=0, output_dim=1),
    # experiments/train_p2s_shared_encoder.sh: one encoder (feat_local_global, its own QSTN) over patch + sub-sample
    'shared_encoder': dict(use_point_stn=1, shared_transformer=0, uniform_subsample=0, single_transformer=1),
}


def make_train_opt(variant='vanilla', points_per_patch=300, sub_sample_size=1000, net_size=1024):
    """The pickled argparse.Namespace the reference stores as <model>_params.pth
    (source/points_to_surf_train.py:420) restricted to the fields eval reads
    (source/points_to_surf_eval.py:110-166,316-328)."""
    v = VARIANTS[variant]
    return argparse.Namespace(
        name='p2s_' + variant, net_size=net_size, points_per_patch=points_per_patch,
        sub_sample_size=sub_sample_size, patch_radius=0.0, patch_center='mean',
        use_point_stn=v['use_point_stn'], use_feat_stn=1, sym_op='max',
        single_transformer=v.get('single_transformer', 0), shared_transformer=v['shared_transformer'],
        uniform_subsample=v['uniform_subsample'], fixed_subsample=0,
        outputs=(['imp_surf'] if v.get('output_dim', 2) == 1 else ['imp_surf_magnitude', 'imp_surf_sign']) +
                ['patch_pts_ids', 'p_index'],
        batchSize=501, seed=3627473)


def _layer_specs(variant, net=1024):
    from .arch import layer_specs
    v = VARIANTS[variant]
    return layer_specs(v['use_point_stn'], v['shared_transformer'], net, v.get('output_dim', 2),
                       bool(v.get('single_transformer', 0)))


def make_state_dict_numpy(variant='vanilla', seed=0, net=1024, module_prefix=''):
    """OrderedDict name -> np.ndarray with the reference's names and shapes
    (Conv1d weights are [Cout, Cin, 1]); `module_prefix='module.'` gives the
    DataParallel-wrapped form the reference saves (points_to_surf_train.py:513)."""
    rng = np.random.RandomState(seed)
    sd = OrderedDict()
    for name, kind, cout, cin in _layer_specs(variant, net):
        p = module_prefix + name
        if kind in ('conv', 'fc'):
            gain = np.sqrt(2.0 / cin)
            if name.endswith('stn2.fc3') or name.endswith('stn1.fc3') or name.endswith('point_stn.fc3'):
                gain *= 0.25  # keep the predicted transforms near identity, like a trained net
            w = (rng.standard_normal((cout, cin)) * gain).astype(np.float32)
            sd[p + '.weight'] = w[:, :, None] if kind == 'conv' else w
            sd[p + '.bias'] = (rng.standard_normal(cout) * 0.1).astype(np.float32)
        else:
            sd[p + '.weight'] = rng.uniform(0.6, 1.4, cout).astype(np.float32)
            sd[p + '.bias'] = (rng.standard_normal(cout) * 0.1).astype(np.float32)
            sd[p + '.running_mean'] = (rng.standard_normal(cout) * 0.2).astype(np.float32)
            sd[p + '.running_var'] = rng.uniform(0.5, 1.5, cout).astype(np.float32)
            sd[p + '.num_batches_tracked'] = np.array(100, dtype=np.int64)
    return sd


FITTED_FC4 = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'fitted_fc4.npz')
# the regression head's fitted fc4 [1,128] (tests/golden/make_regression_golden.py fit), as text: every value is written
# with enough digits to give back the same float32
FITTED_FC4_REGRESSION = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'fitted_fc4_regression.json')
# the shared encoder's fitted fc4 [2,128] (tests/golden/make_shared_encoder_golden.py fit), as text like the regression head
FITTED_FC4_SHARED_ENCODER = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'fitted_fc4_shared_encoder.json')
_FITTED_FC4_JSON = {'regression': FITTED_FC4_REGRESSION, 'shared_encoder': FITTED_FC4_SHARED_ENCODER}


def fitted_fc4(variant, seed):
    """Last layer (fc4 weight [output_dim,128], bias [output_dim]) fitted on a 10k-point sphere so that the otherwise
    rand-init checkpoint `make_state_dict(variant, seed)` produces a surface-like SDF (tests/golden/make_e2e_golden.py
    and, for 'regression' and 'shared_encoder', tests/golden/make_regression_golden.py and
    tests/golden/make_shared_encoder_golden.py: ridge regression on the fc3 activations against the analytic signed
    distance; everything in front of fc4 stays random).
    Only the (variant, seed) pairs the files were fitted for are available."""
    if variant in _FITTED_FC4_JSON:
        path = _FITTED_FC4_JSON[variant]
        with open(path) as fp:
            f = json.load(fp)
        if int(f['seed']) != int(seed):
            raise ValueError('no fitted fc4 for (%s, seed %d) in %s' % (variant, seed, path))
        return np.array(f['weight'], np.float32), np.array(f['bias'], np.float32)
    f = np.load(FITTED_FC4)
    if variant + '_seed' not in f or int(f[variant + '_seed']) != int(seed):
        raise ValueError('no fitted fc4 for (%s, seed %d) in %s' % (variant, seed, FITTED_FC4))
    return f[variant + '_weight'].copy(), f[variant + '_bias'].copy()


def make_state_dict(variant='vanilla', seed=0, net=1024, module_prefix='', fitted=False):
    import torch
    sd = OrderedDict((k, torch.from_numpy(v.copy())) for k, v in
                     make_state_dict_numpy(variant, seed, net, module_prefix).items())
    if fitted:
        w, b = fitted_fc4(variant, seed)
        sd[module_prefix + 'fc4.weight'] = torch.from_numpy(w)
        sd[module_prefix + 'fc4.bias'] = torch.from_numpy(b)
    return sd


def make_cloud(kind='sphere', n=10000, seed=0, noise=0.005):
    """Synthetic clouds of SURVEY.md section 8(d): surface samples in [-1,1)^3, float32."""
    rng = np.random.RandomState(seed)
    if kind == 'sphere':
        d = rng.standard_normal((n, 3))
        p = 0.5 * d / np.linalg.norm(d, axis=1, keepdims=True)
    elif kind == 'torus':
        u, v = rng.uniform(0, 2 * np.pi, n), rng.uniform(0, 2 * np.pi, n)
        R, r = 0.45, 0.18
        p = np.stack([(R + r * np.cos(v)) * np.cos(u), (R + r * np.cos(v)) * np.sin(u), r * np.sin(v)], 1)
    elif kind == 'box':
        p = rng.uniform(-0.45, 0.45, (n, 3))
        ax = rng.randint(0, 3, n)
        sg = rng.randint(0, 2, n) * 2 - 1
        p[np.arange(n), ax] = 0.45 * sg
    else:
        raise ValueError('unknown cloud kind: %s' % kind)
    p = p + rng.standard_normal((n, 3)) * noise
    return np.clip(p, -0.999, 0.999).astype(np.float32)


def make_model_inputs(batch, points_per_patch=300, sub_sample_size=1000, seed=0):
    """Model-boundary inputs shaped like PointcloudPatchDataset.__getitem__ output
    (source/data_loader.py:395-402): patch in patch space (max norm 1), sub-sample and
    query in model space."""
    rng = np.random.RandomState(seed)
    patch = rng.uniform(-1, 1, (batch, points_per_patch, 3))
    patch /= np.linalg.norm(patch, axis=2).max(axis=1)[:, None, None]
    sub = rng.uniform(-0.8, 0.8, (batch, sub_sample_size, 3))
    q = rng.uniform(-0.5, 0.5, (batch, 3))
    return dict(patch_pts_ps=patch.astype(np.float32), pts_sub_sample_ms=sub.astype(np.float32),
                imp_surf_query_point_ms=q.astype(np.float32))
