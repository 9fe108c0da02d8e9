"""Fold eval-mode BatchNorm into the preceding Conv1d / Linear and pack the blob the C ABI expects
(layout documented in include/p2s_b200.h).  Layer names follow source/points_to_surf_model.py."""
import numpy as np

BN_EPS = 1e-5  # nn.BatchNorm1d default, used everywhere in the reference (e.g. points_to_surf_model.py:31-35)


def _np(v):
    return v.detach().cpu().numpy() if hasattr(v, 'detach') else np.asarray(v)


def strip_module_prefix(sd):
    """The reference saves the DataParallel wrapper's state_dict (points_to_surf_train.py:513)."""
    return {(k[7:] if k.startswith('module.') else k): v for k, v in sd.items()}


def fold(sd, layer, bn=None):
    w = _np(sd[layer + '.weight']).astype(np.float64)
    if w.ndim == 3:
        w = w[:, :, 0]
    b = _np(sd[layer + '.bias']).astype(np.float64)
    if bn is not None:
        g = _np(sd[bn + '.weight']).astype(np.float64)
        beta = _np(sd[bn + '.bias']).astype(np.float64)
        mu = _np(sd[bn + '.running_mean']).astype(np.float64)
        var = _np(sd[bn + '.running_var']).astype(np.float64)
        s = g / np.sqrt(var + BN_EPS)
        w = w * s[:, None]
        b = (b - mu) * s + beta
    return [w.astype(np.float32).ravel(), b.astype(np.float32).ravel()]


def _stn(sd, p):
    out = []
    for conv, bn in (('conv1', 'bn1'), ('conv2', 'bn2'), ('conv3', 'bn3'), ('fc1', 'bn4'), ('fc2', 'bn5')):
        out += fold(sd, p + conv, p + bn)
    out += fold(sd, p + 'fc3', None)
    return out


def _feat(sd, p, qstn):
    out = []
    if qstn:
        out += _stn(sd, p + 'stn1.')
    out += _stn(sd, p + 'stn2.')
    for conv, bn in (('conv0a', 'bn0a'), ('conv0b', 'bn0b'), ('conv1', 'bn1'), ('conv2', 'bn2'), ('conv3', 'bn3')):
        out += fold(sd, p + conv, p + bn)
    return out


def pack_blob(state_dict, use_point_stn, shared_transformer, output_dim=2, single_transformer=False):
    """output_dim: 2 for the (imp_surf_magnitude, imp_surf_sign) head, 1 for the regression head (imp_surf).
    single_transformer: the shared-encoder ablation (one `feat_local_global` with its own QSTN, `fc1_local_global`
    1024 -> 1024); it needs use_point_stn and no shared_transformer, like the published checkpoints."""
    sd = strip_module_prefix(state_dict)
    if output_dim not in (1, 2):
        raise ValueError('Unsupported output_dim %r: 1 (imp_surf) or 2 (imp_surf_magnitude, imp_surf_sign)' % (output_dim,))
    fc4 = tuple(_np(sd['fc4.weight']).shape)
    if fc4[0] != output_dim:
        raise ValueError('fc4 has %d outputs, expected output_dim %d' % (fc4[0], output_dim))
    parts = []
    if single_transformer:
        if not use_point_stn or shared_transformer:
            raise ValueError('Unsupported option: single_transformer=1 needs use_point_stn=1 and shared_transformer=0')
        parts += _feat(sd, 'feat_local_global.', True)
        parts += fold(sd, 'fc1_local_global', 'bn1_local_global')
    else:
        if use_point_stn and shared_transformer:
            parts += _stn(sd, 'point_stn.')
        parts += _feat(sd, 'feat_local.', False)
        parts += _feat(sd, 'feat_global.', bool(use_point_stn and not shared_transformer))
        parts += fold(sd, 'fc1_local', 'bn1_local') + fold(sd, 'fc1_global', 'bn1_global')
    parts += fold(sd, 'fc2', 'bn2') + fold(sd, 'fc3', 'bn3') + fold(sd, 'fc4', None)
    return np.ascontiguousarray(np.concatenate(parts), dtype=np.float32)
