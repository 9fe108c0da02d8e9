"""TEST INFRASTRUCTURE ONLY -- the shared-encoder ablation (single_transformer=1, experiments/*_p2s_shared_encoder.sh)
restated on top of oracle/p2s_oracle.py and oracle/net_bound.py, whose building blocks it reuses unchanged.

  model_forward   PointsToSurfModel.forward in eval mode with single_transformer=1, use_point_stn=1
                  (source/points_to_surf_model.py:253-263,296-352): x = cat(patch, shape - q) (:303,321), one PointNetfeat
                  `feat_local_global` with its own QSTN over all P + S points (:177-234), fc1_local_global + bn + ReLU
                  (:323), then fc2, fc3, fc4.  Pinned against the unmodified reference by
                  tests/golden/make_shared_encoder_golden.py.
  fold_params,    the float64 model with a per-element error bound of oracle/net_bound.py for this network: the same
  network         rules, applied to the one encoder over the concatenated points (the engine centres the sub-sample and
                  applies R in fp32 like the vanilla network's shared QSTN, which net_bound bounds the same way).
"""
import numpy as np
import torch

from oracle import net_bound as nb
from oracle import p2s_oracle as orc
from points2surf_b200 import weights as _weights

ENC = 'feat_local_global.'


def _forward_impl(sd, patch_pts_ps, pts_sub_sample_ms, imp_surf_query_point_ms, return_aux):
    as_t = lambda a: a.clone() if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))
    patch = as_t(patch_pts_ps).float().transpose(1, 2)
    shape = as_t(pts_sub_sample_ms).float().transpose(1, 2)
    q = as_t(imp_surf_query_point_ms).float().unsqueeze(2)
    shape = shape - q.expand(shape.shape)                                   # :303
    x = torch.cat((patch, shape), dim=2)                                    # :321
    feat, trans = orc._pointnetfeat(sd, ENC, x, True)                       # :322
    aux = {'trans': trans.numpy(), 'feat_max': feat.numpy()}
    x = orc._fc_bn(sd, feat, 'fc1_local_global', 'bn1_local_global')       # :323
    x = orc._fc_bn(sd, x, 'fc2', 'bn2')                                     # :348
    x = orc._fc_bn(sd, x, 'fc3', 'bn3')
    aux['fc3_out'] = x.numpy()
    out = orc._fc_bn(sd, x, 'fc4', None, relu=False).numpy()
    return (out, aux) if return_aux else out


def model_forward(sd, patch_pts_ps, pts_sub_sample_ms, imp_surf_query_point_ms, return_aux=False):
    """The shared-encoder network in eval mode.  `sd` without the 'module.' prefix; [B,P,3], [B,S,3], [B,3] float32 in;
    -> logits [B, output_dim] float32 (numpy), and with return_aux the dict of 'trans' [B,3,3], 'feat_max' [B,1024]
    (max feature incl. the conv3 bias) and 'fc3_out' [B,128]."""
    with torch.no_grad():
        return _forward_impl(sd, patch_pts_ps, pts_sub_sample_ms, imp_surf_query_point_ms, return_aux)


def fold_params(sd):
    """name -> (W [N, K], b [N]) float64 tensors holding the float32 folded parameters the engine receives."""
    sd = _weights.strip_module_prefix(sd)
    names = []
    for stn in (ENC + 'stn1.', ENC + 'stn2.'):
        names += [(stn + c, stn + bn) for c, bn in (('conv1', 'bn1'), ('conv2', 'bn2'), ('conv3', 'bn3'), ('fc1', 'bn4'),
                                                     ('fc2', 'bn5'))]
        names.append((stn + 'fc3', None))
    names += [(ENC + c, ENC + bn) for c, bn in (('conv0a', 'bn0a'), ('conv0b', 'bn0b'), ('conv1', 'bn1'), ('conv2', 'bn2'),
                                                ('conv3', 'bn3'))]
    names += [('fc1_local_global', 'bn1_local_global'), ('fc2', 'bn2'), ('fc3', 'bn3'), ('fc4', None)]
    out = {}
    for layer, bn in names:
        w, b = _weights.fold(sd, layer, bn)
        out[layer] = (torch.from_numpy(w.astype(np.float64)).reshape(b.size, -1), torch.from_numpy(b.astype(np.float64)))
    return out


def network(P, patch, sub, query, model, R=None):
    """Float64 forward of the shared-encoder network with its bound under `model` ('fp32', 'tc', 'tc_precise'; see
    oracle/net_bound.py).  P: `fold_params(...)` on the inputs' device; R [B,3,3] (optional): the engine's rotation, used
    for everything downstream of the quaternion.  -> dict of nb.V: 'q4', 'feat_max', 'logits'; 'R' = (float64 R, bound)."""
    m = nb.MODELS[model]
    patch, sub, query = patch.double(), sub.double(), query.double()
    pts = torch.cat([patch, sub - query.unsqueeze(1)], 1)
    q4 = nb._qstn(P, ENC + 'stn1.', pts, None, m)
    out = {'q4': q4, 'R': nb._rotation(q4)}
    Rq = out['R'][0] if R is None else R.double()
    f = nb._feat(P, ENC, pts, None, Rq, model)
    out['feat_max'] = f
    h = nb._linear(f, *P['fc1_local_global'], m['fc']).relu()
    h = nb._linear(h, *P['fc2'], m['fc']).relu()
    h = nb._linear(h, *P['fc3'], m['fc']).relu()
    out['logits'] = nb._linear(h, *P['fc4'], nb.FP32_FC)
    return out
