"""Generate the regression-ablation fixtures (outputs imp_surf, experiments/{train,eval}_p2s_regression.sh).

Run in the build container only (imports the UNMODIFIED reference through oracle/ref_shims.py):
    python tests/golden/make_regression_golden.py [fit] [golden]

1. `fit`: the regression head's last layer (fc4: 1 x 128 + 1) of the synthetic checkpoint
   `synth.make_state_dict('regression', MODEL_SEED)` is fitted by ridge regression on the fp32 oracle's fc3 activations
   of 1024 queries around a 10k-point sphere (weighted sub-sample, like the ablation's training), against
   l* = sign(d) atanh(sqrt(min(|d| / r, 0.999))), d the sphere's analytic signed distance (+ inside), r the query's kNN
   patch radius -- the inverse of the post-process d = tanh(l)^2 sign(l) r.  The recipe of make_e2e_golden.py's `fit`.
   Written to points2surf_b200/fitted_fc4_regression.json (a checkpoint piece, as text: float32 values written so that
   they read back exactly) with the held-out sign accuracy.
2. `golden`: PointsToSurfModel(output_dim=1, use_point_stn=1, shared_transformation=0) of the reference on the fitted
   checkpoint with its fc4 bias re-centred on the inputs (so the logits have mixed signs), then the reference's
   points_to_surf_eval.post_process with the regression outputs, with per-query radii and in the fixed-radius case.
   Asserted equal to the oracle (network: oracle/p2s_oracle.py, post-process: tests/regression_oracle.py) in the same
   run; written to tests/golden/regression.npz.
"""
import argparse
import json
import os
import sys
import warnings

import numpy as np

warnings.filterwarnings('ignore')
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_shims  # noqa: E402
ref_shims.install()
import torch  # noqa: E402
from oracle import p2s_oracle as orc  # noqa: E402
from points2surf_b200 import synth  # noqa: E402
sys.path.insert(0, os.path.dirname(HERE))
import regression_oracle as rorc  # noqa: E402

torch.set_grad_enabled(False)
VARIANT = 'regression'
MODEL_SEED = 10
INPUT_SEED = 110
BATCH = 32
OUTPUTS = ['imp_surf', 'patch_pts_ids', 'p_index']


def fit():
    v = synth.VARIANTS[VARIANT]
    cloud = synth.make_cloud('sphere', 10000, seed=0)
    kd = orc.make_kdtree(cloud)
    sd = synth.make_state_dict(VARIANT, MODEL_SEED)
    rng = np.random.RandomState(100 + MODEL_SEED)
    n = 1024
    dirs = rng.standard_normal((n, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    q = (dirs * (0.5 + rng.uniform(-0.06, 0.06, n))[:, None]).astype(np.float32)
    d = 0.5 - np.linalg.norm(q.astype(np.float64), axis=1)          # + inside (reference convention, sdf.py:204)
    rs = np.random.RandomState(200 + MODEL_SEED)
    items = [orc.assemble_query(cloud, kd, q[i], 300, 1000, rs, bool(v['uniform_subsample'])) for i in range(n)]
    r = np.array([it['patch_radius_ms'] for it in items], np.float64)
    feats = []
    for b in range(0, n, 128):
        _, aux = orc.model_forward(sd, np.stack([it['patch_pts_ps'] for it in items[b:b + 128]]),
                                   np.stack([it['pts_sub_sample_ms'] for it in items[b:b + 128]]), q[b:b + 128],
                                   v['use_point_stn'], v['shared_transformer'], return_aux=True)
        feats.append(aux['fc3_out'])
    F = np.concatenate(feats).astype(np.float64)
    A = np.concatenate([F, np.ones((n, 1))], 1)
    target = np.sign(d) * np.arctanh(np.sqrt(np.minimum(np.abs(d) / r, 0.999)))
    ntr = 896
    W = np.linalg.solve(A[:ntr].T @ A[:ntr] + 0.1 * np.eye(129), A[:ntr].T @ target[:ntr])
    pred = A @ W
    acc = ((pred[ntr:] >= 0) == (d[ntr:] >= 0)).mean()
    print('fit regression: held-out sign accuracy %.3f (%d queries), train %.3f'
          % (acc, n - ntr, ((pred[:ntr] >= 0) == (d[:ntr] >= 0)).mean()))
    doc = {'variant': VARIANT, 'seed': MODEL_SEED, 'heldout_sign_accuracy': float(acc),
           'weight': [[float(x) for x in W[:128].astype(np.float32)]], 'bias': [float(x) for x in W[128:].astype(np.float32)]}
    with open(synth.FITTED_FC4_REGRESSION, 'w') as fp:
        json.dump(doc, fp, indent=1)
        fp.write('\n')
    print('written', synth.FITTED_FC4_REGRESSION)


def golden():
    from source.points_to_surf_model import PointsToSurfModel
    from source import points_to_surf_eval as ref_eval
    v = synth.VARIANTS[VARIANT]
    inp = synth.make_model_inputs(BATCH, seed=INPUT_SEED)

    def ref_logits(sd):
        m = PointsToSurfModel(net_size_max=1024, num_points=300, output_dim=1, use_point_stn=v['use_point_stn'],
                              use_feat_stn=1, sym_op='max', use_query_point=True, sub_sample_size=1000,
                              do_augmentation=False, single_transformer=0, shared_transformation=v['shared_transformer'])
        m.load_state_dict(sd)
        m.eval()
        x = {k: torch.from_numpy(a.copy()) for k, a in inp.items()}
        return m(x).numpy()

    sd = synth.make_state_dict(VARIANT, MODEL_SEED, fitted=True)
    # the fitted head is one-signed on these (non-surface) inputs: re-centre its bias on them so both signs occur
    fc4_bias = (sd['fc4.bias'].numpy() - np.median(ref_logits(sd), axis=0)).astype(np.float32)
    sd['fc4.bias'] = torch.from_numpy(fc4_bias)
    logits = ref_logits(sd)
    assert logits.shape == (BATCH, 1)
    o = orc.model_forward(sd, inp['patch_pts_ps'], inp['pts_sub_sample_ms'], inp['imp_surf_query_point_ms'],
                          v['use_point_stn'], v['shared_transformer'])
    err = float(np.abs(o - logits).max())
    assert err < 1e-4, err

    train_opt = argparse.Namespace(outputs=OUTPUTS)
    output_ids = ref_eval.get_output_ids(train_opt)
    pred_dim, output_pred_ind = ref_eval.get_output_dimensions(train_opt)
    assert pred_dim == 1
    radius = np.linspace(0.02, 0.3, BATCH).astype(np.float32)
    out = {}
    for key, fixed in (('sdf', False), ('sdf_fixed_radius', True)):
        pred = torch.from_numpy(logits.copy())
        ref_eval.post_process(pred, train_opt, output_ids, output_pred_ind, torch.from_numpy(radius), fixed)
        ref = pred[:, 0].numpy().copy()
        ref[np.isnan(ref)] = 1.0                                    # save_reconstruction_data, :205-207
        assert np.array_equal(rorc.post_process_distance(logits, None if fixed else radius), ref), key
        out[key] = ref
    print('golden regression: oracle-vs-reference max abs logit err %.3g, positive fraction %.2f, |l| range [%.3g, %.3g]'
          % (err, (logits > 0).mean(), np.abs(logits).min(), np.abs(logits).max()))
    np.savez_compressed(os.path.join(HERE, 'regression.npz'), model_seed=MODEL_SEED, input_seed=INPUT_SEED, batch=BATCH,
                        fc4_bias=fc4_bias, logits=logits, radius=radius, **out,
                        input_checksum=np.float64(sum(float(np.abs(a).sum()) for a in inp.values())))


if __name__ == '__main__':
    stages = sys.argv[1:] or ['fit', 'golden']
    if 'fit' in stages:
        fit()
    if 'golden' in stages:
        golden()
