"""Generate the shared-encoder ablation fixtures (single_transformer=1, experiments/{train,eval}_p2s_shared_encoder.sh).

Run in the build container only (imports the UNMODIFIED reference through oracle/ref_shims.py):
    python tests/golden/make_shared_encoder_golden.py [fit] [golden]

1. `fit`: the last layer (fc4: 2 x 128 + 2) of the synthetic checkpoint `synth.make_state_dict('shared_encoder',
   MODEL_SEED)` is fitted by ridge regression on the fp32 oracle's fc3 activations (tests/shared_encoder_oracle.py) of
   1024 queries around a 10k-point sphere (weighted sub-sample, like the ablation's training), against the targets of
   make_e2e_golden.py's `fit`: the sign logit towards sign(d) min(|d| / 0.01, 3), the magnitude logit towards
   atanh(sqrt(min(|d| / r, 0.98))), d the sphere's analytic signed distance (+ inside), r the query's kNN patch radius.
   Written to points2surf_b200/fitted_fc4_shared_encoder.json (a checkpoint piece, as text: float32 values written so
   that they read back exactly) with the held-out sign accuracy.
2. `golden`: PointsToSurfModel(single_transformer=1, use_point_stn=1, shared_transformation=0, output_dim=2,
   num_points=300, sub_sample_size=1000) of the reference on the fitted checkpoint with its fc4 bias re-centred on the
   inputs (so both logits have mixed signs), with the rotation and the max feature taken from its `feat_local_global`.
   Asserted equal to the oracle in the same run; written to tests/golden/shared_encoder.npz together with the
   reference's state_dict key order.
"""
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
import shared_encoder_oracle as sorc  # noqa: E402

torch.set_grad_enabled(False)
VARIANT = 'shared_encoder'
MODEL_SEED = 12
INPUT_SEED = 112
BATCH = 32


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
        _, aux = sorc.model_forward(sd, np.stack([it['patch_pts_ps'] for it in items[b:b + 128]]),
                                    np.stack([it['pts_sub_sample_ms'] for it in items[b:b + 128]]), q[b:b + 128],
                                    return_aux=True)
        feats.append(aux['fc3_out'])
    F = np.concatenate(feats).astype(np.float64)
    A = np.concatenate([F, np.ones((n, 1))], 1)
    t_sign = np.where(d >= 0, 1.0, -1.0) * np.minimum(np.abs(d) / 0.01, 3.0)
    t_mag = np.arctanh(np.sqrt(np.clip(np.abs(d) / r, 0.0, 0.98)))
    ntr = 896
    W = np.linalg.solve(A[:ntr].T @ A[:ntr] + 0.1 * np.eye(129), A[:ntr].T @ np.stack([t_mag[:ntr], t_sign[:ntr]], 1))
    pred = A @ W
    acc = ((pred[ntr:, 1] >= 0) == (d[ntr:] >= 0)).mean()
    print('fit shared_encoder: held-out sign accuracy %.3f (%d queries), train %.3f'
          % (acc, n - ntr, ((pred[:ntr, 1] >= 0) == (d[:ntr] >= 0)).mean()))
    w32, b32 = W[:128].T.astype(np.float32), W[128].astype(np.float32)
    doc = {'variant': VARIANT, 'seed': MODEL_SEED, 'heldout_sign_accuracy': float(acc),
           'weight': [[float(x) for x in row] for row in w32], 'bias': [float(x) for x in b32]}
    with open(synth.FITTED_FC4_SHARED_ENCODER, 'w') as fp:
        json.dump(doc, fp, indent=1)
        fp.write('\n')
    w, b = synth.fitted_fc4(VARIANT, MODEL_SEED)
    assert np.array_equal(w, w32) and np.array_equal(b, b32), 'the text form must read back exactly'
    print('written', synth.FITTED_FC4_SHARED_ENCODER)


def golden():
    from source.points_to_surf_model import PointsToSurfModel
    v = synth.VARIANTS[VARIANT]
    inp = synth.make_model_inputs(BATCH, seed=INPUT_SEED)

    def ref_model():
        return PointsToSurfModel(net_size_max=1024, num_points=300, output_dim=2, use_point_stn=v['use_point_stn'],
                                 use_feat_stn=1, sym_op='max', use_query_point=True, sub_sample_size=1000,
                                 do_augmentation=False, single_transformer=v['single_transformer'],
                                 shared_transformation=v['shared_transformer'])

    def ref_run(sd):
        m = ref_model()
        m.load_state_dict(sd)
        m.eval()
        taps = {}
        m.feat_local_global.register_forward_hook(lambda mod, x, y: taps.update(feat_max=y[0], trans=y[1]))
        x = {k: torch.from_numpy(a.copy()) for k, a in inp.items()}
        return m(x).numpy(), {k: t.numpy() for k, t in taps.items()}

    keys = list(ref_model().state_dict().keys())
    sd = synth.make_state_dict(VARIANT, MODEL_SEED, fitted=True)
    assert list(sd.keys()) == keys, 'synth key order differs from the reference'
    # the fitted head is one-signed on these (non-surface) inputs: re-centre its bias on them so both signs occur
    fc4_bias = (sd['fc4.bias'].numpy() - np.median(ref_run(sd)[0], axis=0)).astype(np.float32)
    sd['fc4.bias'] = torch.from_numpy(fc4_bias)
    logits, taps = ref_run(sd)
    assert logits.shape == (BATCH, 2)
    o, aux = sorc.model_forward(sd, inp['patch_pts_ps'], inp['pts_sub_sample_ms'], inp['imp_surf_query_point_ms'],
                                return_aux=True)
    err = float(np.abs(o - logits).max())
    assert err < 1e-4, err
    assert np.abs(aux['trans'] - taps['trans']).max() < 1e-5
    assert np.abs(aux['feat_max'] - taps['feat_max']).max() < 1e-4
    print('golden shared_encoder: oracle-vs-reference max abs logit err %.3g, trans %.3g, feat %.3g; positive fraction '
          '%s, |sign logit| range [%.3g, %.3g]'
          % (err, np.abs(aux['trans'] - taps['trans']).max(), np.abs(aux['feat_max'] - taps['feat_max']).max(),
             (logits > 0).mean(0), np.abs(logits[:, 1]).min(), np.abs(logits[:, 1]).max()))
    np.savez_compressed(os.path.join(HERE, 'shared_encoder.npz'), model_seed=MODEL_SEED, input_seed=INPUT_SEED,
                        batch=BATCH, fc4_bias=fc4_bias, logits=logits, trans=taps['trans'], feat_max=taps['feat_max'],
                        state_dict_keys=np.array(keys),
                        input_checksum=np.float64(sum(float(np.abs(a).sum()) for a in inp.values())))


if __name__ == '__main__':
    stages = sys.argv[1:] or ['fit', 'golden']
    if 'fit' in stages:
        fit()
    if 'golden' in stages:
        golden()
