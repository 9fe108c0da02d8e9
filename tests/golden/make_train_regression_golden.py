"""Generate tests/golden/train_regression.npz: one training iteration of the regression ablation (outputs imp_surf
patch_pts_ids p_index, experiments/train_p2s_regression.sh) in the UNMODIFIED reference.

Run in the build container only (imports the reference through oracle/ref_shims.py):
    python tests/golden/make_train_regression_golden.py

For fixed_radius False and True: PointsToSurfModel(output_dim=1, use_point_stn=1, shared_transformation=0) on
synth.make_state_dict('regression', SEED) in train(), the reference's compute_loss with the regression outputs, backward
and SGD(lr=0.01, momentum=0.9) on a 32-query batch (tests/helpers_train_regression.py:make_regression_train_batch; only
its checksum is stored), then the reference's calc_metrics on the logits and the batch compute_loss left behind.  The
digest is that of make_golden.py:gen_train (logits, loss, gradient norms and sampled entries, updated tensors, running
statistics), asserted equal to tests/train_regression_oracle.py with gen_train's bars in the same run.  The fixture also
pins the initialisation of PointsToSurfModel(output_dim=1, ...) under a torch seed (per-tensor sum and first entry), the
way train_init.npz pins the two-output head, after asserting points_to_surf_train.initial_state_dict equal to it.
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
from points2surf_b200 import synth  # noqa: E402
sys.path.insert(0, os.path.dirname(HERE))
import train_regression_oracle as trorc  # noqa: E402
from helpers_train_regression import make_regression_train_batch  # noqa: E402
from helpers import train_digest_indices  # noqa: E402

from source import points_to_surf_train as ref_train  # noqa: E402
from source.points_to_surf_model import PointsToSurfModel  # noqa: E402

torch.set_grad_enabled(False)
VARIANT = 'regression'
SEED = 24
INIT_SEED = 3627473
BATCH = 32
OUTPUTS = ['imp_surf', 'patch_pts_ids', 'p_index']


def _model(do_augmentation=False):
    v = synth.VARIANTS[VARIANT]
    return PointsToSurfModel(net_size_max=1024, num_points=300, output_dim=1, use_point_stn=v['use_point_stn'],
                             use_feat_stn=1, sym_op='max', use_query_point=0, sub_sample_size=1000,
                             do_augmentation=do_augmentation, single_transformer=0,
                             shared_transformation=v['shared_transformer'])


def gen_iteration(out):
    v = synth.VARIANTS[VARIANT]
    sd = synth.make_state_dict(VARIANT, seed=SEED)
    batch = make_regression_train_batch(BATCH, 300, 1000, seed=SEED)
    out['batch'] = np.array(BATCH)
    out['input_checksum'] = np.array(sum(float(t.double().abs().sum()) for t in batch.values()))
    for fixed_radius in (False, True):
        pre = 'fixed_' if fixed_radius else 'radius_'
        torch.manual_seed(0)
        m = _model()
        m.load_state_dict(sd)
        m.train()
        opt = torch.optim.SGD(m.parameters(), lr=0.01, momentum=0.9)
        opt.zero_grad()
        bd = {k: t.clone() for k, t in batch.items()}
        with torch.enable_grad():
            pred = m(bd)
            loss = ref_train.compute_loss(pred=pred, batch_data=bd, outputs=OUTPUTS, output_loss_weights={'imp_surf': 1.0},
                                          fixed_radius=fixed_radius)
            assert len(loss) == 1
            sum(loss).backward()
        grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
        opt.step()
        new_sd = {k: t.detach().clone() for k, t in m.state_dict().items()}
        # the training loop's calc_metrics reads the batch compute_loss normalised in place, and mutates the logits
        metrics = ref_train.calc_metrics(outputs=OUTPUTS, pred=pred.detach().clone(), gt_data=bd)

        orc_out = trorc.train_iteration(sd, batch, v['use_point_stn'], v['shared_transformer'], lr=0.01, momentum=0.9,
                                        outputs=trorc.REGRESSION, fixed_radius=fixed_radius)
        assert np.allclose(orc_out['logits'].numpy(), pred.detach().numpy(), atol=2e-5), fixed_radius
        assert abs(orc_out['losses'][0] - float(loss[0])) < 1e-6, (orc_out['losses'], float(loss[0]))
        nscale = max(float(g.norm()) for g in grads.values())
        for k, g in grads.items():
            err = float((orc_out['grads'][k] - g).norm())
            assert err <= 2e-2 * float(g.norm()) + 1e-4 * nscale, (fixed_radius, k, err, float(g.norm()))
        for k, t in new_sd.items():
            if k.endswith('num_batches_tracked'):
                continue
            assert float((orc_out['new_state'][k] - t).norm()) <= 1e-3 * (1e-3 + float(t.norm())), (fixed_radius, k)

        out[pre + 'logits'] = pred.detach().numpy()
        out[pre + 'losses'] = np.array([float(loss[0])])
        names = sorted(grads)
        out[pre + 'names'] = np.array(names)
        out[pre + 'grad_norm'] = np.array([float(grads[k].double().norm()) for k in names])
        out[pre + 'grad_max'] = np.array([float(grads[k].abs().max()) for k in names])
        out[pre + 'grad_samples'] = np.stack([np.pad(grads[k].reshape(-1).numpy()[train_digest_indices(k, grads[k].numel())],
                                                     (0, 48 - min(48, grads[k].numel()))) for k in names])
        out[pre + 'new_samples'] = np.stack([np.pad(new_sd[k].reshape(-1).numpy()[train_digest_indices(k, new_sd[k].numel())],
                                                    (0, 48 - min(48, new_sd[k].numel()))) for k in names])
        bn = sorted(k for k in new_sd if k.endswith('running_mean') or k.endswith('running_var'))
        out[pre + 'buffer_names'] = np.array(bn)
        out[pre + 'buffer_samples'] = np.stack([np.pad(new_sd[k].numpy()[train_digest_indices(k, new_sd[k].numel())],
                                                       (0, 48 - min(48, new_sd[k].numel()))) for k in bn])
        out[pre + 'metrics_json'] = np.array(json.dumps(metrics, sort_keys=True))
        print('fixed_radius %s: loss %.6g, metrics %s, oracle == reference' % (fixed_radius, float(loss[0]), metrics))


def gen_init(out):
    from points2surf_b200 import points_to_surf_train as mine
    v = synth.VARIANTS[VARIANT]
    torch.manual_seed(INIT_SEED)
    ref_sd = _model(do_augmentation=True).state_dict()
    torch.manual_seed(INIT_SEED)
    my_sd = mine.initial_state_dict(v['use_point_stn'], v['shared_transformer'], 1024, 1)
    assert list(ref_sd.keys()) == list(my_sd.keys())
    for k in ref_sd:
        assert ref_sd[k].shape == my_sd[k].shape and torch.equal(ref_sd[k], my_sd[k]), k
    assert tuple(ref_sd['fc4.weight'].shape) == (1, 128)
    names = [k for k in ref_sd if ref_sd[k].is_floating_point()]
    out['init_seed'] = np.array(INIT_SEED)
    out['init_names'] = np.array(names)
    out['init_sums'] = np.array([float(ref_sd[k].double().sum()) for k in names])
    out['init_first'] = np.array([float(ref_sd[k].reshape(-1)[0]) for k in names])


if __name__ == '__main__':
    res = {}
    gen_iteration(res)
    gen_init(res)
    np.savez_compressed(os.path.join(HERE, 'train_regression.npz'), **res)
    print('train_regression.npz written')
