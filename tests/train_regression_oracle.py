"""TEST INFRASTRUCTURE ONLY -- CPU restatement of one training iteration of the reference with a choice of outputs:
oracle/train_oracle.py's forward with the loss of source/points_to_surf_train.py:compute_loss (:537-563) for either head.
For outputs (imp_surf_magnitude, imp_surf_sign) the loss is oracle/train_oracle.losses; for the regression ablation
(outputs imp_surf, experiments/train_p2s_regression.sh) it is sdf_nn.calc_loss_distance, restated with the reference's
torch CPU operations in its order.  tests/golden/make_train_regression_golden.py asserts this module equal to the
unmodified reference before it writes tests/golden/train_regression.npz."""
import torch
import torch.nn.functional as F

from oracle import train_oracle

MAGNITUDE_SIGN = ('imp_surf_magnitude', 'imp_surf_sign')
REGRESSION = ('imp_surf',)


def losses(pred, batch, outputs=MAGNITUDE_SIGN, output_loss_weights=None, fixed_radius=False):
    """compute_loss (points_to_surf_train.py:537-563) -> list of 0-d loss tensors.  The batch is not modified (the
    reference divides its target by the radius in place)."""
    if 'imp_surf' not in outputs:
        w = output_loss_weights or {'imp_surf_magnitude': 1.0, 'imp_surf_sign': 1.0}
        return train_oracle.losses(pred, batch, w['imp_surf_magnitude'], w['imp_surf_sign'], fixed_radius)
    w = output_loss_weights or {'imp_surf': 1.0}
    o_pred = pred.squeeze(1)
    o_target = batch['imp_surf_ms'].reshape(-1)
    if not fixed_radius:
        o_target = o_target / batch['patch_radius_ms'].reshape(-1)
    return [F.mse_loss(torch.tanh(o_pred), torch.tanh(o_target)) * w['imp_surf']]


def train_iteration(state_dict, batch, use_point_stn, shared_transformer, lr=0.01, momentum=0.9, mom_bufs=None,
                    dtype=torch.float32, outputs=MAGNITUDE_SIGN, fixed_radius=False):
    """oracle/train_oracle.train_iteration with the loss of `outputs`:
    -> dict(logits, losses, grads{name}, new_state{name}, mom_bufs{name}); `state_dict` is not modified."""
    batch = {k: v.to(dtype) for k, v in batch.items()}
    sd, bufs = {}, {}
    for k, v in state_dict.items():
        if k.endswith('num_batches_tracked'):
            continue
        if k.endswith('running_mean') or k.endswith('running_var'):
            bufs[k] = v.detach().clone().to(dtype)
        else:
            sd[k] = v.detach().clone().to(dtype).requires_grad_(True)
    with torch.enable_grad():
        logits = train_oracle.forward_train(sd, bufs, batch, use_point_stn, shared_transformer)
        ls = losses(logits, batch, outputs, fixed_radius=fixed_radius)
        sum(ls).backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in sd.items()}
    new_state, new_mom = {}, {}
    for k, v in sd.items():
        buf = grads[k].clone() if mom_bufs is None else momentum * mom_bufs[k] + grads[k]
        new_mom[k] = buf
        new_state[k] = (v.detach() - lr * buf)
    new_state.update(bufs)
    return {'logits': logits.detach(), 'losses': [float(l.detach()) for l in ls], 'grads': grads, 'new_state': new_state,
            'mom_bufs': new_mom}
