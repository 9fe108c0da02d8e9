"""Test helpers of the regression head's training (outputs imp_surf): the torch stand-in primitives with the regression
loss, and a training batch that carries the signed distance imp_surf_ms.  Never imported by the product."""
import torch

from helpers_train import TorchPrims, make_train_batch


class RegressionTorchPrims(TorchPrims):
    """helpers_train.TorchPrims plus `loss_distance`, the counterpart of CudaPrims.loss_distance (plain torch autograd)."""

    def loss_distance(self, pred, target, radius, w, fixed_radius=False, need_grad=True):
        p = pred.detach().clone().requires_grad_(True)
        t = target if fixed_radius else target / radius
        with torch.enable_grad():
            l0 = torch.nn.functional.mse_loss(torch.tanh(p[:, 0]), torch.tanh(t)) * w
            l0.backward()
        return l0.detach().double().reshape(1), (p.grad if need_grad else None)


def make_regression_train_batch(B, P=300, S=1000, seed=0):
    """make_train_batch's fields plus imp_surf_ms, the signed distance the reference's DataLoader yields beside its
    magnitude and sign (data_loader.py:369,402): +magnitude where the sign flag is 1, -magnitude elsewhere."""
    out = make_train_batch(B, P, S, seed)
    mag = out['imp_surf_magnitude_ms']
    out['imp_surf_ms'] = torch.where(out['imp_surf_dist_sign_ms'] == 1, mag, -mag)
    return out
