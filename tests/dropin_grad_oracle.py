"""Test-only pieces for the eval-mode gradients of points2surf_b200.model.PointsToSurfModel (train.EvalGrad):

* `EvalTorchPrims`: the torch stand-in of helpers_train.TorchPrims with the eval-mode ops of train_ops.CudaPrims
  (bn_maxpool_apply, bn_eval_backward, bn_maxpool_eval_backward) written as the plain dense math they replace, so the
  host sequencing of EvalGrad can be checked in float64 on a CPU against autograd.
* `forward_eval`: a float64-capable functional restatement of the reference's eval-mode forward
  (source/points_to_surf_model.py:296-352, BatchNorm with running_mean / running_var, eps 1e-5), built from
  oracle/train_oracle.py's network walk with its BatchNorm switched to eval mode, for torch.autograd.
Never imported by the product."""
import contextlib

import torch
import torch.nn.functional as F

from oracle import train_oracle
from points2surf_b200 import synth
from helpers_train import TorchPrims

EPS = 1e-5


class EvalTorchPrims(TorchPrims):
    name = 'torch-test-eval'

    def bn_maxpool_apply(self, z, B, npts, mean, invstd, gamma, beta, relu):
        return self.maxpool_fwd(self.bn_apply(z, mean, invstd, gamma, beta, relu), B, npts)

    def bn_eval_backward(self, dy, z, y_mask, mean, invstd, gamma):
        g = dy if y_mask is None else dy * (y_mask > 0)
        dz = gamma * invstd * g
        # column sums in float64, like the kernel's
        return dz, *((t.double().sum(0).to(z.dtype)) for t in (g * ((z - mean) * invstd), g, dz))

    def bn_maxpool_eval_backward(self, dout, arg, out, z, x, W, mean, invstd, gamma, relu, B, npts, dW, need_dx=True):
        # the dense path: scatter dout to the arg rows, eval BatchNorm backward, dW += dz^T x, dx = dz W
        dy = self.maxpool_bwd(dout, arg, npts)
        y = self.maxpool_bwd(out, arg, npts) if relu else None
        dz, dgamma, dbeta, dbias = self.bn_eval_backward(dy, z, y, mean, invstd, gamma)
        self.gemm_tn(dz, x, out=dW)
        return (dz @ W if need_dx else None), dgamma, dbeta, dbias


@contextlib.contextmanager
def _eval_batch_norm():
    """train_oracle's walk calls F.batch_norm(..., training=True): run it with training=False (running statistics)."""
    orig = train_oracle.F

    class _F:
        def __getattr__(self, k):
            return getattr(F, k)

        @staticmethod
        def batch_norm(x, rm, rv, w, b, training=True, momentum=0.1, eps=EPS):
            return F.batch_norm(x, rm, rv, w, b, training=False, momentum=momentum, eps=eps)

    train_oracle.F = _F()
    try:
        yield
    finally:
        train_oracle.F = orig


def forward_eval(sd, bufs, patch, sub, query, use_point_stn, shared_transformer):
    """Eval-mode logits of the reference network; sd: parameters, bufs: running statistics (not modified)."""
    with _eval_batch_norm():
        return train_oracle.forward_train(sd, bufs, {'patch_pts_ps': patch, 'pts_sub_sample_ms': sub,
                                                     'imp_surf_query_point_ms': query}, use_point_stn, shared_transformer)


def make_case(variant, output_dim, P, S, B, seed, dtype=torch.float64, negative_gamma=True):
    """(state dict, inputs) for `variant` ('vanilla' | 'max' | 'uniform') with `output_dim` columns: the synthetic
    checkpoint, every third BatchNorm channel's gamma negated (so the max-pool's order is reversed there)."""
    sd = synth.make_state_dict(variant, seed)
    if output_dim == 1:
        sd['fc4.weight'], sd['fc4.bias'] = sd['fc4.weight'][:1].clone(), sd['fc4.bias'][:1].clone()
    if negative_gamma:
        for k in list(sd):
            if '.bn' in k and k.endswith('.weight') or k.startswith('bn') and k.endswith('.weight'):
                sd[k] = sd[k].clone()
                sd[k][::3] *= -1
    sd = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}
    g = torch.Generator().manual_seed(seed)
    patch = (torch.rand(B, P, 3, generator=g, dtype=torch.float64) * 2 - 1) * 0.1
    query = torch.rand(B, 3, generator=g, dtype=torch.float64) * 2 - 1
    sub = query.unsqueeze(1) + (torch.rand(B, S, 3, generator=g, dtype=torch.float64) * 2 - 1) * 0.5
    return sd, patch.to(dtype), sub.to(dtype), query.to(dtype)


def autograd_reference(sd, patch, sub, query, dlogits, use_point_stn, shared_transformer):
    """-> (logits, {param name: grad}, dpatch, dsub, dquery) of sum(logits * dlogits) by torch.autograd."""
    params = {k: v.detach().clone().requires_grad_(True) for k, v in sd.items()
              if not (k.endswith('running_mean') or k.endswith('running_var') or k.endswith('num_batches_tracked'))}
    bufs = {k: v for k, v in sd.items() if k.endswith('running_mean') or k.endswith('running_var')}
    ins = [t.detach().clone().requires_grad_(True) for t in (patch, sub, query)]
    with torch.enable_grad():
        logits = forward_eval(params, bufs, *ins, use_point_stn, shared_transformer)
        (logits * dlogits).sum().backward()
    return logits.detach(), {k: v.grad for k, v in params.items()}, ins[0].grad, ins[1].grad, ins[2].grad
