"""CPU checks of the conditioned float64 training step and its error scale (tests/train_step_bound.py) before any GPU run.

* Consistent: with its own decisions the value part equals TrainStep(dtype=float64, prims=TorchPrims()) to 1e-11 of each
  tensor's largest element (float64 sums taken in another order reach 1.5e-12 on the cancelling weight-gradient sums).
* Sound: an fp32 CPU step (TrainStep(dtype=float32) on the torch stand-in primitives) stays inside LAMBDA e on every
  logit, loss, gradient, updated parameter, momentum buffer and running statistic, for every variant.
* Has teeth: single faults patched into the fp32 step break the bound; the output says which of them the relative-L2
  bars of tests/test_gpu_train.py (0.15 per gradient tensor, 0.05 over all of them) would have let through.
* Not vacuous: the median width LAMBDA e / |v| of every tensor is printed and held to a ceiling."""
import pytest
import torch

import train_step_bound as tsb
from points2surf_b200 import synth
from points2surf_b200.train import TrainStep
from helpers import compare_gradients_l2
from helpers_train import TorchPrims, make_train_batch
from helpers_train_regression import RegressionTorchPrims, make_regression_train_batch

VARIANTS = ['vanilla', 'max', 'uniform', 'regression']
SEEDS = {'vanilla': 21, 'max': 22, 'uniform': 23, 'regression': 24}


def make_step(variant, B, P, S, dtype, prims=None, **kw):
    v = synth.VARIANTS[variant]
    reg = variant == 'regression'
    if prims is None:
        prims = RegressionTorchPrims() if reg else TorchPrims()
    if reg:
        kw.setdefault('outputs', ('imp_surf',))
    return TrainStep(synth.make_state_dict(variant, seed=SEEDS[variant]), v['use_point_stn'], v['shared_transformer'],
                     points_per_patch=P, sub_sample_size=S, lr=0.01, momentum=0.9, device='cpu', prims=prims, dtype=dtype, **kw)


def make_batch(variant, B, P, S, seed, dtype=torch.float32):
    mk = make_regression_train_batch if variant == 'regression' else make_train_batch
    return {k: t.to(dtype) for k, t in mk(B, P, S, seed=seed).items()}


def run_steps(ts, variant, B, P, S, steps=2, fp32_only=True):
    """-> per step (drive record, reference, check items)."""
    out = []
    for k in range(steps):
        batch = make_batch(variant, B, P, S, seed=100 + k, dtype=ts.dtype)
        run = tsb.drive(ts, batch)
        ref = tsb.reference(ts, run, batch, fp32_only, exact_scalars=ts.dtype == torch.float64)
        out.append((run, ref, tsb.checks(ts, run, ref)))
    return out


def worst_of(items):
    return max(tsb.ratios(items), key=lambda r: r[1])


# ---------------------------------------------------------------------------------------------- consistency
@pytest.mark.parametrize('variant', VARIANTS)
def test_restatement_equals_float64_train_step(variant):
    B, P, S = 6, 20, 30
    for fixed in ([False, True] if variant == 'regression' else [False]):
        ts = make_step(variant, B, P, S, torch.float64, fixed_radius=fixed)
        for k, (run, ref, items) in enumerate(run_steps(ts, variant, B, P, S)):
            assert tsb.num_batches_tracked_ok(run)
            # the bias gradients of the BatchNorms behind a max-pool are zero in exact arithmetic (see _ceiling) and pure
            # rounding in both steps: they are measured against the largest gradient
            gscale = max(float(r.v.abs().max()) for n, _, r in items if n.startswith('grad'))
            bad = []
            for name, got, r in items:
                scale = float(r.v.abs().max())
                if name.startswith(('grad', 'mom')) and _ceiling(name) is None:
                    scale = gscale
                err = float((got.double().reshape(r.v.shape) - r.v).abs().max())
                if err > 1e-11 * scale:
                    bad.append((name, err / scale))
            assert not bad, (variant, k, bad[:5])


# ---------------------------------------------------------------------------------------------- soundness
SOUND = [(v, 32, 300, 1000) for v in VARIANTS] + [('vanilla', 7, 75, 130), ('regression', 7, 75, 130)]


@pytest.mark.parametrize('variant,B,P,S', SOUND)
def test_fp32_step_inside_the_bound(variant, B, P, S):
    ts = make_step(variant, B, P, S, torch.float32)
    for k, (run, ref, items) in enumerate(run_steps(ts, variant, B, P, S, steps=2 if B < 32 else 1)):
        assert tsb.num_batches_tracked_ok(run)
        rs = tsb.ratios(items)
        name, r, idx = max(rs, key=lambda x: x[1])
        print('%s (B, P, S) = (%d, %d, %d) step %d: worst ratio %.3f at %s %s' % (variant, B, P, S, k + 1, r, name, idx))
        assert r <= 1.0, [x for x in rs if x[1] > 1.0]
        if B == 32:
            check_widths(variant, items)


# ---------------------------------------------------------------------------------------------- non-vacuity
# Ceiling on the median of LAMBDA e / |v| per tensor, above the largest median measured at (32, 300, 1000) (in
# brackets).  Gradients, momentum buffers, logits and losses: 0.5 (0.26; 0.38 in the QSTN's fc1 weight).  Parameters: 2e-3 (7e-4): one step moves them
# by little, so their check sits a few hundred fp32 ulps wide.  Running statistics: 1e-2 (3e-3, the head's BatchNorms over
# 32 rows).  Named exceptions:
#  - the QSTN's parameters (point_stn., feat_global.stn1.): 0.05 (0.026).  Its gradient comes from dR summed over all P + S
#    points into four quaternion entries, a cancelling sum, and every layer below it inherits the width of dq;
#  - the bias gradients of the BatchNorms behind a max-pool (the conv3s' bn3): zero in exact arithmetic (sums of dx of a
#    BatchNorm'd FC layer, whose dz sums to zero over the batch), so |v| is rounding and the ratio is unbounded (1e13 to
#    6e13); they are held by the bound alone.
WIDTH_GRAD, WIDTH_PARAM, WIDTH_STATS, WIDTH_QSTN_PARAM = 0.5, 2e-3, 1e-2, 0.05


def _ceiling(name):
    if name.endswith('bn3.bias') and ('stn' in name or 'feat_' in name) and name.startswith(('grad', 'mom')):
        return None
    if name.startswith('param'):
        return WIDTH_QSTN_PARAM if ('point_stn.' in name or 'stn1.' in name) else WIDTH_PARAM
    if name.endswith(('running_mean', 'running_var')):
        return WIDTH_STATS
    return WIDTH_GRAD


def check_widths(variant, items):
    med = tsb.width_medians(items)
    print(variant, 'median LAMBDA e / |v|:', ', '.join('%s %.3g' % kv for kv in med.items()))
    bad = {n: w for n, w in med.items() if _ceiling(n) is not None and w > _ceiling(n)}
    assert not bad, bad


# ---------------------------------------------------------------------------------------------- faults
class FaultyPrims(TorchPrims):
    """TorchPrims with one fault, aimed at one layer through the data pointer of its parameter or gradient."""

    def __init__(self, fault):
        self.fault, self.target, self.calls = fault, None, 0

    def axpy_(self, y, x, a=1.0):
        if self.fault == 'drop_patch_dR' and tuple(y.shape[-2:]) == (3, 3):
            return y
        return super().axpy_(y, x, a)

    def transpose(self, x):
        if self.fault == 'T_not_transposed' and x.dim() == 3:
            return x.clone()
        return super().transpose(x)

    def bn_backward(self, dy, z, y_mask, mean, invstd, gamma):
        hit = self.target is not None and gamma.data_ptr() == self.target
        if hit and self.fault == 'drop_xh_m2':
            g = dy if y_mask is None else dy * (y_mask > 0)
            M = z.shape[0]
            s1, s2 = g.double().sum(0), (g * (z - mean) * invstd).double().sum(0)
            return gamma * invstd * (g - (s1 / M).to(z.dtype)), s2.to(z.dtype), s1.to(z.dtype)
        dz, dg, db = super().bn_backward(dy, z, y_mask, mean, invstd, gamma)
        if hit and self.fault == 'swap_dgamma_dbeta':
            return dz, db, dg
        return dz, dg, db

    def bn_maxpool_backward(self, dout, arg, out, z, mean, invstd, gamma, relu, B, npts):
        if self.fault == 'move_arg' and gamma.data_ptr() == self.target:
            arg = arg.clone()
            arg[0, 0] = (arg[0, 0] + 1) % npts
        return super().bn_maxpool_backward(dout, arg, out, z, mean, invstd, gamma, relu, B, npts)

    def gemm_tn(self, A, B, out=None):
        r = super().gemm_tn(A, B, out)
        if self.fault == 'wgrad_10_channels' and out is not None and out.data_ptr() == self.target:
            out[:10].zero_()
        return r

    def bn_forward(self, z, gamma, beta, relu, running_mean=None, running_var=None, eps=1e-5, momentum=0.1):
        old = running_var.clone() if running_var is not None else None
        res = super().bn_forward(z, gamma, beta, relu, running_mean, running_var, eps, momentum)
        if self.fault == 'biased_running_var' and gamma.data_ptr() == self.target:
            running_var.copy_((1 - momentum) * old + momentum * z.double().var(0, unbiased=False).to(z.dtype))
        return res

    def sgd_(self, param, grad, buf, lr, momentum, first):
        return super().sgd_(param, grad, buf, lr, momentum, True if self.fault == 'no_momentum_step2' else first)


# fault -> (what it is aimed at: a parameter or gradient name, or None)
FAULTS = {
    'drop_patch_dR': None,                                   # the patch branch's dR contribution (axpy_ in backward)
    'T_not_transposed': None,                                # T where dhb = dht T^T needs T^T
    'swap_dgamma_dbeta': ('param', 'feat_global.bn2.weight'),
    'drop_xh_m2': ('param', 'feat_local.bn1.weight'),        # the xh m2 term of one BatchNorm backward
    'move_arg': ('param', 'feat_global.bn3.weight'),         # one max-pool arg, one (query, channel)
    'wgrad_10_channels': ('grad', 'feat_global.conv3.weight'),  # 10 of 1024 output channels of a weight gradient
    'biased_running_var': ('param', 'bn2.weight'),
    'no_momentum_step2': None,
}


@pytest.mark.parametrize('fault', list(FAULTS))
def test_single_fault_breaks_the_bound(fault):
    B, P, S = 8, 64, 128
    prims = FaultyPrims(fault)
    ts = make_step('vanilla', B, P, S, torch.float32, prims=prims)
    aim = FAULTS[fault]
    if aim is not None:
        prims.target = (ts.params if aim[0] == 'param' else ts.grads)[aim[1]].data_ptr()
    steps = run_steps(ts, 'vanilla', B, P, S, steps=2)
    run, ref, items = steps[-1] if fault == 'no_momentum_step2' else steps[0]
    name, r, idx = worst_of(items)
    # the relative-L2 gradient bars of the GPU step test (helpers.compare_gradients_l2), against the same float64 step
    grads = {k: run['grads'][k] for k in ts.grads}
    ref_grads = {k: ref['grads'][k].v for k in ts.grads}
    try:
        compare_gradients_l2(grads, ref_grads, 0.15, 0.05)
        l2 = 'missed'
    except AssertionError:
        l2 = 'caught'
    print('%s: worst ratio %.3g at %s %s; the relative-L2 gradient bars (0.15 per tensor, 0.05 overall): %s'
          % (fault, r, name, idx, l2))
    assert r > 1.0, (fault, name, r)
