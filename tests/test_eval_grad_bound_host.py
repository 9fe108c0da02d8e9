"""CPU checks of the conditioned float64 eval-mode backward and its error scale (tests/eval_grad_bound.py) before any GPU
run:

* Consistent: with the float64 EvalGrad's own decisions its values equal EvalGrad(dtype=float64) on the torch stand-in
  primitives to 1e-10 of each tensor's largest element.
* Sound: an fp32 EvalGrad on the stand-ins stays inside LAMBDA e on every parameter and input gradient element.
* Has teeth: a 1e-4 relative error on one element of a head or conv3 gradient, below what a relative-L2 or a 1e-3
  tolerance sees, breaks the bound."""
import pytest
import torch

import dropin_grad_oracle as dgo
import eval_grad_bound as egb
import train_step_bound as tsb
from points2surf_b200 import synth
from points2surf_b200.train import EvalGrad


def _run(variant, output_dim, P, S, dtype):
    v = synth.VARIANTS[variant]
    B = 3
    sd, patch, sub, query = dgo.make_case(variant, output_dim, P, S, B, seed=11 + P, dtype=dtype)
    batch = {'patch_pts_ps': patch, 'pts_sub_sample_ms': sub, 'imp_surf_query_point_ms': query}
    dlogits = torch.randn(B, output_dim, generator=torch.Generator().manual_seed(5), dtype=dtype)
    eg = EvalGrad(sd, v['use_point_stn'], v['shared_transformer'], P, S, output_dim=output_dim, device='cpu',
                  prims=dgo.EvalTorchPrims(), dtype=dtype)
    logits = eg.forward(batch)
    dec = tsb.decisions(eg._rec, logits)
    got_in = eg.backward_inputs(dlogits)
    ref = egb.reference(eg, dec, {k: t.double() for k, t in batch.items()}, dlogits.double(), fp32_only=True)
    return eg, got_in, ref


@pytest.mark.parametrize('output_dim', [2, 1])
@pytest.mark.parametrize('variant', ['vanilla', 'uniform', 'max'])
def test_bound_values_equal_float64_evalgrad(variant, output_dim):
    eg, got_in, ref = _run(variant, output_dim, 8, 64, torch.float64)
    for name, got, r in egb.checks(eg, got_in, ref):
        scale = float(r.v.abs().max())
        assert float((got.reshape(r.v.shape) - r.v).abs().max()) <= 1e-10 * max(scale, 1e-300), name


@pytest.mark.parametrize('output_dim', [2, 1])
@pytest.mark.parametrize('variant', ['vanilla', 'uniform', 'max'])
def test_fp32_run_is_inside_the_bound(variant, output_dim):
    eg, got_in, ref = _run(variant, output_dim, 8, 64, torch.float32)
    res = tsb.ratios(egb.checks(eg, got_in, ref))
    print(variant, output_dim, 'worst', max(res, key=lambda r: r[1]))
    assert all(r[1] <= 1.0 for r in res), [r for r in res if r[1] > 1.0]
    med = tsb.width_medians(egb.checks(eg, got_in, ref))
    # not vacuous: the median width is a few thousand ulps at most (the QSTN gradients, ~40 layers deep), where the
    # train-mode step needs 0.5 for its gradients
    assert max(med.values()) < 5e-3, med


@pytest.mark.parametrize('name', ['grad fc4.weight', 'grad bn2.weight', 'grad feat_local.conv3.bias',
                                  'grad feat_local.bn3.weight', 'grad feat_global.conv3.bias'])
def test_a_small_error_breaks_the_bound(name):
    """A 1e-4 relative error on the largest element of a head or conv3 gradient (the fused gather kernel's outputs)."""
    eg, got_in, ref = _run('vanilla', 2, 8, 64, torch.float32)
    got, r = [(g, v) for n, g, v in egb.checks(eg, got_in, ref) if n == name][0]
    i = int(r.v.abs().argmax())
    bad = got.clone()
    bad.view(-1)[i] *= 1 + 1e-4
    assert tsb.ratios([(name, bad, r)])[0][1] > 1.0, name
