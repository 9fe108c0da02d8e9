"""CPU checks of the eval-mode backward behind PointsToSurfModel's autograd (points2surf_b200.train.EvalGrad):

* its host sequencing, run in float64 on the torch stand-in primitives, gives every parameter gradient and the
  gradients of patch, sub-sample and query of torch.autograd over a float64 eval-mode restatement of the reference
  network, to 1e-10 of each tensor's largest element, for the three point-STN layouts and both heads;
* the restatement itself passes torch.autograd.gradcheck;
* the two eval-mode entry points are exported with the signatures include/p2s_b200.h documents."""
import ctypes as C
import os
import re

import pytest
import torch

import dropin_grad_oracle as dgo
from points2surf_b200 import _lib, synth
from points2surf_b200.train import EvalGrad

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAYOUTS = ['vanilla', 'uniform', 'max']


def _rel(got, ref):
    scale = float(ref.abs().max())
    return float((got.reshape(ref.shape) - ref).abs().max()) / (scale if scale > 0 else 1.0)


@pytest.mark.parametrize('P,S', [(8, 64), (63, 65)])
@pytest.mark.parametrize('output_dim', [2, 1])
@pytest.mark.parametrize('variant', LAYOUTS)
def test_eval_backward_matches_autograd(variant, output_dim, P, S):
    v = synth.VARIANTS[variant]
    B = 3
    sd, patch, sub, query = dgo.make_case(variant, output_dim, P, S, B, seed=40 + P)
    dlogits = torch.randn(B, output_dim, generator=torch.Generator().manual_seed(7), dtype=torch.float64)
    logits_ref, grads_ref, dpatch_ref, dsub_ref, dquery_ref = dgo.autograd_reference(
        sd, patch, sub, query, dlogits, v['use_point_stn'], v['shared_transformer'])

    eg = EvalGrad(sd, v['use_point_stn'], v['shared_transformer'], P, S, output_dim=output_dim, device='cpu',
                  prims=dgo.EvalTorchPrims(), dtype=torch.float64)
    before = {k: t.clone() for k, t in eg.buffers.items()}
    logits = eg.forward({'patch_pts_ps': patch, 'pts_sub_sample_ms': sub, 'imp_surf_query_point_ms': query})
    assert _rel(logits, logits_ref) < 1e-12
    dpatch, dsub, dquery = eg.backward_inputs(dlogits)
    grads = eg.named_gradients()
    assert sorted(grads) == sorted(grads_ref)
    worst = max((_rel(grads[k], grads_ref[k]), k) for k in grads_ref)
    assert worst[0] < 1e-10, worst
    # in eval mode the bias in front of a BatchNorm has a gradient (TrainStep leaves it at 0 in train mode)
    assert float(grads['feat_local.conv1.bias'].abs().max()) > 0
    for name, got, ref in (('patch', dpatch, dpatch_ref), ('sub', dsub, dsub_ref), ('query', dquery, dquery_ref)):
        assert _rel(got, ref) < 1e-10, name
    # nothing is updated in eval mode
    assert all(torch.equal(before[k], eg.buffers[k]) for k in before)


def test_eval_backward_takes_the_extra_subsample_gradient():
    """A gradient that reaches the centred sub-sample by another way (a later use of the caller's centred tensor)
    adds to d sub-sample, and minus its sum over the points to d query."""
    v = synth.VARIANTS['vanilla']
    sd, patch, sub, query = dgo.make_case('vanilla', 2, 8, 64, 2, seed=5)
    dlogits = torch.randn(2, 2, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    extra = torch.randn(2, 64, 3, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    batch = {'patch_pts_ps': patch, 'pts_sub_sample_ms': sub, 'imp_surf_query_point_ms': query}

    def run(ex):
        eg = EvalGrad(sd, v['use_point_stn'], v['shared_transformer'], 8, 64, device='cpu', prims=dgo.EvalTorchPrims(),
                      dtype=torch.float64)
        eg.forward(batch)
        return eg.backward_inputs(dlogits, ex)

    _, dsub0, dq0 = run(None)
    _, dsub1, dq1 = run(extra)
    assert torch.allclose(dsub1 - dsub0, extra, rtol=0, atol=1e-12)
    assert torch.allclose(dq1 - dq0, -extra.sum(1), rtol=0, atol=1e-12)


@pytest.mark.parametrize('variant', LAYOUTS)
def test_restatement_passes_gradcheck(variant):
    v = synth.VARIANTS[variant]
    sd, patch, sub, query = dgo.make_case(variant, 2, 8, 8, 1, seed=3)
    params = {k: t for k, t in sd.items() if not (k.endswith('running_mean') or k.endswith('running_var')
                                                  or k.endswith('num_batches_tracked'))}
    bufs = {k: t for k, t in sd.items() if k.endswith('running_mean') or k.endswith('running_var')}
    # a few small tensors as the checked variables (every parameter would make gradcheck take minutes)
    names = ['fc4.weight', 'bn3.bias', 'feat_local.conv0a.weight', 'feat_global.bn3.weight']
    if v['use_point_stn']:
        names.append(('point_stn.' if v['shared_transformer'] else 'feat_global.stn1.') + 'fc3.bias')

    def f(p_, s_, q_, *ts):
        sd2 = dict(params)
        sd2.update(zip(names, ts))
        return dgo.forward_eval(sd2, bufs, p_, s_, q_, v['use_point_stn'], v['shared_transformer'])

    ins = [t.clone().requires_grad_(True) for t in (patch, sub, query)] + \
          [params[n].clone().requires_grad_(True) for n in names]
    assert torch.autograd.gradcheck(f, ins, eps=1e-6, atol=1e-6, rtol=1e-5)


def test_eval_entry_points_are_exported_with_their_documented_signatures():
    txt = open(os.path.join(ROOT, 'include', 'p2s_b200.h')).read()
    txt = re.sub(r'/\*.*?\*/', '', txt, flags=re.S)
    ctype = {'const float*': C.c_void_p, 'float*': C.c_void_p, 'const int32_t*': C.c_void_p, 'double*': C.c_void_p,
             'void*': C.c_void_p, 'int64_t': C.c_int64, 'int': C.c_int}
    lib = _lib.load()
    for name in ('p2s_op_bn_eval_backward', 'p2s_op_bn_maxpool_eval_bwd'):
        m = re.search(r'int\s+' + name + r'\s*\(([^)]*)\)', txt)
        assert m, name
        decl = [re.sub(r'\s+', ' ', a.strip()).rsplit(' ', 1)[0] for a in m.group(1).split(',')]
        want = [ctype[a] for a in decl]
        res, args = _lib.SIGNATURES[name]
        assert res is C.c_int and args == want, name
        assert hasattr(lib, name)
