"""GPU tests of autograd through PointsToSurfModel in eval mode (points2surf_b200.train.EvalGrad and the kernels
p2s_op_bn_eval_backward / p2s_op_bn_maxpool_eval_bwd).

* The two kernels alone, per element, against a float64 restatement of the dense math with the bounds of
  include/p2s_b200.h (u = 2^-24): odd C, B = 1 with n = 1, tied arg-maxes, negative gamma, NaN in dout / dy.  The row
  offsets are 64-bit, so B * n * K past 2^31 cannot overflow; that case is not run (it would need 2 x 8.6 GB).
* The whole backward: every parameter and input gradient element of the CUDA EvalGrad within LAMBDA e of the float64
  backward of tests/eval_grad_bound.py, conditioned on the CUDA run's ReLU masks and arg-maxes (the worst ratio is
  printed), for the three layouts, both heads and (P, S) in {(8, 64), (63, 65), (300, 1000), (1200, 1000)}.
* The module: logits bit-identical with and without a recorded graph, the reference's in-place centring semantics,
  frozen parameters, the engine rebuild after optimizer.step(), and test-time fine-tuning of a checkpoint."""
import numpy as np
import pytest
import torch

import dropin_grad_oracle as dgo
import eval_grad_bound as egb
import train_step_bound as tsb
from points2surf_b200 import ops, synth
from points2surf_b200.model import PointsToSurfModel
from points2surf_b200.train import EvalGrad, compute_loss
from points2surf_b200.train_ops import CudaPrims

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
U = 2.0 ** -24


def _gamma(n):
    return n * U / (1 - n * U)


def _first_argmax(y, B, n):
    """Index of the first maximum over the points (NaN-free y) [B, C]."""
    yv = y.view(B, n, -1)
    mx = yv.max(1, keepdim=True)[0]
    idx = torch.arange(n, device=y.device).view(1, n, 1).expand_as(yv)
    return torch.where(yv == mx, idx, torch.full_like(idx, n)).min(1)[0]


def _check(name, got, ref, bound):
    """got fp32, ref / bound float64: NaN where ref is NaN, else |got - ref| <= bound; -> worst ratio."""
    got = got.double()
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(got), nan), name
    err = (got - ref).abs()[~nan]
    b = bound[~nan]
    assert bool((err <= b).all()), '%s: worst excess %g' % (name, float((err - b).max()))
    return float((err / b.clamp_min(1e-300)).max()) if err.numel() else 0.0


# ------------------------------------------------------------------ the kernels alone
@pytest.mark.parametrize('M,C,relu,nan', [(1, 1, True, False), (257, 77, True, True), (1000, 1024, False, False),
                                          (3000, 129, False, True)])
def test_bn_eval_backward_kernel(M, C, relu, nan):
    g = torch.Generator(device=DEV).manual_seed(M + C)
    z = torch.randn(M, C, device=DEV, generator=g) * 2 + 0.3
    dy = torch.randn(M, C, device=DEV, generator=g)
    if nan:
        dy.view(-1)[::97] = float('nan')
    mean = torch.randn(C, device=DEV, generator=g) * 0.2
    invstd = torch.rsqrt(torch.rand(C, device=DEV, generator=g) + 0.5 + 1e-5)
    gamma = torch.randn(C, device=DEV, generator=g)                    # about half negative
    beta = torch.randn(C, device=DEV, generator=g) * 0.1
    p = CudaPrims()
    y = p.bn_apply(z, mean, invstd, gamma, beta, relu)
    dz, dgamma, dbeta, dbias = p.bn_eval_backward(dy, z, y if relu else None, mean, invstd, gamma)
    gd = dy.double()
    if relu:
        gd = torch.where(y > 0, gd, torch.zeros_like(gd))
    gi = gamma.double() * invstd.double()
    xh = (z.double() - mean.double()) * invstd.double()
    dz_ref = gi * gd
    worst = [_check('dz', dz, dz_ref, 2.01 * U * dz_ref.abs()),
             _check('dgamma', dgamma, (gd * xh).sum(0), 2.01 * U * (gd * xh).abs().sum(0) + U * (gd * xh).sum(0).abs() + 1e-300),
             _check('dbeta', dbeta, gd.sum(0), U * gd.sum(0).abs() + 1e-300),
             _check('dbias', dbias, dz_ref.sum(0), 2.01 * U * dz_ref.abs().sum(0) + U * dz_ref.sum(0).abs() + 1e-300)]
    print('bn_eval_backward M=%d C=%d relu=%d nan=%d: worst error / bound %.3g' % (M, C, relu, nan, max(worst)))


@pytest.mark.parametrize('B,n,C,K,relu,ties,nan', [
    (1, 1, 7, 5, False, False, False),        # B = 1, n = 1, odd C
    (1, 1, 33, 3, True, False, True),
    (3, 50, 1023, 128, True, False, False),   # odd C in a conv3 shape
    (4, 64, 256, 128, False, True, False),    # every max tied with the next point
    (4, 64, 256, 128, True, True, True),
    (16, 300, 1024, 128, False, False, True),
])
def test_bn_maxpool_eval_backward_kernel(B, n, C, K, relu, ties, nan):
    g = torch.Generator(device=DEV).manual_seed(B * 1000 + n + C)
    x = torch.randn(B * n, K, device=DEV, generator=g)
    W = torch.randn(C, K, device=DEV, generator=g) * 0.1
    z = torch.randn(B * n, C, device=DEV, generator=g)
    if ties:
        zv = z.view(B, n, C)
        zv[:, 1::2] = zv[:, 0::2]
    mean = torch.randn(C, device=DEV, generator=g) * 0.2
    invstd = torch.rsqrt(torch.rand(C, device=DEV, generator=g) + 0.5 + 1e-5)
    gamma = torch.randn(C, device=DEV, generator=g)                    # about half negative: the order reverses there
    beta = torch.randn(C, device=DEV, generator=g) * 0.1
    p = CudaPrims()
    out, arg = p.bn_maxpool_apply(z, B, n, mean, invstd, gamma, beta, relu)
    # the arg-max is taken on the normalised values (the kernel's own fp32 y), first maximum
    y = p.bn_apply(z, mean, invstd, gamma, beta, relu)
    assert torch.equal(arg.long(), _first_argmax(y, B, n))
    assert torch.equal(out, y.view(B, n, C).max(1)[0])
    if ties:
        assert bool((arg % 2 == 0).all())
    dout = torch.randn(B, C, device=DEV, generator=g)
    if nan:
        dout.view(-1)[::13] = float('nan')
    dW0 = torch.randn(C, K, device=DEV, generator=g) * 0.01
    dW = dW0.clone()
    dx, dgamma, dbeta, dbias = p.bn_maxpool_eval_backward(dout, arg, out, z, x, W, mean, invstd, gamma, relu, B, n, dW)
    # float64 restatement of the dense path: scatter to the arg rows, eval BatchNorm backward, dW += dz^T x, dx = dz W
    gd = dout.double()
    if relu:
        gd = torch.where(out > 0, gd, torch.zeros_like(gd))
    gi = gamma.double() * invstd.double()
    dzb = gi * gd                                                       # [B, C]
    rows = (torch.arange(B, device=DEV).view(B, 1) * n + arg.long())   # [B, C]
    dense = torch.zeros(B * n, C, dtype=torch.float64, device=DEV)
    dense.scatter_(0, rows, dzb)
    xd, Wd = x.double(), W.double()
    xg = xd[rows]                                                       # [B, C, K]
    dW_ref = dW0.double() + torch.einsum('bc,bck->ck', dzb, xg)
    dW_mag = dW0.double().abs() + torch.einsum('bc,bck->ck', dzb.abs().nan_to_num(), xg.abs())
    cnt = torch.zeros(B * n, dtype=torch.float64, device=DEV).scatter_add_(0, rows.view(-1), torch.ones(B * C, dtype=torch.float64, device=DEV))
    dx_ref = dense @ Wd
    dx_mag = dense.abs().nan_to_num() @ Wd.abs()
    splits = 8 * torch.cuda.get_device_properties(0).multi_processor_count
    xh = (z.double()[rows, torch.arange(C, device=DEV).view(1, C)] - mean.double()) * invstd.double()
    worst = [
        _check('dW', dW, dW_ref, (2.01 * U + _gamma(B + splits + 2)) * dW_mag + 1e-300),
        _check('dx', dx, dx_ref.view(B * n, K), ((2.01 * U + _gamma(cnt + 2)).unsqueeze(1) * dx_mag) + 1e-300),
        _check('dgamma', dgamma, (gd * xh).sum(0), 2.01 * U * (gd * xh).abs().sum(0) + U * (gd * xh).sum(0).abs() + 1e-300),
        _check('dbeta', dbeta, gd.sum(0), U * gd.sum(0).abs() + 1e-300),
        _check('dbias', dbias, dzb.sum(0), 2.01 * U * dzb.abs().sum(0) + U * dzb.sum(0).abs() + 1e-300)]
    print('bn_maxpool_eval_bwd B=%d n=%d C=%d K=%d relu=%d ties=%d nan=%d: worst error / bound %.3g'
          % (B, n, C, K, relu, ties, nan, max(worst)))
    # need_dx=False leaves dx out and gives the same parameter gradients
    dW2 = dW0.clone()
    dx2, dg2, db2, dbi2 = p.bn_maxpool_eval_backward(dout, arg, out, z, x, W, mean, invstd, gamma, relu, B, n, dW2, need_dx=False)
    assert dx2 is None and torch.allclose(dW2, dW, rtol=1e-5, atol=1e-6, equal_nan=True)


# ------------------------------------------------------------------ the whole backward, per element
CASES = [(v, od, P, S) for v in ('vanilla', 'uniform', 'max') for od in (2, 1)
         for P, S in ((8, 64), (63, 65), (300, 1000), (1200, 1000))]


@pytest.mark.parametrize('variant,output_dim,P,S', CASES)
def test_eval_backward_per_element(variant, output_dim, P, S):
    """Every parameter and input gradient of the CUDA EvalGrad within LAMBDA e of the conditioned float64 backward of
    tests/eval_grad_bound.py; prints the worst ratio per tensor, in backward order."""
    v = synth.VARIANTS[variant]
    B = 4
    sd, patch, sub, query = dgo.make_case(variant, output_dim, P, S, B, seed=P + S, dtype=torch.float32)
    sd = {k: t.to(DEV) for k, t in sd.items()}
    batch = {'patch_pts_ps': patch.to(DEV), 'pts_sub_sample_ms': sub.to(DEV), 'imp_surf_query_point_ms': query.to(DEV)}
    dlogits = torch.randn(B, output_dim, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    eg = EvalGrad(sd, v['use_point_stn'], v['shared_transformer'], P, S, output_dim=output_dim, device=DEV)
    logits = eg.forward(batch)
    dec = tsb.decisions(eg._rec, logits)
    got_in = eg.backward_inputs(dlogits)
    ref = egb.reference(eg, dec, batch, dlogits, fp32_only=False,
                        sm_count=torch.cuda.get_device_properties(0).multi_processor_count)
    res = tsb.ratios(egb.checks(eg, got_in, ref))
    name, worst, at = max(res, key=lambda r: r[1])
    print('%s head %d P=%d S=%d: worst error / (LAMBDA e) %.3g (%s %s)' % (variant, output_dim, P, S, worst, name, at))
    bad = [r for r in res if not r[1] <= 1.0]
    assert not bad, bad


# ------------------------------------------------------------------ the module
def _model(variant='vanilla', output_dim=2, precision='fp32', P=300, S=1000, fitted=False):
    v = synth.VARIANTS[variant]
    m = PointsToSurfModel(net_size_max=1024, num_points=P, output_dim=output_dim, use_point_stn=bool(v['use_point_stn']),
                          sub_sample_size=S, shared_transformation=bool(v['shared_transformer']), precision=precision)
    sd = synth.make_state_dict(variant, 0 if not fitted else _fitted_seed(variant), fitted=fitted)
    if output_dim == 1:
        sd['fc4.weight'], sd['fc4.bias'] = sd['fc4.weight'][:1], sd['fc4.bias'][:1]
    m.load_state_dict(sd)
    return m.to(DEV).eval()


def _fitted_seed(variant):
    return int(np.load(synth.FITTED_FC4)[variant + '_seed'])


def _inputs(B=8, P=300, S=1000, seed=0):
    inp = synth.make_model_inputs(B, P, S, seed)
    return {k: torch.from_numpy(a).to(DEV) for k, a in inp.items()}


@pytest.mark.parametrize('precision', ['tc', 'fp32'])
@pytest.mark.parametrize('output_dim', [2, 1])
def test_logits_do_not_change_with_a_graph(precision, output_dim):
    m = _model(output_dim=output_dim, precision=precision)
    x0 = _inputs()
    with torch.no_grad():
        y0 = m({k: t.clone() for k, t in x0.items()})
    x = {k: t.clone() for k, t in x0.items()}
    x['patch_pts_ps'].requires_grad_(True)
    y1 = m(x)
    assert y1.grad_fn is not None and torch.equal(y1.detach(), y0)
    y1.sum().backward()
    assert x['patch_pts_ps'].grad is not None
    # train mode ignores .train() and records nothing
    m.train()
    y2 = m({k: t.clone() for k, t in x0.items()})
    assert not y2.requires_grad and torch.equal(y2, y0)


def test_in_place_centring_like_the_reference():
    m = _model()
    x0 = _inputs(B=4)
    # a leaf sub-sample that requires grad raises, like `shape_features -= query` does, and is left as it was
    x = {k: t.clone() for k, t in x0.items()}
    x['pts_sub_sample_ms'].requires_grad_(True)
    with pytest.raises(RuntimeError, match='leaf Variable'):
        m(x)
    assert torch.equal(x['pts_sub_sample_ms'].detach(), x0['pts_sub_sample_ms'])
    # a non-leaf sub-sample passes its gradient to the source tensor; the query gets minus its sum over the points,
    # and a later use of the (centred) caller's tensor adds its own gradient to both
    src = x0['pts_sub_sample_ms'].clone().requires_grad_(True)
    q = x0['imp_surf_query_point_ms'].clone().requires_grad_(True)
    shape = src * 1.0
    y = m({'patch_pts_ps': x0['patch_pts_ps'].clone(), 'pts_sub_sample_ms': shape, 'imp_surf_query_point_ms': q})
    assert torch.equal(shape.detach(), x0['pts_sub_sample_ms'] - x0['imp_surf_query_point_ms'].unsqueeze(1))
    c = torch.randn_like(shape)
    (y[:, 0].sum() + (shape * c).sum()).backward()
    # the same through EvalGrad directly
    eg = EvalGrad({k: t.detach() for k, t in m.state_dict().items()}, 1, 1, 300, 1000, device=DEV)
    eg.forward({'patch_pts_ps': x0['patch_pts_ps'], 'pts_sub_sample_ms': x0['pts_sub_sample_ms'],
                'imp_surf_query_point_ms': x0['imp_surf_query_point_ms']})
    dl = torch.zeros(4, 2, device=DEV)
    dl[:, 0] = 1
    _, dsub, dq = eg.backward_inputs(dl)
    assert torch.allclose(src.grad, dsub + c, rtol=1e-4, atol=1e-5)
    assert torch.allclose(q.grad, -(dsub + c).sum(1), rtol=1e-4, atol=1e-4)
    assert torch.allclose(q.grad, -src.grad.sum(1), rtol=1e-5, atol=1e-5)


def test_frozen_parameters_and_inputs_only():
    m = _model('uniform')
    x = _inputs(B=4)
    frozen = ['feat_local.conv1.weight', 'bn3.weight', 'fc4.bias']
    for n, t in m.named_parameters():
        if n in frozen:
            t.requires_grad_(False)
    m(x).sum().backward()
    for n, t in m.named_parameters():
        assert (t.grad is None) == (n in frozen), n
    # the bias in front of an eval-mode BatchNorm has a gradient
    assert float(m.feat_local.conv1.bias.grad.abs().max()) > 0
    m.zero_grad(set_to_none=True)
    for t in m.parameters():
        t.requires_grad_(False)
    x = _inputs(B=4)
    q = x['imp_surf_query_point_ms'].requires_grad_(True)
    y = m(x)
    assert y.grad_fn is not None
    y.sum().backward()
    assert q.grad is not None and bool(torch.isfinite(q.grad).all())
    assert all(t.grad is None for t in m.parameters())


def _sphere_batch(B=256, P=300, S=1000, seed=0):
    """Queries around the sphere of radius 0.5 (synth.make_cloud) with kNN patches in patch space (centred on the
    query, scaled by the patch radius) and a uniform sub-sample of the cloud; targets: |d|, sign(d > 0)."""
    rng = np.random.RandomState(seed)
    cloud = torch.from_numpy(synth.make_cloud('sphere', 10000, seed)).to(DEV)
    d = rng.standard_normal((B, 3))
    q = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0.35, 0.65, (B, 1))
    q = torch.from_numpy(q.astype(np.float32)).to(DEV)
    dist, idx = torch.cdist(q, cloud).topk(P, largest=False)
    radius = dist[:, -1]
    patch = (cloud[idx] - q.unsqueeze(1)) / radius.view(B, 1, 1)
    sub = cloud[torch.from_numpy(rng.randint(0, cloud.shape[0], (B, S))).to(DEV)]
    sd = q.norm(dim=1) - 0.5
    return {'patch_pts_ps': patch.contiguous(), 'pts_sub_sample_ms': sub.contiguous(), 'imp_surf_query_point_ms': q,
            'patch_radius_ms': radius, 'imp_surf_magnitude_ms': sd.abs(), 'imp_surf_dist_sign_ms': (sd > 0).float()}


def test_test_time_fine_tuning():
    m = _model('vanilla', fitted=True)
    batch = _sphere_batch()
    opt = torch.optim.SGD(m.parameters(), lr=1e-4, momentum=0.9)   # gradients of norm ~250 at the start
    outputs = ('imp_surf_magnitude', 'imp_surf_sign')
    weights = {'imp_surf_magnitude': 1.0, 'imp_surf_sign': 1.0}
    losses = []
    eng0 = None
    for it in range(30):
        x = {k: batch[k].clone() for k in ('patch_pts_ps', 'pts_sub_sample_ms', 'imp_surf_query_point_ms')}
        opt.zero_grad()
        y = m(x)
        eng0 = eng0 or m._engine
        ls, dpred = compute_loss(y.detach(), batch, outputs, weights, False, need_grad=True)
        y.backward(dpred)
        losses.append(float(sum(ls)))
        opt.step()
    print('fine-tuning loss: %.4f -> %.4f (x%.2f)' % (losses[0], losses[-1], losses[0] / losses[-1]))
    assert losses[-1] < losses[0] / 2
    # after step() the engine is rebuilt from the new weights: the module's forward equals a fresh Engine's
    x = {k: batch[k].clone() for k in ('patch_pts_ps', 'pts_sub_sample_ms', 'imp_surf_query_point_ms')}
    with torch.no_grad():
        y = m({k: t.clone() for k, t in x.items()})
    assert m._engine is not eng0
    fresh = ops.Engine({k: t.detach() for k, t in m.state_dict().items()}, 1, 1, 300, 1000, device=0, precision='fp32')
    assert torch.equal(y, fresh.forward(*x.values()))
    fresh.close()

