"""GPU tests of the training step (SURVEY.md section 8a row a14): the `p2s_op_*` primitives against plain torch ops on
the same device, and one full iteration of points2surf_b200.train.TrainStep against the digest of the unmodified
reference's iteration (tests/golden/train_*.npz) and against the CPU training oracle."""
import numpy as np
import pytest
import torch

from oracle import train_oracle
from oracle.p2s_oracle import quat_to_rotmat
from points2surf_b200 import synth
from points2surf_b200.train import TrainStep, compute_loss
from points2surf_b200.train_ops import CudaPrims
from helpers import TRAIN_SEEDS, check_train_digest, compare_gradients_l2, train_fixture_batch
from helpers_train import TorchPrims, make_train_batch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def close(a, b, rtol, what=''):
    a, b = a.double().cpu(), b.double().cpu()
    err = float((a - b).abs().max())
    assert err <= rtol * (float(b.abs().max()) + 1e-30), (what, err, float(b.abs().max()))


@pytest.mark.parametrize('M,N,K,Z', [(1, 1, 1, 1), (300, 64, 3, 1), (1000, 3, 64, 1), (5000, 128, 64, 1), (4097, 1024, 128, 1),
                                     (37, 4, 256, 1), (300, 64, 64, 7), (1000, 3, 3, 5), (129, 4096, 256, 1),
                                     (5000, 64, 64, 1), (2048, 192, 96, 1), (70000, 1024, 128, 1), (70000, 128, 1024, 1)])
def test_gemm_nt_and_tn(M, N, K, Z):
    p = CudaPrims()
    A = rnd(Z, M, K, seed=1) if Z > 1 else rnd(M, K, seed=1)
    W = rnd(Z, N, K, seed=2) if Z > 1 else rnd(N, K, seed=2)
    bias = rnd(N, seed=3)
    ref = torch.matmul(A.double(), W.double().transpose(-1, -2)) + bias.double()
    close(p.gemm_nt(A, W, bias), ref, 2e-6 * max(1, K ** 0.5), 'nt')
    close(p.gemm_nt(A, W, bias, relu=True), torch.relu(ref), 2e-6 * max(1, K ** 0.5), 'nt relu')
    Bm = rnd(Z, M, N, seed=4) if Z > 1 else rnd(M, N, seed=4)     # dZ [M,N], X = A [M,K]
    ref_tn = torch.matmul(Bm.double().transpose(-1, -2), A.double())
    close(p.gemm_tn(Bm, A), ref_tn, 3e-6 * max(1, M ** 0.5), 'tn')
    close(p.transpose(A), A.transpose(-1, -2), 0.0, 'transpose')
    acc = ref_tn.float().clone()
    p.gemm_tn(Bm, A, out=acc)           # accumulate form used for the weight gradients
    close(acc, 2 * ref_tn, 3e-6 * max(1, M ** 0.5), 'tn accumulate')
    close(p.gemm_nt(A, W), ref - bias.double(), 2e-6 * max(1, K ** 0.5), 'nt without bias')


def test_gemm_tn_split_reduction_large_m():
    p = CudaPrims()
    A, Bm = rnd(200000, 64, seed=5), rnd(200000, 128, seed=6)
    close(p.gemm_tn(A, Bm), A.double().t() @ Bm.double(), 1e-4, 'tn large M')


@pytest.mark.parametrize('M,C,relu', [(5, 512, True), (1300 * 6, 64, True), (3000, 1024, False), (2, 3, True), (70000, 128, True)])
def test_batchnorm_forward_backward(M, C, relu):
    p = CudaPrims()
    z = rnd(M, C, seed=7, scale=2.0) + 0.5
    gamma, beta = rnd(C, seed=8) * 0.2 + 1.0, rnd(C, seed=9) * 0.1
    rm, rv = rnd(C, seed=10) * 0.1, torch.rand(C, device=DEV) + 0.5
    rm_ref, rv_ref = rm.clone(), rv.clone()
    y, mean, invstd = p.bn_forward(z, gamma, beta, relu, rm, rv)
    zt = z.double().requires_grad_(True)
    gt, bt = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    with torch.enable_grad():
        yr = torch.nn.functional.batch_norm(zt, rm_ref.double(), rv_ref.double(), gt, bt, training=True, momentum=0.1, eps=1e-5)
        yr = torch.relu(yr) if relu else yr
    close(y, yr.detach(), 1e-5, 'bn y')
    close(rm, 0.9 * rm_ref.double() + 0.1 * z.double().mean(0), 1e-5, 'running mean')
    if M > 1:
        close(rv, 0.9 * rv_ref.double() + 0.1 * z.double().var(0, unbiased=True), 1e-5, 'running var')
    dy = rnd(M, C, seed=11)
    yr.backward(dy.double())
    dz, dgamma, dbeta = p.bn_backward(dy, z, y if relu else None, mean, invstd, gamma)
    tol = 2e-4 if M > 4 else 5e-2       # tiny batches: invstd ~ 1/sqrt(eps)-amplified rounding
    close(dz, zt.grad, tol, 'bn dz')
    close(dgamma, gt.grad, tol, 'dgamma')
    close(dbeta, bt.grad, tol, 'dbeta')
    close(p.col_sum(dy), dy.double().sum(0), 1e-5, 'col_sum')


@pytest.mark.parametrize('B,n,C', [(3, 300, 1024), (5, 1000, 64), (1, 1, 7), (9, 1300, 128)])
def test_maxpool_forward_backward(B, n, C):
    p = CudaPrims()
    y = rnd(B * n, C, seed=12)
    out, arg = p.maxpool_fwd(y, B, n)
    vr, ar = y.view(B, n, C).max(dim=1)
    assert torch.equal(out, vr) and torch.equal(arg.long(), ar)
    dout = rnd(B, C, seed=13)
    dy = p.maxpool_bwd(dout, arg, n)
    ref = torch.zeros(B, n, C, device=DEV).scatter_(1, ar.unsqueeze(1), dout.unsqueeze(1))
    assert torch.equal(dy.view(B, n, C), ref)
    # ReLU plateaus: ties resolve to the first maximum, like torch.max / MaxPool1d
    yt = torch.relu(y - 2.5)
    _, arg_t = p.maxpool_fwd(yt, B, n)
    first = (yt.view(B, n, C) == yt.view(B, n, C).max(dim=1, keepdim=True)[0]).float().argmax(dim=1)
    assert torch.equal(arg_t.long(), first)


@pytest.mark.parametrize('B,n,C,relu', [(4, 300, 1024, True), (3, 1000, 1024, False), (6, 1300, 128, True), (2, 5, 3, True)])
def test_fused_batchnorm_maxpool_matches_unfused(B, n, C, relu):
    p = CudaPrims()
    z = rnd(B * n, C, seed=30, scale=1.5) - (0.8 if relu else 0.0)
    gamma, beta = rnd(C, seed=31) * 0.3 + 1.0, rnd(C, seed=32) * 0.2
    gamma[::7] *= -1.0                       # negative scales: the arg-max of the output is the arg-min of z
    y, mean, invstd = p.bn_forward(z, gamma, beta, relu)
    out_ref, arg_ref = p.maxpool_fwd(y, B, n)
    out, arg, mean2, invstd2 = p.bn_maxpool_forward(z, B, n, gamma, beta, relu)
    assert torch.equal(out, out_ref) and torch.equal(arg, arg_ref)
    assert torch.equal(mean, mean2) and torch.equal(invstd, invstd2)
    dout = rnd(B, C, seed=33)
    dz_ref, dg_ref, db_ref = p.bn_backward(p.maxpool_bwd(dout, arg_ref, n), z, y if relu else None, mean, invstd, gamma)
    dz, dg, db = p.bn_maxpool_backward(dout, arg, out, z, mean, invstd, gamma, relu, B, n)
    close(dz, dz_ref, 1e-5, 'fused dz')
    close(dg, dg_ref, 1e-5, 'fused dgamma')
    close(db, db_ref, 1e-5, 'fused dbeta')


def test_loss_quaternion_and_elementwise_ops():
    p, tp = CudaPrims(), TorchPrims()
    B = 1024
    pred = rnd(B, 2, seed=14, scale=2.0)
    pred[0, 0] = 0.0
    tmag, rad = torch.rand(B, device=DEV) * 0.1, torch.rand(B, device=DEV) * 0.3 + 0.05
    tsign = (torch.rand(B, device=DEV) < 0.5).float()
    for fixed in (False, True):
        ls, dp = p.loss(pred, tmag, rad, tsign, 1.0, 0.7, fixed_radius=fixed)
        lr_, dr = tp.loss(pred.cpu(), tmag.cpu(), rad.cpu(), tsign.cpu(), 1.0, 0.7, fixed_radius=fixed)
        close(ls, lr_, 1e-5, 'loss')
        close(dp, dr, 1e-4, 'dloss')
    q = rnd(B, 4, seed=15, scale=0.3)
    R = p.quat_to_rot(q)
    close(R, quat_to_rotmat((q + q.new_tensor([1, 0, 0, 0])).double()), 1e-5, 'quat_to_rot')
    dR = rnd(B, 9, seed=16)
    close(p.quat_to_rot_bwd(q, dR), tp.quat_to_rot_bwd(q.double().cpu(), dR.double().cpu()), 1e-4, 'quat bwd')
    x, v = rnd(B, 64, seed=17), rnd(64, seed=18)
    close(p.add_row_(x.clone(), v), x + v, 0.0, 'add_row')
    pts, qq = rnd(7, 1000, 3, seed=19), rnd(7, 3, seed=20)
    close(p.center(pts, qq), pts - qq.unsqueeze(1), 0.0, 'center')
    yv = x.clone()
    close(p.axpy_(yv, x, 0.5), x * 1.5, 1e-7, 'axpy')
    par, grad, buf = rnd(1000, seed=21), rnd(1000, seed=22), torch.zeros(1000, device=DEV)
    par0 = par.clone()
    p.sgd_(par, grad, buf, 0.01, 0.9, True)
    close(par, par0 - 0.01 * grad, 1e-6, 'sgd first')
    p.sgd_(par, grad, buf, 0.01, 0.9, False)
    close(par, par0 - 0.01 * grad - 0.01 * 1.9 * grad, 1e-6, 'sgd second')


def _cuda_batch(batch):
    return {k: t.to(DEV) for k, t in batch.items()}


@pytest.mark.parametrize('variant', ['vanilla', 'max', 'uniform'])
def test_train_iteration_matches_reference_digest(variant):
    # fp32 CUDA iteration vs (a) the digest of the unmodified reference's fp32 CPU iteration on the same 32-query batch
    # and (b) the full gradients of the CPU training oracle evaluated in float64 (the rounding-free truth).
    # Tolerances are relative L2: per tensor <= 1.5e-1, all gradients together <= 5e-2.  Any fp32 implementation sits a
    # few percent from the f64 truth here, because max-pool arg-max / ReLU decisions flip under rounding and the
    # rotation gradient of the QSTN is a cancelling sum over 1300 points; tools/train_noise_study.py measures how far
    # torch CPU autograd, TrainStep over torch CUDA ops and these kernels each sit from the float64 truth.
    v = synth.VARIANTS[variant]
    sd = synth.make_state_dict(variant, seed=TRAIN_SEEDS[variant])
    batch = train_fixture_batch(variant)
    ts = TrainStep({k: t.to(DEV) for k, t in sd.items()}, v['use_point_stn'], v['shared_transformer'], lr=0.01, momentum=0.9)
    losses = ts.step(_cuda_batch(batch))
    grads = {k: t.cpu() for k, t in ts.named_gradients().items()}
    new = {k: t.cpu() for k, t in ts.state_dict().items()}
    wn, se = check_train_digest(variant, grads, new, [float(l) for l in losses], ts.last_logits.cpu().numpy(), tol=5e-2)
    ref = train_oracle.train_iteration(sd, batch, v['use_point_stn'], v['shared_transformer'], lr=0.01, momentum=0.9,
                                       dtype=torch.float64)
    wt, glob = compare_gradients_l2(grads, ref['grads'], tol_tensor=1.5e-1, tol_global=5e-2)
    print(variant, 'digest: worst norm err %.4f, sample rel-L2 %.4f | oracle: worst tensor rel-L2 %.4f, global %.4f' % (wn, se, wt, glob))


def test_train_two_steps_match_cpu_oracle_and_feed_inference():
    # two iterations (momentum path) of 32 queries against the f64 CPU oracle, on the `max` variant whose gradients are
    # well conditioned in fp32 (no QSTN: 0.01 / 0.004 worst-tensor / global noise); then a vanilla model takes two steps
    # and its state_dict drives the inference engine (the train -> eval hand-over of the reference,
    # points_to_surf_train.py:512-517)
    from points2surf_b200 import ops
    lr = 1e-4
    sd = synth.make_state_dict('max', seed=31)
    b1, b2 = make_train_batch(32, seed=5), make_train_batch(32, seed=6)
    r1 = train_oracle.train_iteration(sd, b1, 0, 0, lr=lr, dtype=torch.float64)
    sd2 = dict(sd)
    sd2.update(r1['new_state'])
    r2 = train_oracle.train_iteration(sd2, b2, 0, 0, lr=lr, mom_bufs=r1['mom_bufs'], dtype=torch.float64)
    ts = TrainStep({k: t.to(DEV) for k, t in sd.items()}, 0, 0, lr=lr)
    l1 = ts.step(_cuda_batch(b1))
    l2 = ts.step(_cuda_batch(b2))
    for got, want in zip(list(l1) + list(l2), r1['losses'] + r2['losses']):
        assert abs(float(got) - want) < 5e-3 * want, (float(got), want)
    new = ts.state_dict()
    moved = {k: (new[k].cpu().double() - sd[k].double()) for k in r2['grads']}       # lr * (1.9 g1 + g2)
    moved_ref = {k: (r2['new_state'][k] - sd[k].double()) for k in r2['grads']}
    # (the second gradient is taken at slightly different parameters on the two sides: arg-max flips compound)
    compare_gradients_l2(moved, moved_ref, tol_tensor=2e-1, tol_global=8e-2)
    assert int(new['bn2.num_batches_tracked']) == 102
    for name in ('bn2.running_mean', 'feat_local.bn3.running_var'):
        r = r2['new_state'][name]
        assert float((new[name].cpu().double() - r).abs().max()) <= 2e-3 * float(r.abs().max()) + 1e-6, name

    sdv = synth.make_state_dict('vanilla', seed=32)
    tv = TrainStep({k: t.to(DEV) for k, t in sdv.items()}, 1, 1, lr=1e-4)
    tv.step(_cuda_batch(b1))
    lv = tv.step(_cuda_batch(b2))
    assert all(np.isfinite(float(l)) for l in lv)
    eng = ops.Engine({k: t.cpu() for k, t in tv.state_dict().items()}, 1, 1, precision='fp32')
    inp = synth.make_model_inputs(4, seed=9)
    out = eng.forward(*(torch.from_numpy(inp[k]).to(DEV) for k in ('patch_pts_ps', 'pts_sub_sample_ms', 'imp_surf_query_point_ms')))
    assert torch.isfinite(out).all()
    with pytest.raises(ValueError):
        tv.forward({'patch_pts_ps': torch.zeros(2, 10, 3, device=DEV), 'pts_sub_sample_ms': torch.zeros(2, 1000, 3, device=DEV),
                    'imp_surf_query_point_ms': torch.zeros(2, 3, device=DEV)})


def test_cuda_graph_replay_matches_eager_steps():
    # the captured step must train exactly like the eager one: same losses, same parameter movement (fp32 atomics in the
    # weight-gradient kernel make both non-deterministic at the 1e-6 level), counters advanced, capture itself trains nothing
    sd = {k: t.to(DEV) for k, t in synth.make_state_dict('max', seed=41).items()}
    b1, b2 = _cuda_batch(make_train_batch(16, seed=7)), _cuda_batch(make_train_batch(16, seed=8))
    eager = TrainStep(sd, 0, 0, lr=1e-3)
    le = [eager.step(b1), eager.step(b2)]
    graph = TrainStep(sd, 0, 0, lr=1e-3)
    before = graph.flat_params.clone()
    graph.capture_graph(b1)
    assert torch.equal(graph.flat_params, before) and graph.steps_done == 0
    assert int(graph.buffers['bn2.num_batches_tracked']) == 100
    lg = [[float(x) for x in graph.step(b1)], [float(x) for x in graph.step(b2)]]
    for a, b in zip(le, lg):
        assert abs(float(a[0]) - b[0]) < 5e-3 * abs(b[0]) and abs(float(a[1]) - b[1]) < 5e-3 * abs(b[1])
    moved_e, moved_g = eager.flat_params - before, graph.flat_params - before
    assert float((moved_e - moved_g).norm()) <= 5e-2 * float(moved_e.norm())
    assert int(graph.buffers['bn2.num_batches_tracked']) == 102 and graph.steps_done == 2
    close(graph.buffers['bn2.running_mean'], eager.buffers['bn2.running_mean'], 1e-3, 'running mean after graph steps')


def test_training_loop_mirror_on_gpu(tmp_path):
    import sys
    sys.path.insert(0, __import__('os').path.dirname(__file__))
    from test_train_loop import _make_dataset
    from points2surf_b200 import points_to_surf_train as p2s_train
    root = str(tmp_path / 'data')
    _make_dataset(root, ['s0', 's1', 's2'], n_pts=2000, n_query=64)
    opt = p2s_train.parse_arguments([
        '--name', 'test', '--indir', root, '--outdir', str(tmp_path / 'models'), '--logdir', str(tmp_path / 'logs'),
        '--nepoch', '2', '--batchSize', '16', '--patches_per_shape', '32', '--points_per_patch', '300', '--sub_sample_size', '1000',
        '--patch_radius', '0.0', '--lr', '0.001', '--shared_transformer', '1',
        '--outputs', 'imp_surf_magnitude', 'imp_surf_sign', 'patch_pts_ids', 'p_index'])
    hist = p2s_train.points_to_surf_train(opt)
    assert len([h for h in hist if h[0] == 'train']) == 8 and all(np.isfinite(h[3]).all() for h in hist)
    assert (tmp_path / 'models' / 'test_model.pth').exists()
