"""GPU tests of the regression ablation's training (outputs imp_surf patch_pts_ids p_index,
experiments/train_p2s_regression.sh): the `p2s_op_loss_distance` kernel against torch autograd, the one-column fc4
GEMMs against the per-element bound of the training GEMMs, one fp32 step against the unmodified reference's digest
(tests/golden/train_regression.npz) and the float64 oracle, CUDA-graph replay, over-fitting one batch, and the hand-over
from the training entry point to points_to_surf_eval."""
import numpy as np
import pytest
import torch

import train_regression_oracle as trorc
from points2surf_b200 import synth
from points2surf_b200.train import TrainStep
from points2surf_b200.train_ops import CudaPrims
from helpers import compare_gradients_l2, load_golden, train_digest_indices
from helpers_train import TorchPrims
from helpers_train_regression import RegressionTorchPrims, make_regression_train_batch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
VARIANT = 'regression'
V = synth.VARIANTS[VARIANT]
FIXTURE_SEED = 24          # tests/golden/make_train_regression_golden.py


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def close(a, b, rtol, what=''):
    a, b = a.double().cpu(), b.double().cpu()
    err = float((a - b).abs().max())
    assert err <= rtol * (float(b.abs().max()) + 1e-30), (what, err, float(b.abs().max()))


def _cuda(batch):
    return {k: t.to(DEV) for k, t in batch.items()}


def _step(sd, **kw):
    return TrainStep({k: t.to(DEV) for k, t in sd.items()}, V['use_point_stn'], V['shared_transformer'],
                     outputs=('imp_surf',), output_loss_weights={'imp_surf': 1.0}, **kw)


# ------------------------------------------------------------------ loss kernel
@pytest.mark.parametrize('B', [1, 7, 1024, 4097])
@pytest.mark.parametrize('fixed', [False, True])
def test_loss_distance_kernel(B, fixed):
    p, tp = CudaPrims(), RegressionTorchPrims()
    pred = rnd(B, 1, seed=B, scale=2.0)
    pred[0, 0] = 0.0
    t = (torch.rand(B, device=DEV) - 0.5) * 0.2
    rad = torch.rand(B, device=DEV) * 0.3 + 0.05
    want_l, want_d = tp.loss_distance(pred.double().cpu(), t.double().cpu(), rad.double().cpu(), 0.7, fixed_radius=fixed)
    for need_grad in (True, False):
        ls, dp = p.loss_distance(pred, t, rad, 0.7, fixed_radius=fixed, need_grad=need_grad)
        assert ls.dtype == torch.float64 and ls.shape == (1,)
        close(ls, want_l, 1e-5, 'loss')
        if need_grad:
            assert dp.shape == (B, 1)
            close(dp, want_d, 1e-4, 'dpred')
        else:
            assert dp is None
    # the two-output loss is unchanged beside it
    pred2 = rnd(B, 2, seed=B + 1, scale=2.0)
    tsign = (torch.rand(B, device=DEV) < 0.5).float()
    ls2, dp2 = p.loss(pred2, t.abs(), rad, tsign, 1.0, 0.7, fixed_radius=fixed)
    lr2, dr2 = TorchPrims().loss(pred2.double().cpu(), t.abs().double().cpu(), rad.double().cpu(), tsign.double().cpu(), 1.0,
                                 0.7, fixed_radius=fixed)
    close(ls2, lr2, 1e-5, 'two-output loss')
    close(dp2, dr2, 1e-4, 'two-output dloss')


# ------------------------------------------------------------------ the one-column fc4 through the training GEMMs
@pytest.mark.parametrize('B', [32, 1024])
@pytest.mark.parametrize('kind', ['forward', 'input_grad', 'weight_grad', 'weight_grad_acc'])
def test_one_column_gemms_per_element_bound(B, kind):
    # the shapes TrainStep issues for fc4 (128 -> 1), with training magnitudes: activations >= 0 after ReLU, weights
    # ~0.05, dlogits ~2^-10 (a batch mean); the bound is oracle/split_gemm.py's, as in test_gpu_train.test_gemm_per_element_bound
    from oracle import split_gemm
    p = CudaPrims()
    x = rnd(B, 128, seed=60).abs()
    W = rnd(1, 128, seed=61, scale=0.05)
    dz = rnd(B, 1, seed=62, scale=2.0 ** -10)
    if kind == 'forward':                         # x W^T: (B, 1, 128)
        got, exact, bound = p.gemm_nt(x, W), x.double() @ W.double().t(), split_gemm.bound_nt(x, W)
    elif kind == 'input_grad':                    # dz W = dz (W^T)^T: (B, 128, 1)
        Wt = p.transpose(W)
        got, exact, bound = p.gemm_nt(dz, Wt), dz.double() @ W.double(), split_gemm.bound_nt(dz, Wt)
    elif kind == 'weight_grad':                   # dz^T x: N = 1, K = 128
        got, exact, bound = p.gemm_tn(dz, x), dz.double().t() @ x.double(), split_gemm.bound_nt(dz.t(), x.t())
    else:
        acc = rnd(1, 128, seed=63, scale=1e-3)
        got = p.gemm_tn(dz, x, out=acc.clone())
        exact = dz.double().t() @ x.double() + acc.double()
        bound = split_gemm.bound_nt(dz.t(), x.t(), extra=acc)
    e = split_gemm.excess(got, exact, bound)
    print(kind, B, 'max error / bound %.3g' % e)
    assert tuple(got.shape) == tuple(exact.shape) and e <= 1.0, (kind, B, e)


# ------------------------------------------------------------------ one step against the reference
def _check_digest(pre, grads, new_state, loss, logits, tol):
    """helpers.check_train_digest for the regression fixture (one loss, keys prefixed by the radius mode)."""
    g = load_golden('train_regression.npz')
    assert abs(loss - g[pre + 'losses'][0]) <= 2e-3 * g[pre + 'losses'][0] + 1e-6
    assert np.abs(np.asarray(logits) - g[pre + 'logits']).max() <= 5e-3 * np.abs(g[pre + 'logits']).max() + 1e-5
    names = [str(n) for n in g[pre + 'names']]
    assert sorted(grads) == names
    nscale = float(g[pre + 'grad_norm'].max())
    bad, worst_norm, num, den, pnum = [], 0.0, 0.0, 0.0, 0.0
    for i, name in enumerate(names):
        t = grads[name].reshape(-1).double().numpy()
        idx = train_digest_indices(name, t.size)
        nerr = abs(float(np.linalg.norm(t)) - float(g[pre + 'grad_norm'][i])) / (float(g[pre + 'grad_norm'][i]) + 1e-3 * nscale)
        worst_norm = max(worst_norm, nerr)
        if nerr > tol:
            bad.append((name, 'norm', round(nerr, 4)))
        scale = float(g[pre + 'grad_max'][i]) + 1e-3 * float(g[pre + 'grad_max'].max())
        ref = g[pre + 'grad_samples'][i][:idx.size]
        num += float((((t[idx] - ref) / scale) ** 2).sum())
        den += float(((ref / scale) ** 2).sum())
        q = new_state[name].reshape(-1).double().numpy()
        pnum += float((((q[idx] - g[pre + 'new_samples'][i][:idx.size]) / (0.01 * scale)) ** 2).sum())   # lr = 0.01
    assert not bad, 'gradient norm mismatches: %s' % bad
    sample_err, param_err = (num / den) ** 0.5, (pnum / den) ** 0.5
    assert sample_err <= tol and param_err <= tol, (sample_err, param_err)
    for i, name in enumerate(str(n) for n in g[pre + 'buffer_names']):
        b = new_state[name].reshape(-1).double().numpy()
        idx = train_digest_indices(name, b.size)
        ref = g[pre + 'buffer_samples'][i][:idx.size]
        assert np.abs(b[idx] - ref).max() <= 2e-3 * (np.abs(ref).max() + 1e-3), (name, 'running statistic')
    return worst_norm, sample_err


@pytest.mark.parametrize('fixed_radius', [False, True])
def test_train_iteration_matches_reference_digest(fixed_radius):
    # the bars of test_gpu_train.test_train_iteration_matches_reference_digest for the `uniform` variant, whose
    # network this is (digest 5e-2; f64 oracle: per tensor relative L2 1.5e-1, global 5e-2)
    g = load_golden('train_regression.npz')
    sd = synth.make_state_dict(VARIANT, seed=FIXTURE_SEED)
    batch = make_regression_train_batch(int(g['batch']), 300, 1000, seed=FIXTURE_SEED)
    assert abs(sum(float(t.double().abs().sum()) for t in batch.values()) - float(g['input_checksum'])) < 1e-9 * float(g['input_checksum'])
    ts = _step(sd, lr=0.01, momentum=0.9, fixed_radius=fixed_radius)
    losses = ts.step(_cuda(batch))
    assert len(losses) == 1 and tuple(ts.last_logits.shape) == (32, 1)
    grads = {k: t.cpu() for k, t in ts.named_gradients().items()}
    new = {k: t.cpu() for k, t in ts.state_dict().items()}
    wn, se = _check_digest('fixed_' if fixed_radius else 'radius_', grads, new, float(losses[0]),
                           ts.last_logits.cpu().numpy(), tol=5e-2)
    ref = trorc.train_iteration(sd, batch, V['use_point_stn'], V['shared_transformer'], lr=0.01, momentum=0.9,
                                dtype=torch.float64, outputs=trorc.REGRESSION, fixed_radius=fixed_radius)
    wt, glob = compare_gradients_l2(grads, ref['grads'], tol_tensor=1.5e-1, tol_global=5e-2)
    print('fixed_radius %s digest: worst norm err %.4f, sample rel-L2 %.4f | oracle: worst tensor rel-L2 %.4f, global %.4f'
          % (fixed_radius, wn, se, wt, glob))


def test_cuda_graph_replay_matches_eager_steps():
    # the bars of test_gpu_train.test_cuda_graph_replay_matches_eager_steps, over two steps like there.  The second batch
    # is the first one with the signed distances negated, so only imp_surf_ms tells the two apart: a replay that did not
    # copy it would train on the first batch's targets again.
    sd = synth.make_state_dict(VARIANT, seed=41)
    b1 = make_regression_train_batch(16, seed=7)
    batches = [_cuda(b1), _cuda(dict(b1, imp_surf_ms=-b1['imp_surf_ms']))]
    eager = _step(sd, lr=1e-3)
    le = [float(eager.step(b)[0]) for b in batches]
    graph = _step(sd, lr=1e-3)
    before = graph.flat_params.clone()
    graph.capture_graph(batches[0])
    assert 'imp_surf_ms' in graph._graph[2] and 'imp_surf_magnitude_ms' not in graph._graph[2]
    assert torch.equal(graph.flat_params, before) and graph.steps_done == 0
    lg = [float(graph.step(b)[0]) for b in batches]
    print('eager losses', le, 'graph losses', lg)
    for a, b in zip(le, lg):
        assert abs(a - b) < 5e-3 * abs(b), (le, lg)
    assert abs(lg[1] - lg[0]) > 0.1 * lg[0]
    moved_e, moved_g = eager.flat_params - before, graph.flat_params - before
    assert float((moved_e - moved_g).norm()) <= 5e-2 * float(moved_e.norm())
    assert int(graph.buffers['bn2.num_batches_tracked']) == 102 and graph.steps_done == 2
    close(graph.buffers['bn2.running_mean'], eager.buffers['bn2.running_mean'], 1e-3, 'running mean after graph steps')


def _sphere_batch(n, seed):
    """n queries around synth's r = 0.5 sphere with their true signed distance (+ inside, the convention of the fitted
    regression head), assembled by the training entry point's GPU assembler (kNN patch, weighted sub-sample)."""
    from points2surf_b200.points_to_surf_train import GpuAssembler
    cloud = synth.make_cloud('sphere', 6000, seed=2)
    rng = np.random.RandomState(seed)
    q = (cloud[rng.choice(len(cloud), n, replace=False)] + rng.normal(0, 0.03, (n, 3))).astype(np.float32)
    d = (0.5 - np.linalg.norm(q, axis=1)).astype(np.float32)
    patch, radius, sub, qd = GpuAssembler(torch.device(DEV), 300, 1000, 0, seed).assemble('sphere', cloud, q)
    dt = torch.from_numpy(d).to(DEV)
    return {'patch_pts_ps': patch, 'patch_radius_ms': radius, 'pts_sub_sample_ms': sub, 'imp_surf_query_point_ms': qd,
            'imp_surf_ms': dt, 'imp_surf_magnitude_ms': dt.abs(), 'imp_surf_dist_sign_ms': (dt >= 0).float()}


def test_overfits_one_batch_of_sphere_queries():
    # measured on an H100 80GB HBM3 (700 W), every fifth step: 0.3471 0.2278 0.0716 0.0204 0.0063 0.0022, and 0.0010 at
    # step 30 (0.3 % of the first loss); a second run (fp32 atomics make runs differ): 0.3471 0.2121 0.0625 0.0150 0.0051
    # 0.0020, and 0.0012 at step 30.  The bars leave a factor 6 or more.
    batch = _sphere_batch(256, 5)
    ts = _step(synth.make_state_dict(VARIANT, seed=0), lr=0.01, momentum=0.9)
    curve = [float(ts.step(batch)[0]) for _ in range(30)]
    print('regression loss over 30 steps:', ' '.join('%.4f' % c for c in curve))
    assert all(np.isfinite(curve))
    assert min(curve[10:15]) < 0.5 * curve[0] and curve[-1] < 0.02 * curve[0], curve


def test_train_then_eval_hand_over(tmp_path):
    # experiments/train_p2s_regression.sh at a small size, refining the fitted regression checkpoint (saved as epoch 48, so
    # the run trains epoch 49 and writes _model_49.pth), then experiments/eval_p2s_regression.sh on what it wrote
    import os
    from points2surf_b200 import eval as p2s_eval, points_to_surf_train as p2s_train
    from test_gpu_regression import _script_args
    root = tmp_path / 'data'
    for sub in ('04_pts', '05_query_pts', '05_query_dist'):
        (root / sub).mkdir(parents=True)
    rng = np.random.RandomState(0)
    names = ['s0', 's1', 's2']
    for i, name in enumerate(names):
        cloud = synth.make_cloud('sphere', 2000, seed=i)
        q = (cloud[rng.choice(2000, 64, replace=False)] + rng.normal(0, 0.02, (64, 3))).astype(np.float32)
        np.save(root / '04_pts' / (name + '.xyz.npy'), cloud)
        np.save(root / '05_query_pts' / (name + '.ply.npy'), q)
        np.save(root / '05_query_dist' / (name + '.ply.npy'), (0.5 - np.linalg.norm(q, axis=1)).astype(np.float32))
    (root / 'trainset.txt').write_text('s0\ns1\n')
    (root / 'valset.txt').write_text('s2\n')
    (root / 'testset.txt').write_text('s2\n')
    start = tmp_path / 'start'
    start.mkdir()
    torch.save(synth.make_state_dict(VARIANT, 10, module_prefix='module.', fitted=True), start / 'p2s_regression_model_48.pth')
    models = tmp_path / 'models'
    opt = p2s_train.parse_arguments([
        '--name', 'p2s_regression', '--desc', 'p2s_regression', '--indir', str(root), '--outdir', str(models),
        '--logdir', str(tmp_path / 'logs'), '--trainset', 'trainset.txt', '--testset', 'valset.txt', '--nepoch', '50',
        '--lr', '0.01', '--scheduler_steps', '75', '125', '--debug', '0', '--workers', '22', '--batchSize', '16',
        '--points_per_patch', '300', '--patches_per_shape', '32', '--sub_sample_size', '1000', '--cache_capacity', '30',
        '--patch_radius', '0.0', '--single_transformer', '0', '--shared_transformer', '0', '--uniform_subsample', '0',
        '--use_point_stn', '1', '--patch_center', 'mean', '--training_order', 'random_shape_consecutive',
        '--outputs', 'imp_surf', 'patch_pts_ids', 'p_index', '--refine', str(start / 'p2s_regression_model_48.pth')])
    hist = p2s_train.points_to_surf_train(opt)
    assert len([h for h in hist if h[0] == 'train']) == 4 and all(len(h[3]) == 1 and np.isfinite(h[3]).all() for h in hist)
    sd = torch.load(models / 'p2s_regression_model_49.pth')
    assert tuple(sd['module.fc4.weight'].shape) == (1, 128)
    out = tmp_path / 'results'
    res = 32
    eopt = p2s_eval.parse_arguments(_script_args(root, out, models, res))
    eopt.reconstruction = True
    p2s_eval.points_to_surf_eval(eopt)
    rec = out / 'rec'
    q = np.load(rec / 'query_pts_ms' / 's2.xyz.npy')
    d = np.load(rec / 'dist_ms' / 's2.xyz.npy')
    print('hand-over: %d queries, %d inside, %d outside' % (d.size, int((d > 0).sum()), int((d < 0).sum())))
    assert d.dtype == np.float32 and d.shape == (q.shape[0],) and np.isfinite(d).all()
    assert (d > 0).any() and (d < 0).any()
    for f in ('eval/s2.xyz.npy', 'eval/s2.xyz.txt', 'vis/s2.ply', 'query_pts_ms_vis/s2.ply'):
        assert os.path.exists(rec / f), f
    assert np.array_equal(np.load(rec / 'eval' / 's2.xyz.npy'), d)
