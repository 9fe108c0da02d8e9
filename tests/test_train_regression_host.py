"""Host logic of the regression ablation's training (outputs imp_surf patch_pts_ids p_index,
experiments/train_p2s_regression.sh) on the CPU: the fixture of the unmodified reference (tests/golden/train_regression.npz),
the hand-written backward of TrainStep with the one-output head against autograd over the training oracle, calc_metrics'
regression branch, the training entry point end to end, the output-list validation shared with the evaluation, and a
two-rank data-parallel step.  The CUDA loss kernel and the fp32 step are tested in tests/test_gpu_train_regression.py."""
import json
import multiprocessing as mp
import os
import socket
from argparse import Namespace

import numpy as np
import pytest
import torch
import torch.distributed as dist

import train_regression_oracle as trorc
from points2surf_b200 import eval as p2s_eval, points_to_surf_train as p2s_train, synth
from points2surf_b200.train import TrainStep, compute_loss
from helpers import load_golden
from helpers_train_regression import RegressionTorchPrims, make_regression_train_batch
from test_train_loop import OracleAssembler, _make_dataset

REGRESSION_OUTPUTS = ['imp_surf', 'patch_pts_ids', 'p_index']
FIXTURE_SEED = 24          # tests/golden/make_train_regression_golden.py
# output lists that evaluation rejects (tests/test_regression_host.py); training must reject them too
BAD_OUTPUTS = [
    ['imp_surf'],
    ['imp_surf', 'patch_pts_ids'],
    ['imp_surf', 'imp_surf_magnitude', 'imp_surf_sign', 'patch_pts_ids', 'p_index'],
    ['imp_surf', 'imp_surf_sign', 'patch_pts_ids', 'p_index'],
    ['imp_surf', 'imp_surf', 'patch_pts_ids', 'p_index'],
    ['imp_surf_magnitude', 'patch_pts_ids', 'p_index'],
]


def _relerr(a, b):
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def test_fixture_loads_and_batch_matches_its_checksum():
    g = load_golden('train_regression.npz')
    batch = make_regression_train_batch(int(g['batch']), 300, 1000, seed=FIXTURE_SEED)
    assert sum(float(t.double().abs().sum()) for t in batch.values()) == float(g['input_checksum'])
    assert np.array_equal(batch['imp_surf_ms'].abs().numpy(), batch['imp_surf_magnitude_ms'].numpy())
    assert np.array_equal((batch['imp_surf_ms'] >= 0).numpy(), batch['imp_surf_dist_sign_ms'].numpy() == 1)
    for pre in ('radius_', 'fixed_'):
        assert g[pre + 'logits'].shape == (32, 1) and g[pre + 'losses'].shape == (1,)
        assert [str(n) for n in g[pre + 'names']] == sorted(k for k in synth.make_state_dict('regression', 0)
                                                            if not k.endswith(('running_mean', 'running_var', 'num_batches_tracked')))


def test_initialisation_of_the_one_output_head_matches_reference():
    g = load_golden('train_regression.npz')
    v = synth.VARIANTS['regression']
    torch.manual_seed(int(g['init_seed']))
    sd = p2s_train.initial_state_dict(v['use_point_stn'], v['shared_transformer'], 1024, 1)
    names = [str(n) for n in g['init_names']]
    assert [k for k in sd if sd[k].is_floating_point()] == names
    assert tuple(sd['fc4.weight'].shape) == (1, 128) and tuple(sd['fc4.bias'].shape) == (1,)
    assert np.array_equal(np.array([float(sd[k].double().sum()) for k in names]), g['init_sums'])
    assert np.array_equal(np.array([float(sd[k].reshape(-1)[0]) for k in names]), g['init_first'])


def _step_against_oracle(fixed_radius, steps):
    v = synth.VARIANTS['regression']
    P, S, B = 20, 30, 5          # small point counts: the sequencing is size-independent
    sd = synth.make_state_dict('regression', seed=3)
    batches = [make_regression_train_batch(B, P, S, seed=1 + i) for i in range(steps)]
    ts = TrainStep(sd, v['use_point_stn'], v['shared_transformer'], points_per_patch=P, sub_sample_size=S, lr=0.01,
                   momentum=0.9, device='cpu', prims=RegressionTorchPrims(), outputs=('imp_surf',),
                   output_loss_weights={'imp_surf': 1.0}, fixed_radius=fixed_radius, dtype=torch.float64)
    state, mom = sd, None
    for b in batches:
        ref = trorc.train_iteration(state, b, v['use_point_stn'], v['shared_transformer'], lr=0.01, momentum=0.9,
                                    mom_bufs=mom, dtype=torch.float64, outputs=trorc.REGRESSION, fixed_radius=fixed_radius)
        losses = ts.step({k: t.double() for k, t in b.items()})
        state = dict(state)
        state.update(ref['new_state'])
        mom = ref['mom_bufs']
    return ts, ref, losses


@pytest.mark.parametrize('fixed_radius', [False, True])
def test_hand_written_backward_matches_autograd(fixed_radius):
    ts, ref, losses = _step_against_oracle(fixed_radius, 1)
    tol = 1e-8
    assert len(losses) == 1 and abs(float(losses[0]) - ref['losses'][0]) <= tol * abs(ref['losses'][0])
    assert tuple(ts.last_logits.shape) == (5, 1) and _relerr(ts.last_logits, ref['logits']) < tol
    grads = ts.named_gradients()
    assert set(grads) == set(ref['grads'])
    assert tuple(grads['fc4.weight'].shape) == (1, 128)
    scale = max(float(r.abs().max()) for r in ref['grads'].values())
    bad = []
    for name, g in grads.items():
        r = ref['grads'][name]
        assert g.shape == r.shape, name
        # conv / fc biases in front of a BatchNorm have an exactly-zero gradient up to rounding: floor on the scale
        err = float((g - r).abs().max()) / (float(r.abs().max()) + 1e-6 * scale)
        if err > tol:
            bad.append((name, err))
    assert not bad, bad
    new = ts.state_dict()
    for name, r in ref['new_state'].items():
        assert float((new[name] - r).abs().max()) <= tol * (1e-3 + float(r.abs().max())), name


@pytest.mark.parametrize('fixed_radius', [False, True])
def test_second_step_uses_momentum(fixed_radius):
    ts, ref, losses = _step_against_oracle(fixed_radius, 2)
    assert abs(float(losses[0]) - ref['losses'][0]) <= 1e-8 * abs(ref['losses'][0])
    new = ts.state_dict()
    for name, r in ref['new_state'].items():
        assert float((new[name] - r).abs().max()) <= 1e-9 * (1.0 + float(r.abs().max())), name


def test_compute_loss_checks_the_head_before_reading_the_batch():
    p = RegressionTorchPrims()
    for pred, outs in ((torch.zeros(2, 2), ['imp_surf']), (torch.zeros(2, 1), ['imp_surf_magnitude', 'imp_surf_sign']),
                       (torch.zeros(2), ['imp_surf']), (torch.zeros(2, 1), ['imp_surf_magnitude']),
                       (torch.zeros(2, 1), ['imp_surf_sign']), (torch.zeros(2, 3), ['imp_surf', 'imp_surf_magnitude', 'imp_surf_sign'])):
        with pytest.raises(ValueError):
            compute_loss(pred, {}, outs, {}, False, prims=p)
    b = make_regression_train_batch(4, 8, 8, seed=3)
    pred = torch.linspace(-2, 2, 4).reshape(4, 1)
    (l,), d = compute_loss(pred, b, ['imp_surf'], {'imp_surf': 0.5}, False, prims=p, need_grad=True)
    t = b['imp_surf_ms'] / b['patch_radius_ms']
    assert abs(float(l) - 0.5 * float(((torch.tanh(pred[:, 0]) - torch.tanh(t)) ** 2).mean())) < 1e-7
    assert tuple(d.shape) == (4, 1)


def test_calc_metrics_matches_reference_fixture():
    g = load_golden('train_regression.npz')
    batch = make_regression_train_batch(32, 300, 1000, seed=FIXTURE_SEED)
    for pre, fixed_radius in (('radius_', False), ('fixed_', True)):
        want = json.loads(str(g[pre + 'metrics_json']))
        logits = torch.from_numpy(g[pre + 'logits'].copy())
        before = {k: t.clone() for k, t in batch.items()}
        got = p2s_train.calc_metrics(logits, batch, fixed_radius=fixed_radius)
        assert torch.equal(logits, torch.from_numpy(g[pre + 'logits']))
        assert all(torch.equal(batch[k], before[k]) for k in batch)
        assert abs(got['abs_dist_rms'] - want['abs_dist_rms']) <= 1e-6
        assert set(got) == set(want)
        for k, w in want.items():
            if k != 'abs_dist_rms':
                assert got[k] == w, (k, got[k], w)


def test_calc_metrics_sign_rule_on_special_logits():
    logits = torch.tensor([[float('nan')], [-0.0], [0.0], [2.0], [-3.0]])
    batch = {'imp_surf_ms': torch.tensor([-0.1, 0.1, 0.1, 0.2, -0.2]), 'patch_radius_ms': torch.full((5,), 0.5),
             'imp_surf_dist_sign_ms': torch.tensor([0.0, 1.0, 1.0, 1.0, 0.0])}
    lb = logits.clone()
    bb = {k: t.clone() for k, t in batch.items()}
    m = p2s_train.calc_metrics(logits, batch)
    # NaN -> -1, -0.0 -> +1, 0.0 -> +1 (points_to_surf_train.py:589-591 then sdf_nn.post_process_sign)
    assert m['positives'] == 3.0 and m['true_pos'] == 3.0 and m['true_neg'] == 2.0 and m['accuracy'] == 1.0
    assert torch.equal(logits[1:], lb[1:]) and torch.isnan(logits[0, 0]) and torch.signbit(logits[1, 0])
    assert all(torch.equal(batch[k], bb[k]) for k in batch)
    m2 = p2s_train.calc_metrics(logits[1:], {k: t[1:] for k, t in batch.items()}, fixed_radius=True)
    want = torch.sqrt(torch.mean((torch.tanh(logits[1:, 0]) ** 2 - batch['imp_surf_ms'][1:].abs()) ** 2))
    assert abs(m2['abs_dist_rms'] - float(want)) < 1e-7


def _regression_args(tmp_path, root, extra=()):
    return ['--name', 'test', '--indir', root, '--outdir', str(tmp_path / 'models'), '--logdir', str(tmp_path / 'logs'),
            '--nepoch', '2', '--batchSize', '5', '--patches_per_shape', '8', '--points_per_patch', '16',
            '--sub_sample_size', '24', '--patch_radius', '0.0', '--lr', '0.01', '--scheduler_steps', '75', '125',
            '--single_transformer', '0', '--shared_transformer', '0', '--uniform_subsample', '0', '--use_point_stn', '1',
            '--patch_center', 'mean', '--training_order', 'random_shape_consecutive',
            '--outputs', 'imp_surf', 'patch_pts_ids', 'p_index', '--save_interval', '1'] + list(extra)


def test_two_epochs_end_to_end(tmp_path, capsys):
    root = str(tmp_path / 'data')
    _make_dataset(root, ['s0', 's1', 's2'])
    opt = p2s_train.parse_arguments(_regression_args(tmp_path, root))
    hist = p2s_train.points_to_surf_train(opt, prims=RegressionTorchPrims(), assembler=OracleAssembler(16, 24, 0, 1),
                                          device=torch.device('cpu'))
    out = capsys.readouterr().out
    assert 'Training set: 16 patches (in 4 batches) | Test set: 8 patches (in 2 batches)' in out
    lines = [ln for ln in out.splitlines() if '[test ' in ln]
    assert lines and all('rmse: ' in ln and 'f1: ' in ln for ln in lines)
    assert len([h for h in hist if h[0] == 'train']) == 8 and len([h for h in hist if h[0] == 'test']) == 4
    assert all(len(l) == 1 and np.isfinite(l).all() for _, _, _, l in hist)
    models = tmp_path / 'models'
    for f in ('test_params.pth', 'test_model.pth'):
        assert (models / f).exists(), f
    assert torch.load(models / 'test_params.pth', weights_only=False).outputs == REGRESSION_OUTPUTS
    sd = torch.load(models / 'test_model.pth')
    assert tuple(sd['module.fc4.weight'].shape) == (1, 128) and tuple(sd['module.fc4.bias'].shape) == (1,)
    assert sorted(sd.keys()) == sorted('module.' + k for k in synth.make_state_dict('regression', 0).keys())
    assert int(sd['module.bn2.num_batches_tracked']) == 8


def test_refine_checks_the_head_of_the_checkpoint(tmp_path):
    root = str(tmp_path / 'data')
    _make_dataset(root, ['s0', 's1', 's2'])
    two = str(tmp_path / 'uniform_model_3.pth')
    torch.save(synth.make_state_dict('uniform', 0, module_prefix='module.'), two)
    opt = p2s_train.parse_arguments(_regression_args(tmp_path, root, ['--refine', two]))
    with pytest.raises(ValueError):
        p2s_train.points_to_surf_train(opt, prims=RegressionTorchPrims(), assembler=OracleAssembler(16, 24, 0, 1),
                                       device=torch.device('cpu'))
    one = str(tmp_path / 'regression_model_3.pth')
    torch.save(synth.make_state_dict('regression', 0, module_prefix='module.'), one)
    args = _regression_args(tmp_path, root, ['--refine', one, '--nepoch', '5'])
    opt = p2s_train.parse_arguments(args)
    hist = p2s_train.points_to_surf_train(opt, prims=RegressionTorchPrims(), assembler=OracleAssembler(16, 24, 0, 1),
                                          device=torch.device('cpu'))
    assert sorted({h[1] for h in hist}) == [4]                         # resumes after epoch 3 of the file name
    k = args.index('--outputs')
    opt = p2s_train.parse_arguments(args[:k] + ['--outputs', 'imp_surf_magnitude', 'imp_surf_sign'] + args[k + 4:])
    with pytest.raises(ValueError):
        p2s_train.points_to_surf_train(opt, prims=RegressionTorchPrims(), assembler=OracleAssembler(16, 24, 0, 1),
                                       device=torch.device('cpu'))
    with pytest.raises(ValueError):
        TrainStep(synth.make_state_dict('uniform', 0), 1, 0, device='cpu', prims=RegressionTorchPrims(), outputs=('imp_surf',))


def test_training_and_evaluation_accept_the_same_output_lists():
    script = p2s_train.parse_arguments(_regression_args(__import__('pathlib').Path('/nonexistent'), 'data'))
    p2s_train._check_supported(script)
    p2s_eval._check_supported(Namespace(**vars(script)), p2s_eval.parse_arguments([]))
    for outs in BAD_OUTPUTS:
        opt = Namespace(**{**vars(script), 'outputs': outs})
        with pytest.raises(ValueError):
            p2s_train._check_supported(opt)
        with pytest.raises(ValueError):
            p2s_eval._check_supported(opt, p2s_eval.parse_arguments([]))
    for outs in (['patch_pts_ids', 'imp_surf', 'p_index'], ['imp_surf_magnitude', 'imp_surf_sign'],
                 ['imp_surf_magnitude', 'imp_surf_sign', 'patch_pts_ids', 'p_index']):
        opt = Namespace(**{**vars(script), 'outputs': outs})
        p2s_train._check_supported(opt)
        p2s_eval._check_supported(opt, p2s_eval.parse_arguments([]))


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _local_step(rank):
    ts = TrainStep(synth.make_state_dict('regression', seed=4), 1, 0, points_per_patch=16, sub_sample_size=24, device='cpu',
                   prims=RegressionTorchPrims(), outputs=('imp_surf',), dtype=torch.float64)
    ts.step({k: t.double() for k, t in make_regression_train_batch(4, 16, 24, seed=60 + rank).items()})
    return ts


def _train_worker(rank, world, port, q):
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        ts = _local_step(rank)
        q.put((rank, ts.flat_params.clone().numpy(), ts.flat_grads.clone().numpy()))
    finally:
        dist.destroy_process_group()


def test_data_parallel_regression_step_gloo():
    """Two ranks, different shards: both end with the same parameters, and the applied gradient is the mean of the two
    per-rank gradients of the regression loss (computed again in this process without a process group)."""
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_train_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=180) for _ in procs), key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert np.array_equal(res[0][1], res[1][1]) and np.array_equal(res[0][2], res[1][2])
    local = [_local_step(rank).flat_grads.clone().numpy() for rank in range(2)]
    assert not np.array_equal(local[0], local[1])
    np.testing.assert_allclose(res[0][2], 0.5 * (local[0] + local[1]), rtol=1e-12, atol=1e-14)
