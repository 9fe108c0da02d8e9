"""GPU: the regression ablation (outputs imp_surf patch_pts_ids p_index, experiments/eval_p2s_regression.sh) -- both
engines with the output_dim 1 head against the reference's fixture, the regression post-process kernel against torch's
formula, the fused reconstruction and its mesh against the reference path (oracle) on the GPU's own sub-sample ids, slab
and batch invariance, and points_to_surf_eval with the script's flags.

The end-to-end checkpoint is synth's 'regression' variant with its fitted fc4 (a ridge fit onto the inverse
post-process of a sphere's signed distance), so the SDF describes a surface and the mesh comparison means something."""
import numpy as np
import pytest
import torch

from oracle import p2s_oracle as orc
from oracle import mc_oracle as mc
from points2surf_b200 import synth, ops, evaluation
from points2surf_b200 import eval as p2s_eval
from test_regression_host import regression_case
import regression_oracle as rorc

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
VARIANT = 'regression'
V = synth.VARIANTS[VARIANT]
MODEL_SEED = 10
SEED = 40938661
FP32_AMBIGUOUS = 2e-3


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def engine(sd, precision, guard_band=0.05):
    return ops.Engine(sd, V['use_point_stn'], V['shared_transformer'], precision=precision, guard_band=guard_band,
                      output_dim=1)


# ------------------------------------------------------------------ engines against the reference's fixture
def test_engines_match_reference_fixture():
    sd, inp, g = regression_case()
    ref = g['logits']
    args = [cu(inp[k]) for k in ('patch_pts_ps', 'pts_sub_sample_ms', 'imp_surf_query_point_ms')]
    e32 = engine(sd, 'fp32', 0.0)
    lo32 = e32.forward(*args).cpu().numpy()
    assert lo32.shape == ref.shape == (int(g['batch']), 1)
    err32 = float(np.abs(lo32 - ref).max())
    host = e32.forward_host(*[inp[k] for k in ('patch_pts_ps', 'pts_sub_sample_ms', 'imp_surf_query_point_ms')])
    assert np.array_equal(host, lo32)
    e32.close()
    etc = engine(sd, 'tc', 0.0)
    lotc = etc.forward(*args).cpu().numpy()
    errtc = float(np.abs(lotc - ref).max())
    etc.set_precision('tc', 0.05)                        # the default guard band of eval / PointsToSurfModel
    log = etc.forward(*args).cpu().numpy()
    n_guard = etc.last_guard_count()
    etc.close()
    decided = np.abs(ref[:, 0]) > FP32_AMBIGUOUS
    mism = int(((log[:, 0] > 0) != (ref[:, 0] > 0))[decided].sum())
    print('regression fixture: fp32 max |dl| %.3g, tc max |dl| %.3g, guard band recomputed %d of %d, sign mismatches %d'
          % (err32, errtc, n_guard, len(ref), mism))
    assert err32 <= 2e-3
    assert errtc <= 3e-2 * max(1.0, float(np.abs(ref).max()))
    assert n_guard == int((np.abs(lotc[:, 0]) < 0.05).sum()) and n_guard > 0
    assert mism == 0


def test_model_module_regression_head():
    from points2surf_b200.model import PointsToSurfModel
    sd, inp, g = regression_case()
    m = PointsToSurfModel(net_size_max=1024, num_points=300, output_dim=1, use_point_stn=True, use_feat_stn=True,
                          sym_op='max', use_query_point=True, sub_sample_size=1000, do_augmentation=False,
                          single_transformer=0, shared_transformation=False, precision='fp32')
    m.load_state_dict({'module.' + k: v for k, v in sd.items()})
    x = {k: cu(a.copy()) for k, a in inp.items()}
    y = m(x)
    assert tuple(y.shape) == (int(g['batch']), 1)
    assert float(np.abs(y.cpu().numpy() - g['logits']).max()) <= 2e-3


# ------------------------------------------------------------------ post-process kernel
def _ulp_diff(a, b):
    ia = a.view(np.int32).astype(np.int64)
    ib = b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)          # monotone integer order of the floats (+0 and -0 coincide)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


@pytest.mark.parametrize('fixed_radius', [False, True])
def test_distance_from_logits_kernel(fixed_radius):
    rng = np.random.RandomState(5)
    tiny = np.finfo(np.float32).smallest_subnormal
    special = np.array([0.0, -0.0, tiny, -tiny, 1e-3, -1e-3, 20.0, -20.0, np.inf, -np.inf, np.nan], np.float32)
    lg = np.concatenate([special, (rng.standard_normal(100000) * 3).astype(np.float32),
                         np.float32(np.logspace(-30, 1.5, 2000)) * rng.choice([-1, 1], 2000).astype(np.float32)])
    r = rng.uniform(0.005, 0.5, lg.size).astype(np.float32)
    lt = cu(lg).unsqueeze(1)
    rt = None if fixed_radius else cu(r)
    got = ops.distance_from_logits(lt, rt).cpu().numpy()
    ref = torch.tanh(lt).pow(2) * torch.sign(lt)                                     # source/sdf_nn.py:6-8
    if rt is not None:
        ref = ref * rt.unsqueeze(1)                                                  # points_to_surf_eval.py:180-181
    ref = ref[:, 0].cpu().numpy()
    nan = np.isnan(ref)
    assert np.array_equal(nan, np.isnan(lg))
    assert (got[nan] == 1.0).all()                                                    # points_to_surf_eval.py:205-207
    assert got[0] == 0.0 and got[1] == 0.0
    d = _ulp_diff(got[~nan], ref[~nan])
    print('distance_from_logits: max %d ulp from torch over %d logits' % (int(d.max()), int((~nan).sum())))
    assert d.max() <= 2
    big = np.abs(lg) > 1e-15                                  # tanh(l)^2 (times the radius) does not underflow
    assert np.array_equal(np.sign(got[big]), np.sign(lg[big]))
    if fixed_radius:
        assert got[6] == 1.0 and got[7] == -1.0 and np.abs(got[~nan]).max() <= 1.0   # not rescaled
    # the magnitude/sign post-process is a different rule: the regression kernel must not be confused with it
    with pytest.raises(ops.P2SError):
        ops.distance_from_logits(cu(np.zeros((4, 2), np.float32)), None)


# ------------------------------------------------------------------ fused reconstruction, end to end
@pytest.fixture(scope='module')
def sphere_case():
    """res 64 on the fitted regression checkpoint: the fused call (tc, default guard band) and the reference path over
    every query on the GPU's own patches and sub-sample ids (fp32 CPU oracle network + regression post-process)."""
    res, eps = 64, 3
    cloud = synth.make_cloud('sphere', 10000, seed=0)
    sd = synth.make_state_dict(VARIANT, MODEL_SEED, fitted=True)
    eng = engine(sd, 'tc')
    pts = cu(cloud)
    lin, sdf = eng.reconstruct(pts, res, eps, 0, SEED)
    n_guard = eng.last_guard_count()
    eng.close()
    qd = ops.query_points(lin, res)
    qpts = qd.cpu().numpy()
    assert np.array_equal(qpts, orc.query_grid(cloud, res, eps))
    Q = len(qpts)
    logits = np.empty((Q, 1), np.float32)
    radius = np.empty((Q,), np.float32)
    for b in range(0, Q, 512):
        q = qd[b:b + 512]
        _, patch, r = ops.knn_patch(pts, q, 300)
        sub = ops.gather_points(pts, ops.subsample(pts, q, 1000, False, SEED, query_index_base=b))
        logits[b:b + 512] = orc.model_forward(sd, patch.cpu().numpy(), sub.cpu().numpy(), qpts[b:b + 512],
                                              V['use_point_stn'], V['shared_transformer'])
        radius[b:b + 512] = r.cpu().numpy()
    return dict(res=res, cloud=cloud, lin=lin, sdf=sdf, qpts=qpts, logits=logits, sdf_o=rorc.post_process_distance(logits, radius),
                n_guard=n_guard)


def test_fused_reconstruction_against_reference_path(sphere_case):
    c = sphere_case
    voxel = 2.0 / c['res']
    got = c['sdf'].cpu().numpy()
    lo, sdf_o = c['logits'][:, 0], c['sdf_o']
    decided = np.abs(lo) > FP32_AMBIGUOUS
    mism = int(((got > 0) != (sdf_o > 0))[decided].sum())
    dv = np.abs(got - sdf_o) / voxel
    print('regression res %d: Q %d, guard recompute %d, fp32-ambiguous %d, positive fraction %.3f, sign mismatches %d, '
          '|dSDF| max %.4f mean %.5f voxel' % (c['res'], len(got), c['n_guard'], int((~decided).sum()), (got > 0).mean(),
                                               mism, dv.max(), dv.mean()))
    assert (got > 0).any() and (got < 0).any()
    assert mism == 0
    assert dv.max() <= 0.25, dv.max()


def test_mesh_against_reference_path(sphere_case):
    c = sphere_case
    res = c['res']
    voxel = 2.0 / res
    vol, _ = ops.sdf_to_volume(c['lin'], c['sdf'], res, 5, 13.0)
    verts, faces = ops.marching_cubes(vol, 0.0)
    verts, faces = verts.cpu().numpy(), faces.cpu().numpy()
    vol_o = orc.sdf_to_volume(c['sdf_o'].astype(np.float32), c['qpts'], res, 5, 13)
    vo, fo = mc.marching_cubes(vol_o.astype(np.float32), 0.0)
    assert len(faces) > 1000 and len(fo) > 1000, 'the fitted checkpoint must reconstruct a surface'
    rng = np.random.RandomState(0)
    s_eng = orc.sample_mesh_surface(verts, faces, 10000, rng)
    s_ref = orc.sample_mesh_surface(vo, fo, 10000, rng)
    s_ref2 = orc.sample_mesh_surface(vo, fo, 10000, rng)
    cd = orc.chamfer(s_eng, s_ref) / 20000.0
    floor = orc.chamfer(s_ref2, s_ref) / 20000.0
    print('regression mesh: engine %d faces, oracle %d faces; Chamfer per sample %.5f = %.3f voxel, sampling floor %.3f voxel'
          % (len(faces), len(fo), cd, cd / voxel, floor / voxel))
    assert cd <= floor + 0.05 * voxel, (cd, floor)


def test_slab_and_batch_invariance():
    cloud = synth.make_cloud('sphere', 10000, seed=0)
    sd = synth.make_state_dict(VARIANT, MODEL_SEED, fitted=True)
    eng = engine(sd, 'tc')
    pts = cu(cloud)
    lin, sdf = eng.reconstruct(pts, 128, 3, 0, SEED)
    Q = lin.numel()
    assert Q > 20000
    lin2, sdf2 = eng.reconstruct(pts, 128, 3, 0, SEED, batch=20000)
    assert torch.equal(lin, lin2) and torch.equal(sdf, sdf2), int((sdf != sdf2).sum())
    for first, num in ((0, 5000), (Q // 3, 12345), (Q - 777, 777)):
        l3, s3 = eng.reconstruct(pts, 128, 3, 0, SEED, first_query=first, num_queries=num)
        assert torch.equal(l3, lin[first:first + num]) and torch.equal(s3, sdf[first:first + num]), (first, num)
    lin4, sdf4 = eng.reconstruct_host(cloud, 128, 3, 0, SEED, cap=Q)
    assert np.array_equal(lin4, lin.cpu().numpy()) and np.array_equal(sdf4, sdf.cpu().numpy())
    eng.close()


# ------------------------------------------------------------------ eval entry point
def _regression_dataset(tmp_path):
    root = tmp_path / 'data'
    (root / '04_pts').mkdir(parents=True)
    clouds = {'sphere': synth.make_cloud('sphere', 6000, seed=2), 'torus': synth.make_cloud('torus', 5000, seed=3)}
    for name, cloud in clouds.items():
        np.save(root / '04_pts' / (name + '.xyz.npy'), cloud)
    (root / 'testset.txt').write_text('sphere\ntorus\n')
    models = tmp_path / 'models'
    models.mkdir()
    sd = synth.make_state_dict(VARIANT, MODEL_SEED, fitted=True)
    torch.save({'module.' + k: v for k, v in sd.items()}, models / 'p2s_regression_model_49.pth')
    torch.save(synth.make_train_opt(VARIANT), models / 'p2s_regression_params.pth')
    return root, models, sd, clouds


def _script_args(root, out, models, res):
    # experiments/eval_p2s_regression.sh, at a small grid resolution
    return ['--indir', str(root), '--outdir', str(out), '--modeldir', str(models), '--dataset', 'testset.txt',
            '--models', 'p2s_regression', '--modelpostfix', '_model_49.pth', '--batchSize', '501', '--workers', '7',
            '--cache_capacity', '5', '--query_grid_resolution', str(res), '--epsilon', '3', '--certainty_threshold', '13',
            '--sigma', '5']


def test_points_to_surf_eval_regression_script(tmp_path):
    from points2surf_b200 import mesh_io
    root, models, sd, clouds = _regression_dataset(tmp_path)
    out = tmp_path / 'results'
    res = 32
    opt = p2s_eval.parse_arguments(_script_args(root, out, models, res))
    opt.reconstruction = True
    p2s_eval.points_to_surf_eval(opt)
    rec = out / 'rec'
    eng = engine(sd, 'tc')
    for name, cloud in clouds.items():
        q = np.load(rec / 'query_pts_ms' / (name + '.xyz.npy'))
        d = np.load(rec / 'dist_ms' / (name + '.xyz.npy'))
        lin, sdf = eng.reconstruct(cu(cloud), res, 3, 0, SEED)
        assert np.array_equal(q, ops.query_points(lin, res).cpu().numpy())
        assert d.dtype == np.float32 and np.array_equal(d, sdf.cpu().numpy())
        assert (d > 0).any() and (d < 0).any()
        assert np.array_equal(np.load(rec / 'eval' / (name + '.xyz.npy')), d)
        assert np.loadtxt(rec / 'eval' / (name + '.xyz.txt')).shape == d.shape
        for sub in ('vis', 'query_pts_ms_vis'):
            v, f = mesh_io.read_ply(str(rec / sub / (name + '.ply')))
            assert v.shape == q.shape and len(f) == 0
    eng.close()

    # --reconstruction 0 on 05_query_pts (full_eval.py:31-41), then the reference's prediction report
    (root / '05_query_pts').mkdir()
    (root / '05_query_dist').mkdir()
    rng = np.random.RandomState(4)
    for name in clouds:
        q = rng.uniform(-0.7, 0.7, (300, 3)).astype(np.float32)
        np.save(root / '05_query_pts' / (name + '.ply.npy'), q)
        np.save(root / '05_query_dist' / (name + '.ply.npy'), (0.5 - np.linalg.norm(q, axis=1)).astype(np.float32))
    opt = p2s_eval.parse_arguments(_script_args(root, out, models, res))
    p2s_eval.points_to_surf_eval(opt)
    pred = out / 'eval' / 'eval'
    for name in clouds:
        d = np.load(pred / (name + '.xyz.npy'))
        assert d.shape == (300,) and np.isfinite(d).all() and (np.abs(d) <= 1.0).all()
    report = tmp_path / 'report.csv'
    evaluation.eval_predictions(str(pred), str(root / '05_query_dist'), str(report))
    text = report.read_text()
    assert all((name + '.xyz.npy')[:10] in text for name in clouds)          # print_list_of_dicts keeps 10 characters

    # --sampling sequential_shapes_random_patches: a random subset of 05_query_pts, indices saved beside the results
    opt = p2s_eval.parse_arguments(_script_args(root, tmp_path / 'results_seq', models, res) +
                                   ['--sampling', 'sequential_shapes_random_patches', '--patches_per_shape', '40'])
    p2s_eval.points_to_surf_eval(opt)
    for name in clouds:
        idx = np.loadtxt(tmp_path / 'results_seq' / 'eval' / (name + '.idx'), dtype=np.int64)
        assert np.load(tmp_path / 'results_seq' / 'eval' / 'eval' / (name + '.xyz.npy')).shape == idx.shape == (40,)
