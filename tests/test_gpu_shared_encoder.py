"""GPU: the shared-encoder ablation (single_transformer=1, experiments/eval_p2s_shared_encoder.sh).

a. Both engines against the reference's fixture (tests/golden/shared_encoder.npz): logits, the rotation and the max
   feature; the tensor-core path also with its FC layers on the fp32 kernels (P2S_FC_FP32=1) and with the guard band
   recomputed on the fp32 path (P2S_GUARD_FP32=1).
b. Per element: every max feature, rotation entry and logit of 'fp32', 'tc' without the guard band and the split-precision
   recompute (guard band 1e9) lies within oracle/net_bound.py's bound of the float64 network (restated for this network
   in tests/shared_encoder_oracle.py), for patch / sub-sample sizes around the tile size.  This covers the pass kernel's
   launch with two segments, a rotation and the per-query conv1 * (T + I) image, which only this network makes.
c. Logits do not depend on batch position, batch size, slab or the fused pipeline's batch.
d. The fused reconstruction of a sphere with the fitted checkpoint against the reference path (fp32 CPU oracle on the
   GPU's own patches and sub-sample ids), and its mesh.
e. points_to_surf_eval with the script's flags in both reconstruction modes, and through the source/ drop-in package."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import net_bound as nb
from oracle import p2s_oracle as orc
from oracle import mc_oracle as mc
from points2surf_b200 import synth, ops
from points2surf_b200 import eval as p2s_eval
from test_shared_encoder_host import shared_encoder_case
import shared_encoder_oracle as sorc

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
VARIANT = 'shared_encoder'
MODEL_SEED = 12
SEED = 40938661
FP32_AMBIGUOUS = 2e-3
KEYS = ('patch_pts_ps', 'pts_sub_sample_ms', 'imp_surf_query_point_ms')
ENGINES = {'fp32': dict(precision='fp32'), 'tc': dict(precision='tc', guard_band=0.0),
           'tc_precise': dict(precision='tc', guard_band=1e9)}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def engine(sd, P=300, S=1000, **kw):
    return ops.Engine(sd, 1, 0, points_per_patch=P, sub_sample_size=S, single_transformer=True, **kw)


# ------------------------------------------------------------------ a. engines against the reference's fixture
def _fixture_errors(eng, args, g):
    lo, aux = eng.forward_with_aux(*args)
    plain = eng.forward(*args)
    return (plain.cpu().numpy(), float(np.abs(aux['trans'].cpu().numpy() - g['trans']).max()),
            float(np.abs(aux['feat_max'].cpu().numpy() - g['feat_max']).max()))


def test_engines_match_reference_fixture():
    sd, inp, g = shared_encoder_case()
    ref = g['logits']
    args = [cu(inp[k]) for k in KEYS]
    fscale = max(1.0, float(np.abs(g['feat_max']).max()))
    e32 = engine(sd, precision='fp32')
    lo32, dR32, df32 = _fixture_errors(e32, args, g)
    assert np.array_equal(e32.forward_host(*[inp[k] for k in KEYS]), lo32)
    e32.close()
    etc = engine(sd, precision='tc', guard_band=0.0)
    lotc, dRtc, dftc = _fixture_errors(etc, args, g)
    etc.set_precision('tc', 0.05)                        # the default guard band of eval
    log = etc.forward(*args).cpu().numpy()
    n_guard = etc.last_guard_count()
    etc.close()
    os.environ['P2S_FC_FP32'] = '1'                      # read when the engine is built
    try:
        efc = engine(sd, precision='tc', guard_band=0.0)
    finally:
        del os.environ['P2S_FC_FP32']
    lofc, dRfc, dffc = _fixture_errors(efc, args, g)
    efc.close()
    err = {k: float(np.abs(x - ref).max()) for k, x in (('fp32', lo32), ('tc', lotc), ('tc fc-fp32', lofc))}
    decided = np.abs(ref[:, 1]) > FP32_AMBIGUOUS
    mism = int(((log[:, 1] > 0) != (ref[:, 1] > 0))[decided].sum())
    print('shared encoder fixture: max |dlogit| %s; |dR| fp32 %.3g tc %.3g tc-fc-fp32 %.3g; |dfeat| fp32 %.3g tc %.3g '
          'tc-fc-fp32 %.3g (scale %.3g); guard band recomputed %d of %d, sign mismatches %d'
          % (err, dR32, dRtc, dRfc, df32, dftc, dffc, fscale, n_guard, len(ref), mism))
    tol_tc = 3e-2 * max(1.0, float(np.abs(ref).max()))
    assert err['fp32'] <= 2e-3 and err['tc'] <= tol_tc and err['tc fc-fp32'] <= tol_tc
    assert dR32 <= 1e-4 and df32 <= 1e-4 * fscale
    assert dRtc <= 1e-2 and dftc <= 1e-2 * fscale and dRfc <= 1e-2 and dffc <= 1e-2 * fscale
    assert n_guard == int((np.abs(lotc[:, 1]) < 0.05).sum())
    assert mism == 0


_GUARD_FP32_SCRIPT = r'''
import json, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + '/tests')
import numpy as np, torch
from points2surf_b200 import ops
from test_shared_encoder_host import shared_encoder_case
sd, inp, g = shared_encoder_case()
args = [torch.from_numpy(inp[k]).cuda() for k in ('patch_pts_ps', 'pts_sub_sample_ms', 'imp_surf_query_point_ms')]
mk = lambda **kw: ops.Engine(sd, 1, 0, single_transformer=True, **kw)
e = mk(precision='tc', guard_band=1e9)
lg, aux = e.forward_with_aux(*args)
n = e.last_guard_count()
f = mk(precision='fp32')
l32, aux32 = f.forward_with_aux(*args)
print(json.dumps({'n': n, 'B': len(lg), 'fixture': float((lg.cpu() - torch.from_numpy(g['logits'])).abs().max()),
                  'vs_fp32': float((lg - l32).abs().max()), 'feat_vs_fp32': float((aux['feat_max'] - aux32['feat_max']).abs().max()),
                  'feat_scale': max(1.0, float(aux32['feat_max'].abs().max()))}))
'''


def test_guard_band_on_the_fp32_path():
    # P2S_GUARD_FP32=1 routes the guard-band recompute through forward_fp32; the variable is read once per process
    env = dict(os.environ, P2S_GUARD_FP32='1')
    r = subprocess.run([sys.executable, '-c', _GUARD_FP32_SCRIPT, ROOT], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    print('P2S_GUARD_FP32=1, guard band 1e9:', out)
    assert out['n'] == out['B'] == 32
    assert out['fixture'] <= 2e-3
    # the recompute is the fp32 engine's arithmetic on the flagged queries
    assert out['vs_fp32'] <= 1e-5 and out['feat_vs_fp32'] <= 1e-5 * out['feat_scale']


# ------------------------------------------------------------------ b. per-element bound
def _oracle(Pm, args, model, R, chunk=16):
    parts = [sorc.network(Pm, *[a[b:b + chunk] for a in args], model, R=R[b:b + chunk])
             for b in range(0, args[0].shape[0], chunk)]
    out = {k: nb.V(torch.cat([p[k].v for p in parts]), torch.cat([p[k].e for p in parts])) for k in ('feat_max', 'logits')}
    out['R'] = (torch.cat([p['R'][0] for p in parts]), torch.cat([p['R'][1] for p in parts]))
    return out


def check_bound(tag, sd, inp, P=300, S=1000):
    Pm = nb.to_device(sorc.fold_params(sd), DEV)
    args = [cu(inp[k]) for k in KEYS]
    bad = []
    for name, kw in ENGINES.items():
        eng = engine(sd, P, S, **kw)
        logits = eng.forward(*args)
        _, aux = eng.forward_with_aux(*args)
        eng.close()
        R = aux['trans']
        ref = _oracle(Pm, args, name, R)
        ratios = {'feat_max': nb.worst(nb.excess(aux['feat_max'], ref['feat_max'])),
                  'logits': nb.worst(nb.excess(logits, ref['logits']))}
        R64, eR = ref['R']
        err = (R.double() - R64).abs()
        ratios['R'] = nb.worst(torch.where(err == 0, torch.zeros_like(err), err / eR))
        print('%s %s: %s' % (tag, name, ', '.join('%s %.3g at %s' % (k, r, at) for k, (r, at) in ratios.items())))
        bad += [(name, k, r, at) for k, (r, at) in ratios.items() if not r <= 1.0]
    assert not bad, bad


def test_fixture_inputs_within_the_bound():
    sd, inp, _ = shared_encoder_case()
    check_bound('fixture', sd, inp)


@pytest.mark.parametrize('P,S', [(8, 64), (63, 65), (300, 1000), (1200, 1000)])
def test_patch_and_subsample_sizes_within_the_bound(P, S):
    sd = synth.make_state_dict(VARIANT, seed=P + 5)
    check_bound('P %d S %d' % (P, S), sd, synth.make_model_inputs(16, P, S, seed=P * 7 + S + 1), P, S)


# ------------------------------------------------------------------ c. batch position, batch size, slabs
@pytest.mark.parametrize('name', ['tc', 'tc_precise'])
def test_logits_do_not_depend_on_batch_position(name):
    N = 16385
    sd = synth.make_state_dict(VARIANT, MODEL_SEED, fitted=True)
    inp = synth.make_model_inputs(N, seed=14)
    args = [cu(inp[k]) for k in KEYS]
    eng = engine(sd, **ENGINES[name])
    full = eng.forward(*args)
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    streams = [sm // 2, sm // 8]
    sizes = sorted({1, 2, 8191, 8192, 8193} | {s + d for s in streams for d in (-1, 0, 1)})
    rng = np.random.RandomState(4)
    for B in sizes:
        for off in sorted({0, 1, N - B, int(rng.randint(0, N - B + 1))}):
            out = eng.forward(*[a[off:off + B] for a in args])
            same = (out == full[off:off + B]).all(1)
            assert bool(same.all()), (B, off, int(torch.nonzero(~same)[0]))
    perm = torch.from_numpy(rng.permutation(N)).to(DEV)
    out = eng.forward(*[a[perm] for a in args])
    same = (out == full[perm]).all(1)
    assert bool(same.all()), ('permutation', int(torch.nonzero(~same)[0]))
    eng.close()


def test_slab_and_batch_invariance():
    cloud = synth.make_cloud('sphere', 10000, seed=0)
    sd = synth.make_state_dict(VARIANT, MODEL_SEED, fitted=True)
    eng = engine(sd, precision='tc', guard_band=0.05)
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


# ------------------------------------------------------------------ d. fused reconstruction, end to end
@pytest.fixture(scope='module')
def sphere_case():
    """res 64 on the fitted checkpoint: the fused call (tc, default guard band) and the reference path over every query
    on the GPU's own patches and sub-sample ids (fp32 CPU oracle network + post-process)."""
    res, eps = 64, 3
    cloud = synth.make_cloud('sphere', 10000, seed=0)
    sd = synth.make_state_dict(VARIANT, MODEL_SEED, fitted=True)
    eng = engine(sd, precision='tc', guard_band=0.05)
    pts = cu(cloud)
    lin, sdf = eng.reconstruct(pts, res, eps, 0, SEED)
    n_guard = eng.last_guard_count()
    eng.close()
    qd = ops.query_points(lin, res)
    qpts = qd.cpu().numpy()
    assert np.array_equal(qpts, orc.query_grid(cloud, res, eps))
    Q = len(qpts)
    logits = np.empty((Q, 2), np.float32)
    radius = np.empty((Q,), np.float32)
    for b in range(0, Q, 512):
        q = qd[b:b + 512]
        _, patch, r = ops.knn_patch(pts, q, 300)
        sub = ops.gather_points(pts, ops.subsample(pts, q, 1000, False, SEED, query_index_base=b))
        logits[b:b + 512] = sorc.model_forward(sd, patch.cpu().numpy(), sub.cpu().numpy(), qpts[b:b + 512])
        radius[b:b + 512] = r.cpu().numpy()
    return dict(res=res, lin=lin, sdf=sdf, qpts=qpts, logits=logits, sdf_o=orc.post_process(logits, radius),
                n_guard=n_guard)


def test_fused_reconstruction_against_reference_path(sphere_case):
    c = sphere_case
    voxel = 2.0 / c['res']
    got = c['sdf'].cpu().numpy()
    decided = np.abs(c['logits'][:, 1]) > FP32_AMBIGUOUS
    mism = int(((got > 0) != (c['sdf_o'] > 0))[decided].sum())
    # the magnitude and the sign come from two logits: |d| on every query, the sign where the fp32 sign is decided
    # (an fp32-ambiguous sign may flip, which moves the SDF by 2 |d|)
    dv = np.abs(np.abs(got) - np.abs(c['sdf_o'])) / voxel
    print('shared encoder res %d: Q %d, guard recompute %d, fp32-ambiguous %d, positive fraction %.3f, sign mismatches %d, '
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
    print('shared encoder mesh: engine %d faces, oracle %d faces; Chamfer per sample %.5f = %.3f voxel, sampling floor '
          '%.3f voxel' % (len(faces), len(fo), cd, cd / voxel, floor / voxel))
    assert cd <= floor + 0.05 * voxel, (cd, floor)


# ------------------------------------------------------------------ e. eval entry point
def _dataset(tmp_path):
    root = tmp_path / 'data'
    (root / '04_pts').mkdir(parents=True)
    clouds = {'sphere': synth.make_cloud('sphere', 6000, seed=2), 'torus': synth.make_cloud('torus', 5000, seed=3)}
    for name, cloud in clouds.items():
        np.save(root / '04_pts' / (name + '.xyz.npy'), cloud)
    (root / 'testset.txt').write_text('sphere\ntorus\n')
    models = tmp_path / 'models'
    models.mkdir()
    sd = synth.make_state_dict(VARIANT, MODEL_SEED, fitted=True)
    torch.save({'module.' + k: v for k, v in sd.items()}, models / 'p2s_shared_encoder_model_49.pth')
    torch.save(synth.make_train_opt(VARIANT), models / 'p2s_shared_encoder_params.pth')
    return root, models, sd, clouds


def _script_args(root, out, models, res):
    # experiments/eval_p2s_shared_encoder.sh, at a small grid resolution
    return ['--indir', str(root), '--outdir', str(out), '--modeldir', str(models), '--dataset', 'testset.txt',
            '--models', 'p2s_shared_encoder', '--modelpostfix', '_model_49.pth', '--batchSize', '501', '--workers', '7',
            '--cache_capacity', '5', '--query_grid_resolution', str(res), '--epsilon', '3', '--certainty_threshold', '13',
            '--sigma', '5']


def _check_rec(rec, eng, clouds, res):
    from points2surf_b200 import mesh_io
    for name, cloud in clouds.items():
        q = np.load(rec / 'query_pts_ms' / (name + '.xyz.npy'))
        d = np.load(rec / 'dist_ms' / (name + '.xyz.npy'))
        lin, sdf = eng.reconstruct(cu(cloud), res, 3, 0, SEED, batch=501)
        assert np.array_equal(q, ops.query_points(lin, res).cpu().numpy())
        assert d.dtype == np.float32 and np.array_equal(d, sdf.cpu().numpy())
        assert (d > 0).any() and (d < 0).any()
        assert np.array_equal(np.load(rec / 'eval' / (name + '.xyz.npy')), d)
        assert np.loadtxt(rec / 'eval' / (name + '.xyz.txt')).shape == d.shape
        for sub in ('vis', 'query_pts_ms_vis'):
            v, f = mesh_io.read_ply(str(rec / sub / (name + '.ply')))
            assert v.shape == q.shape and len(f) == 0


def test_points_to_surf_eval_shared_encoder_script(tmp_path):
    root, models, sd, clouds = _dataset(tmp_path)
    out = tmp_path / 'results'
    res = 32
    opt = p2s_eval.parse_arguments(_script_args(root, out, models, res))
    opt.reconstruction = True
    p2s_eval.points_to_surf_eval(opt)
    eng = engine(sd, precision='tc', guard_band=0.05)
    _check_rec(out / 'rec', eng, clouds, res)

    # --reconstruction 0 on 05_query_pts: the rotation-augmented pass, equal to the engine on the same rotated inputs
    (root / '05_query_pts').mkdir()
    rng = np.random.RandomState(4)
    qs = {}
    for name in clouds:
        qs[name] = rng.uniform(-0.7, 0.7, (300, 3)).astype(np.float32)
        np.save(root / '05_query_pts' / (name + '.ply.npy'), qs[name])
    opt = p2s_eval.parse_arguments(_script_args(root, out, models, res))
    p2s_eval.points_to_surf_eval(opt)
    train_opt = synth.make_train_opt(VARIANT)
    for name, cloud in clouds.items():
        d = np.load(out / 'eval' / 'eval' / (name + '.xyz.npy'))
        want = p2s_eval._eval_given_queries(eng, train_opt, opt, cu(cloud), qs[name], torch.device(DEV))
        assert d.shape == (300,) and np.isfinite(d).all() and np.array_equal(d, want.cpu().numpy())
    eng.close()

    # --sampling sequential_shapes_random_patches
    opt = p2s_eval.parse_arguments(_script_args(root, tmp_path / 'results_seq', models, res) +
                                   ['--sampling', 'sequential_shapes_random_patches', '--patches_per_shape', '40'])
    p2s_eval.points_to_surf_eval(opt)
    for name in clouds:
        idx = np.loadtxt(tmp_path / 'results_seq' / 'eval' / (name + '.idx'), dtype=np.int64)
        assert np.load(tmp_path / 'results_seq' / 'eval' / 'eval' / (name + '.xyz.npy')).shape == idx.shape == (40,)


def test_points_to_surf_eval_through_the_source_package(tmp_path):
    root, models, sd, clouds = _dataset(tmp_path)
    sys.modules.pop('source', None)
    from source import points_to_surf_eval as src_eval
    out = tmp_path / 'results'
    opt = src_eval.parse_arguments(_script_args(root, out, models, 32))
    opt.reconstruction = True
    src_eval.points_to_surf_eval(opt)
    eng = engine(sd, precision='tc', guard_band=0.05)
    _check_rec(out / 'rec', eng, clouds, 32)
    eng.close()


def test_ball_patches_and_the_fixed_uniform_subsample(tmp_path):
    """Options orthogonal to the encoder: fixed-radius ball patches and the one fixed uniform sub-sample per shape run
    through the same engine and match it."""
    root, models, sd, clouds = _dataset(tmp_path)
    opt = synth.make_train_opt(VARIANT)
    opt.patch_radius, opt.uniform_subsample, opt.fixed_subsample = 0.1, 1, 1
    torch.save(opt, models / 'p2s_shared_encoder_params.pth')
    out = tmp_path / 'results'
    eval_opt = p2s_eval.parse_arguments(_script_args(root, out, models, 32))
    eval_opt.reconstruction = True
    p2s_eval.points_to_surf_eval(eval_opt)
    eng = engine(sd, precision='tc', guard_band=0.05)
    for name, cloud in clouds.items():
        lin, sdf = p2s_eval._reconstruct_fixed_subsample(eng, opt, eval_opt, cu(cloud))
        d = np.load(out / 'rec' / 'dist_ms' / (name + '.xyz.npy'))
        assert np.array_equal(d, sdf.cpu().numpy()) and np.isfinite(d).all() and np.abs(d).max() <= 1.0
    eng.close()
