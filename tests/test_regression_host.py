"""CPU: the regression ablation (outputs imp_surf patch_pts_ids p_index, experiments/eval_p2s_regression.sh) -- the oracle
(network: oracle/p2s_oracle.py, post-process: tests/regression_oracle.py) against the fixture the unmodified reference produced (tests/golden/make_regression_golden.py), the blob size of the
output_dim 1 head, the evaluation option matrix and the post-process on special values."""
import ctypes as C
import json
from argparse import Namespace

import numpy as np
import pytest
import torch

from oracle import p2s_oracle as orc
from points2surf_b200 import _lib, synth, weights
from points2surf_b200 import eval as p2s_eval
from helpers import load_golden
import regression_oracle as rorc

REGRESSION_OUTPUTS = ['imp_surf', 'patch_pts_ids', 'p_index']


def regression_case():
    """-> (state dict with the fixture's fc4 bias, inputs, fixture)."""
    g = load_golden('regression.npz')
    sd = synth.make_state_dict('regression', int(g['model_seed']), fitted=True)
    sd['fc4.bias'] = torch.from_numpy(g['fc4_bias'].copy())
    inp = synth.make_model_inputs(int(g['batch']), seed=int(g['input_seed']))
    chk = sum(float(np.abs(a).sum()) for a in inp.values())
    assert abs(chk - float(g['input_checksum'])) < 1e-6 * chk, 'synthetic input generator drifted'
    return sd, inp, g


def test_oracle_matches_reference_fixture():
    sd, inp, g = regression_case()
    v = synth.VARIANTS['regression']
    lo = orc.model_forward(sd, inp['patch_pts_ps'], inp['pts_sub_sample_ms'], inp['imp_surf_query_point_ms'],
                           v['use_point_stn'], v['shared_transformer'])
    assert lo.shape == g['logits'].shape == (int(g['batch']), 1)
    assert np.abs(lo - g['logits']).max() <= 1e-5
    assert (g['logits'] > 0).any() and (g['logits'] < 0).any(), 'the fixture must have both signs'
    assert np.array_equal(rorc.post_process_distance(g['logits'], g['radius']), g['sdf'])
    assert np.array_equal(rorc.post_process_distance(g['logits'], None), g['sdf_fixed_radius'])


def test_blob_size_of_the_regression_head():
    lib = _lib.load()
    v = synth.VARIANTS['regression']
    sd = synth.make_state_dict_numpy('regression', 0, module_prefix='module.')
    assert sd['module.fc4.weight'].shape == (1, 128)
    blob = weights.pack_blob(sd, v['use_point_stn'], v['shared_transformer'], output_dim=1)
    cfg = _lib.ModelConfig(v['use_point_stn'], v['shared_transformer'], 300, 1000, 1024)
    assert blob.size == lib.p2s_model_blob_floats_ex(C.byref(cfg), 1)
    assert lib.p2s_model_blob_floats_ex(C.byref(cfg), 2) == lib.p2s_model_blob_floats(C.byref(cfg))
    assert lib.p2s_model_blob_floats_ex(C.byref(cfg), 2) - blob.size == 129
    for bad in (0, 3, -1):
        assert lib.p2s_model_blob_floats_ex(C.byref(cfg), bad) == 0
    with pytest.raises(ValueError):
        weights.pack_blob(sd, v['use_point_stn'], v['shared_transformer'])          # fc4 has 1 output, not 2
    with pytest.raises(ValueError):
        weights.pack_blob(sd, v['use_point_stn'], v['shared_transformer'], output_dim=3)


def test_fitted_regression_head():
    w, b = synth.fitted_fc4('regression', 10)
    assert w.shape == (1, 128) and b.shape == (1,) and np.isfinite(w).all()
    with open(synth.FITTED_FC4_REGRESSION) as fp:
        assert json.load(fp)['heldout_sign_accuracy'] > 0.8
    with pytest.raises(ValueError):
        synth.fitted_fc4('regression', 11)


def test_eval_accepts_regression_outputs_and_keeps_the_other_rejections():
    ok = Namespace(**vars(synth.make_train_opt('regression')))
    assert ok.outputs == REGRESSION_OUTPUTS and p2s_eval._output_dim(ok) == 1
    p2s_eval._check_supported(ok, p2s_eval.parse_arguments([]))
    p2s_eval._check_supported(ok, p2s_eval.parse_arguments(['--sampling', 'sequential_shapes_random_patches']))
    p2s_eval._check_supported(Namespace(**{**vars(ok), 'outputs': ['patch_pts_ids', 'imp_surf', 'p_index']}),
                              p2s_eval.parse_arguments([]))
    assert p2s_eval._output_dim(synth.make_train_opt('vanilla')) == 2
    bad = [
        ['imp_surf'],                                                               # save_evaluation needs ids + p_index
        ['imp_surf', 'patch_pts_ids'],
        ['imp_surf', 'imp_surf_magnitude', 'imp_surf_sign', 'patch_pts_ids', 'p_index'],   # the reference default (3 outputs)
        ['imp_surf', 'imp_surf_sign', 'patch_pts_ids', 'p_index'],
        ['imp_surf', 'imp_surf', 'patch_pts_ids', 'p_index'],
    ]
    for outs in bad:
        with pytest.raises(ValueError):
            p2s_eval._check_supported(Namespace(**{**vars(ok), 'outputs': outs}), p2s_eval.parse_arguments([]))
    for key, value in (('single_transformer', 1), ('sym_op', 'sum')):
        with pytest.raises(ValueError):
            p2s_eval._check_supported(Namespace(**{**vars(ok), key: value}), p2s_eval.parse_arguments([]))


def test_model_module_accepts_the_regression_head_only():
    from points2surf_b200.model import PointsToSurfModel
    m = PointsToSurfModel(net_size_max=1024, num_points=300, output_dim=1, use_point_stn=True, shared_transformation=False,
                          sub_sample_size=1000)
    assert list(m.state_dict().keys()) == list(synth.make_state_dict('regression', 0).keys())
    assert tuple(m.fc4.weight.shape) == (1, 128)
    for kw in (dict(output_dim=3), dict(output_dim=0), dict(output_dim=1, single_transformer=True),
               dict(output_dim=1, sym_op='sum')):
        with pytest.raises(ValueError):
            PointsToSurfModel(**kw)


def _special_logits():
    tiny = np.finfo(np.float32).smallest_subnormal
    return np.array([0.0, -0.0, tiny, -tiny, 3 * tiny, -1e-40, 1e-3, -1e-3, 20.0, -20.0, np.inf, -np.inf, np.nan],
                    np.float32)


def numpy_distance(logits, radius):
    """NumPy restatement of sdf_nn.post_process_distance (+ the radius, + save_reconstruction_data's NaN rule)."""
    with np.errstate(invalid='ignore'):
        t = np.tanh(logits.astype(np.float64)).astype(np.float32)
        d = (t * t) * np.sign(logits)
        if radius is not None:
            d = d * radius
    d[np.isnan(d)] = np.float32(1.0)
    return d.astype(np.float32)


@pytest.mark.parametrize('fixed_radius', [False, True])
def test_post_process_restatement_on_special_values(fixed_radius):
    lg = _special_logits()
    r = None if fixed_radius else np.linspace(0.01, 0.4, lg.size).astype(np.float32)
    lt = torch.from_numpy(lg.copy()).unsqueeze(1)
    ref = torch.tanh(lt).pow(2) * torch.sign(lt)                                     # source/sdf_nn.py:6-8
    if r is not None:
        ref = ref * torch.from_numpy(r).unsqueeze(1)                                  # points_to_surf_eval.py:180-181
    ref = ref[:, 0].numpy().copy()
    ref[np.isnan(ref)] = 1.0                                                          # points_to_surf_eval.py:205-207
    got = numpy_distance(lg, r)
    assert np.array_equal(got, ref)
    assert np.array_equal(rorc.post_process_distance(lg, r), ref)
    assert got[0] == 0.0 and got[1] == 0.0 and got[-1] == 1.0
    unit = np.array([1, -1, 1, -1], np.float32)
    assert np.array_equal(got[8:12], unit if r is None else unit * r[8:12])      # tanh(+-20) and tanh(+-inf) are +-1
