"""CPU: the shared-encoder ablation (single_transformer=1, experiments/eval_p2s_shared_encoder.sh) -- the oracle
(tests/shared_encoder_oracle.py) against the fixture the unmodified reference produced
(tests/golden/make_shared_encoder_golden.py), the synthetic checkpoint's key order, the blob layout and its size in the
library, the library's rejection of unsupported configurations, the evaluation option matrix and the fitted head."""
import ctypes as C
import json
from argparse import Namespace

import numpy as np
import pytest
import torch

from points2surf_b200 import _lib, arch, synth, weights
from points2surf_b200 import eval as p2s_eval
from helpers import load_golden
import shared_encoder_oracle as sorc

VARIANT = 'shared_encoder'
V = synth.VARIANTS[VARIANT]


def shared_encoder_case():
    """-> (state dict with the fixture's fc4 bias, inputs, fixture)."""
    g = load_golden('shared_encoder.npz')
    sd = synth.make_state_dict(VARIANT, int(g['model_seed']), fitted=True)
    sd['fc4.bias'] = torch.from_numpy(g['fc4_bias'].copy())
    inp = synth.make_model_inputs(int(g['batch']), seed=int(g['input_seed']))
    chk = sum(float(np.abs(a).sum()) for a in inp.values())
    assert abs(chk - float(g['input_checksum'])) < 1e-6 * chk, 'synthetic input generator drifted'
    return sd, inp, g


def test_oracle_matches_reference_fixture():
    sd, inp, g = shared_encoder_case()
    lo, aux = sorc.model_forward(sd, inp['patch_pts_ps'], inp['pts_sub_sample_ms'], inp['imp_surf_query_point_ms'],
                                 return_aux=True)
    assert lo.shape == g['logits'].shape == (int(g['batch']), 2)
    assert np.abs(lo - g['logits']).max() <= 1e-5
    assert np.abs(aux['trans'] - g['trans']).max() <= 1e-6
    assert np.abs(aux['feat_max'] - g['feat_max']).max() <= 1e-5
    for col in range(2):
        assert (g['logits'][:, col] > 0).any() and (g['logits'][:, col] < 0).any(), 'the fixture must have both signs'


def test_state_dict_key_order_matches_reference():
    g = load_golden('shared_encoder.npz')
    keys = [str(k) for k in g['state_dict_keys']]
    assert list(synth.make_state_dict_numpy(VARIANT, 0).keys()) == keys
    assert keys[0].startswith('feat_local_global.stn1.') and 'fc1_local_global.weight' in keys
    assert not any(k.startswith(('feat_local.', 'feat_global.', 'point_stn.', 'fc1_local.', 'fc1_global.')) for k in keys)
    names = [s[0] for s in arch.layer_specs(1, 0, single_transformer=True)]
    assert names[names.index('fc1_local_global'):] == ['fc1_local_global', 'bn1_local_global', 'fc2', 'fc3', 'fc4', 'bn2', 'bn3']
    # shared_transformation plays no part in the shared encoder (points_to_surf_model.py:253-263)
    assert arch.layer_specs(1, 1, single_transformer=True) == arch.layer_specs(1, 0, single_transformer=True)
    # the other variants are unchanged
    for variant in ('vanilla', 'max', 'uniform', 'regression'):
        assert synth.make_train_opt(variant).single_transformer == 0
    assert synth.make_train_opt(VARIANT).single_transformer == 1


def _cfg():
    return _lib.ModelConfig(V['use_point_stn'], V['shared_transformer'], 300, 1000, 1024)


def _layer_floats(sd, name):
    return int(np.prod(sd[name + '.weight'].shape)) + int(sd[name + '.bias'].shape[0])


def test_blob_size_and_layout():
    lib = _lib.load()
    sd = synth.make_state_dict_numpy(VARIANT, 0, module_prefix='module.')
    blob = weights.pack_blob(sd, V['use_point_stn'], V['shared_transformer'], single_transformer=True)
    cfg = _cfg()
    assert blob.size == lib.p2s_model_blob_floats_enc(C.byref(cfg), 2, 1)
    assert blob.dtype == np.float32 and np.isfinite(blob).all()
    # FEAT(feat_local_global, 1) fc1_local_global fc2 fc3 fc4: the tail is the head, fc4 last
    bare = weights.strip_module_prefix(sd)
    head = ['fc1_local_global', 'fc2', 'fc3', 'fc4']
    tail = sum(_layer_floats(bare, n) for n in head)
    w4, b4 = weights.fold(bare, 'fc4')
    assert np.array_equal(blob[-b4.size:], b4) and np.array_equal(blob[-b4.size - w4.size:-b4.size], w4)
    w1, b1 = weights.fold(bare, 'fc1_local_global', 'bn1_local_global')
    assert np.array_equal(blob[-tail:-tail + w1.size], w1)
    # the _ex sizes are unchanged and equal the _enc sizes with single_transformer 0
    for variant in ('vanilla', 'max', 'uniform', 'regression'):
        v = synth.VARIANTS[variant]
        c = _lib.ModelConfig(v['use_point_stn'], v['shared_transformer'], 300, 1000, 1024)
        od = v.get('output_dim', 2)
        b = weights.pack_blob(synth.make_state_dict_numpy(variant, 0), v['use_point_stn'], v['shared_transformer'], od)
        assert b.size == lib.p2s_model_blob_floats_ex(C.byref(c), od) == lib.p2s_model_blob_floats_enc(C.byref(c), od, 0)
    # the regression head on the shared encoder is a one-row-shorter fc4 (the library sizes it; eval rejects it)
    assert lib.p2s_model_blob_floats_enc(C.byref(cfg), 2, 1) - lib.p2s_model_blob_floats_enc(C.byref(cfg), 1, 1) == 129


def test_unsupported_configurations_are_rejected():
    lib = _lib.load()
    sd = synth.make_state_dict_numpy(VARIANT, 0)
    blob = weights.pack_blob(sd, 1, 0, single_transformer=True)
    bad = [(_lib.ModelConfig(0, 0, 300, 1000, 1024), 1, 'use_point_stn=1'),
           (_lib.ModelConfig(1, 1, 300, 1000, 1024), 1, 'shared_transformer=0'),
           (_cfg(), 2, 'single_transformer must be 0 or 1'),
           (_cfg(), -1, 'single_transformer must be 0 or 1')]
    for cfg, st, msg in bad:
        assert lib.p2s_model_blob_floats_enc(C.byref(cfg), 2, st) == 0
        h = C.c_void_p()
        # the configuration is checked before any device work: the same message with or without a GPU
        rc = lib.p2s_model_create_enc(C.byref(cfg), 2, st, blob.ctypes.data_as(C.c_void_p), blob.size, 0, C.byref(h))
        assert rc != 0 and not h.value
        assert msg in lib.p2s_last_error().decode()
    for bad_od in (0, 3):
        assert lib.p2s_model_blob_floats_enc(C.byref(_cfg()), bad_od, 1) == 0
    # a blob of the two-branch layout does not fit the shared encoder
    h = C.c_void_p()
    vb = weights.pack_blob(synth.make_state_dict_numpy('uniform', 0), 1, 0)
    assert lib.p2s_model_create_enc(C.byref(_cfg()), 2, 1, vb.ctypes.data_as(C.c_void_p), vb.size, 0, C.byref(h)) != 0
    assert 'blob size' in lib.p2s_last_error().decode()
    for upst, shared in ((0, 0), (1, 1)):
        with pytest.raises(ValueError):
            weights.pack_blob(sd, upst, shared, single_transformer=True)


def test_fitted_shared_encoder_head():
    w, b = synth.fitted_fc4(VARIANT, 12)
    assert w.shape == (2, 128) and b.shape == (2,) and np.isfinite(w).all()
    with open(synth.FITTED_FC4_SHARED_ENCODER) as fp:
        assert json.load(fp)['heldout_sign_accuracy'] > 0.8
    with pytest.raises(ValueError):
        synth.fitted_fc4(VARIANT, 13)
    sd = synth.make_state_dict(VARIANT, 12, fitted=True)
    assert torch.equal(sd['fc4.weight'], torch.from_numpy(w))


def test_eval_accepts_the_published_shared_encoder_only():
    ok = synth.make_train_opt(VARIANT)
    assert ok.single_transformer == 1 and ok.use_point_stn == 1 and ok.shared_transformer == 0
    assert ok.outputs == ['imp_surf_magnitude', 'imp_surf_sign', 'patch_pts_ids', 'p_index']
    p2s_eval._check_supported(ok, p2s_eval.parse_arguments([]))
    p2s_eval._check_supported(ok, p2s_eval.parse_arguments(['--sampling', 'sequential_shapes_random_patches']))
    # shared_transformer is ignored by the shared encoder (as in the reference)
    p2s_eval._check_supported(Namespace(**{**vars(ok), 'shared_transformer': 1}), p2s_eval.parse_arguments([]))
    no_stn = Namespace(**vars(ok))
    del no_stn.use_point_stn
    bad = [
        Namespace(**{**vars(ok), 'outputs': ['imp_surf', 'patch_pts_ids', 'p_index']}),      # the regression head
        Namespace(**{**vars(ok), 'use_point_stn': 0}),
        no_stn,                                                                             # no use_point_stn field
        Namespace(**{**vars(ok), 'sym_op': 'sum'}),
        Namespace(outputs=ok.outputs, patch_radius=0.0, sym_op='max', single_transformer=1),
    ]
    for train_opt in bad:
        with pytest.raises(ValueError):
            p2s_eval._check_supported(train_opt, p2s_eval.parse_arguments([]))
    with pytest.raises(ValueError):
        p2s_eval._check_supported(ok, p2s_eval.parse_arguments(['--sampling', 'sequential_shapes_random_patches',
                                                                '--reconstruction', '1']))


def test_training_and_the_module_still_reject_the_shared_encoder():
    from points2surf_b200.model import PointsToSurfModel
    with pytest.raises(ValueError):
        PointsToSurfModel(single_transformer=True, output_dim=2)
