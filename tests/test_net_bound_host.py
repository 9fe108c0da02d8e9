"""CPU checks of the network error bound (oracle/net_bound.py) before any GPU run.

* Sound: float32 CPU emulations of the three arithmetics (fp16-rounded operands, hi | lo splits, plain fp32) stay inside
  the bound, on the golden inputs of the three variants and on random inputs at ragged patch / sub-sample sizes.
* Has teeth: emulations with one fault each (a dropped MMA of the split path, a dropped or zero-padded point, a skipped
  k-step of the big layer) break it.
* Not vacuous: the width of the check relative to |value| on the max features is small, and stated per model."""
import numpy as np
import pytest
import torch

from oracle import net_bound as nb
from oracle import p2s_oracle as orc
from points2surf_b200 import synth
from helpers import golden_model_case, calibrated_state_dict

# (P, S) with tile tails on both sides of the 64-point tile, each with one of the variants
SHAPES = [(8, 64, 'vanilla'), (63, 65, 'max'), (64, 128, 'uniform'), (65, 127, 'vanilla'), (300, 1000, 'max'),
          (1200, 1000, 'uniform')]


def f16(x):
    return x.half().float()


def split(x):
    hi = x.half().float()
    return hi, (x - hi).half().float()


def emu_linear(x, W, b, op, drop_hi_lo=False):
    """float32 x W^T (+ b) with the operands rounded like the engine; drop_hi_lo omits the a_hi * w_lo MMA."""
    Wt = W.transpose(-1, -2)
    if op == 'fp32':
        y = x @ Wt
    elif op == 'fp16':
        y = f16(x) @ f16(Wt)
    else:
        (xh, xl), (wh, wl) = split(x), split(Wt)
        y = xl @ wh + xh @ wh if drop_hi_lo else xl @ wh + xh @ wl + xh @ wh
    return y if b is None else y + b


def emulate(P32, variant, patch, sub, query, model, mutation=None):
    """The engine's arithmetic in float32 on the CPU.  mutation: None, 'drop_hi_lo' (the a_hi * w_lo MMA of the final
    local stack's big layer), 'drop_last' (the last patch point in every pass), 'zero_pad' (segments padded to the 64-point
    tile with zero coordinates instead of a duplicate point), 'skip_kstep' (k 16..31 of channels 0..63 of the final local
    stack's big layer)."""
    m = nb.MODELS[model]
    conv, fc = m['conv'][0], m['fc'][0]
    v = synth.VARIANTS[variant]

    def points(raw, center, is_patch):
        if mutation == 'drop_last' and is_patch:
            raw = raw[:, :-1]
        if mutation == 'zero_pad' and raw.shape[1] % 64:
            raw = torch.cat([raw, raw.new_zeros(raw.shape[0], 64 - raw.shape[1] % 64, 3)], 1)
        return raw - center[:, None, :] if center is not None else raw

    def first(xc, R, name):
        W0, b0 = P32[name]
        if R is None:
            return (xc @ W0.t() + b0).relu()
        if model == 'fp32':
            return ((xc @ R.transpose(1, 2)) @ W0.t() + b0).relu()
        wq = torch.einsum('oi,bij->boj', W0, R)              # (W0 R) per query, net_tc.cu:185-187
        return (xc @ wq.transpose(1, 2) + b0).relu()

    def big_max(x, name, mut=False):
        W, b = P32[name]
        if mut and mutation == 'skip_kstep':
            W = W.clone()
            W[0:64, 16:32] = 0.0
        return emu_linear(x, W, None, conv, mut and mutation == 'drop_hi_lo').amax(1) + b

    def fc_tail(p, g):
        f1 = emu_linear(g, *P32[p + 'fc1'], fc).relu()
        return emu_linear(f1, *P32[p + 'fc2'], fc).relu()

    def qstn(p, xc):
        x = first(xc, None, p + 'conv1')
        x = emu_linear(x, *P32[p + 'conv2'], conv).relu()
        g = big_max(x, p + 'conv3').relu()
        return emu_linear(fc_tail(p, g), *P32[p + 'fc3'], 'fp32')

    def feat(p, xc, R, final_mut):
        x = first(xc, R, p + 'conv0a')
        x = emu_linear(x, *P32[p + 'conv0b'], conv).relu()
        s = p + 'stn2.'
        h = emu_linear(x, *P32[s + 'conv1'], conv).relu()
        h = emu_linear(h, *P32[s + 'conv2'], conv).relu()
        f2 = fc_tail(s, big_max(h, s + 'conv3').relu())
        W1, b1 = P32[p + 'conv1']
        Wf, bf = P32[s + 'fc3']
        B = x.shape[0]
        if model == 'fp32':
            T = (f2 @ Wf.t() + bf) + torch.eye(64).reshape(-1)
            y = emu_linear(emu_linear(x, T.view(B, 64, 64), None, 'fp32'), W1, b1, 'fp32').relu()
        else:
            G = torch.einsum('oj,jik->oik', W1, Wf.view(64, 64, 256)).reshape(4096, 256)
            g0 = (W1 + W1 @ bf.view(64, 64)).reshape(-1)
            M = emu_linear(f2, G, g0, fc)
            y = emu_linear(x, M.view(B, 64, 64), b1, conv).relu()
        y = emu_linear(y, *P32[p + 'conv2'], conv).relu()
        return big_max(y, p + 'conv3', final_mut)

    R = None
    if v['use_point_stn']:
        if v['shared_transformer']:
            q4 = qstn('point_stn.', torch.cat([points(patch, None, True), points(sub, query, False)], 1))
        else:
            q4 = qstn('feat_global.stn1.', points(sub, query, False))
        q = q4 + torch.tensor([1.0, 0.0, 0.0, 0.0])
        R = nb.quat_to_rot(q.double()).float()
    fg = feat('feat_global.', points(sub, query, False), R, False)
    fl = feat('feat_local.', points(patch, None, True), R, True)
    h = torch.cat([emu_linear(fl, *P32['fc1_local'], fc).relu(), emu_linear(fg, *P32['fc1_global'], fc).relu()], -1)
    h = emu_linear(h, *P32['fc2'], fc).relu()
    h = emu_linear(h, *P32['fc3'], fc).relu()
    logits = emu_linear(h, *P32['fc4'], 'fp32')
    return dict(R=R, feat_global_max=fg, feat_local_max=fl, logits=logits)


def _case(name):
    if name in synth.VARIANTS:
        sd, inp, _ = golden_model_case(name)
        return name, sd, inp
    P, S, variant = SHAPES[int(name)]
    inp = synth.make_model_inputs(3, points_per_patch=P, sub_sample_size=S, seed=P + S)
    return variant, synth.make_state_dict(variant, seed=P), inp


def _run(variant, sd, inp, model, mutation=None):
    """-> dict key -> (max error-to-bound ratio, worst index), plus the oracle's outputs."""
    P = nb.fold_params(sd, variant)
    P32 = {k: (W.float(), b.float()) for k, (W, b) in P.items()}
    args = [torch.from_numpy(inp[k]) for k in ('patch_pts_ps', 'pts_sub_sample_ms', 'imp_surf_query_point_ms')]
    emu = emulate(P32, variant, *args, model, mutation)
    ref = nb.network(P, variant, *args, model, R=emu['R'])
    res = {k: nb.worst(nb.excess(emu[k], ref[k])) for k in ('feat_global_max', 'feat_local_max', 'logits')}
    if ref['R'] is not None:
        R64, eR = ref['R']
        err = (emu['R'].double() - R64).abs()
        res['R'] = nb.worst(torch.where(err == 0, torch.zeros_like(err), err / eR))
    return res, ref


CASES = ['vanilla', 'max', 'uniform'] + [str(i) for i in range(len(SHAPES))]


@pytest.mark.parametrize('model', ['fp32', 'tc', 'tc_precise'])
@pytest.mark.parametrize('case', CASES)
def test_emulation_stays_inside_the_bound(case, model):
    variant, sd, inp = _case(case)
    res, _ = _run(variant, sd, inp, model)
    print(case, model, res)
    for k, (r, at) in res.items():
        assert r <= 1.0, (k, r, at)


def test_float64_values_match_the_reference_network():
    # the bound's float64 values are the reference network's (torch fp32 on the unfolded BatchNorm, fp32 round-off apart)
    for variant in ('vanilla', 'max', 'uniform'):
        sd, inp, g = golden_model_case(variant)
        v = synth.VARIANTS[variant]
        P = nb.fold_params(sd, variant)
        args = [torch.from_numpy(inp[k]) for k in ('patch_pts_ps', 'pts_sub_sample_ms', 'imp_surf_query_point_ms')]
        out = nb.network(P, variant, *args, 'fp32')
        _, raux = orc.model_forward(sd, *[inp[k] for k in ('patch_pts_ps', 'pts_sub_sample_ms', 'imp_surf_query_point_ms')],
                                    v['use_point_stn'], v['shared_transformer'], return_aux=True)
        assert np.abs(out['logits'].v.numpy() - g['logits']).max() < 1e-3
        for k in ('feat_global_max', 'feat_local_max'):
            assert np.abs(out[k].v.numpy() - raux[k]).max() < 1e-4 * np.abs(raux[k]).max()
        if 'trans' in raux:
            assert np.abs(out['R'][0].numpy() - raux['trans']).max() < 1e-5


# each fault must push some element past its bound; the key that shows it is named
# A zero-coordinate pad point moves the fp16 path's features by less than its bound (about 0.3 of it on this batch): on
# that path the padding is pinned by the bit-equality tests of tests/test_gpu_net_kernels.py instead.
MUTATIONS = [(mut, model, 'feat_local_max') for mut in ('drop_last', 'zero_pad', 'skip_kstep') for model in ('fp32', 'tc', 'tc_precise')
             if (mut, model) != ('zero_pad', 'tc')] + [('drop_hi_lo', 'tc_precise', 'feat_local_max')]


@pytest.mark.parametrize('mutation,model,key', MUTATIONS)
def test_mutated_emulation_breaks_the_bound(mutation, model, key):
    sd = calibrated_state_dict('vanilla', 21)
    inp = synth.make_model_inputs(4, seed=5)
    res, _ = _run('vanilla', sd, inp, model, mutation)
    print(mutation, model, res)
    assert res[key][0] > 1.0, res


# width of the check (LAMBDA e) / |value| on the max features with |value| >= 1 (the features are O(1) to O(10)): median and
# 99th percentile per model on the golden inputs, asserted with a margin of about 1.5 over the measured values (printed)
RELATIVE = {'fp32': (2e-4, 1.5e-3), 'tc': (0.13, 1.0), 'tc_precise': (5e-4, 4e-3)}


@pytest.mark.parametrize('model', ['fp32', 'tc', 'tc_precise'])
def test_bound_is_not_vacuous(model):
    rel = []
    for variant in ('vanilla', 'max', 'uniform'):
        sd, inp, _ = golden_model_case(variant)
        _, ref = _run(variant, sd, inp, model)
        for k in ('feat_global_max', 'feat_local_max'):
            v, e = ref[k].v.abs().reshape(-1), ref[k].e.reshape(-1)
            rel.append((nb.LAMBDA * e / v)[v >= 1.0])
    rel = torch.cat(rel)
    med, p99 = float(rel.median()), float(torch.quantile(rel, 0.99))
    print(model, 'check width / |feature|: median %.3g, 99th percentile %.3g' % (med, p99))
    assert med < RELATIVE[model][0] and p99 < RELATIVE[model][1], (med, p99)
