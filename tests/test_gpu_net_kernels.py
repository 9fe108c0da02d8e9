"""The inference network's kernels per element, per point slot and per batch position.

a. Every max feature, rotation and logit of the three engines ('fp32', 'tc' without guard band, 'tc' with every query on
   the split-precision recompute path) lies within oracle/net_bound.py's bound of the float64 network, evaluated with
   the engine's own rotation.  Features and R come from `forward_with_aux`; logits from plain `forward`, the production
   path (`debug_aux` turns off the fused conv3 bias and routes the head through the fp32-row producers).
b. Every point slot is read exactly once: B = max(P, S) queries share one query point, and query j sees its patch rotated
   by j mod P and its sub-sample by j mod S.  Every point's column of every layer is computed without reference to the
   other points and the max is exact, and every query's row of every FC layer is computed without reference to the other
   rows, so all rows of logits and aux are bit-identical.  Every point visits every slot, so a slot that is dropped, read
   twice or read from another segment or query changes the rows in which an arg-max point lands there.
c. The padding of a segment's last tile is a duplicate point: P = 75 and P = 128 (the same patch plus 53 of its own
   points again) give bit-identical local features.
d. A query's logits do not depend on its position in the batch, on the batch size or on the chunking of forward_tc_core.
"""
import numpy as np
import pytest
import torch

from oracle import net_bound as nb
from points2surf_b200 import synth, ops
from helpers import golden_model_case, calibrated_state_dict

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
SHAPES = [(8, 64), (63, 65), (64, 128), (65, 127), (300, 1000), (1200, 1000)]
VARIANTS = ['vanilla', 'max', 'uniform']
ENGINES = {'fp32': dict(precision='fp32'), 'tc': dict(precision='tc', guard_band=0.0),
           'tc_precise': dict(precision='tc', guard_band=1e9)}
KEYS = ('patch_pts_ps', 'pts_sub_sample_ms', 'imp_surf_query_point_ms')


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def engine(sd, variant, name, P=300, S=1000):
    v = synth.VARIANTS[variant]
    return ops.Engine(sd, v['use_point_stn'], v['shared_transformer'], points_per_patch=P, sub_sample_size=S, **ENGINES[name])


def oracle(Pm, variant, args, model, R, chunk=32):
    """nb.network in chunks of queries (float64 on the GPU) -> dict key -> V."""
    parts = []
    for b in range(0, args[0].shape[0], chunk):
        parts.append(nb.network(Pm, variant, *[a[b:b + chunk] for a in args], model, R=None if R is None else R[b:b + chunk]))
    out = {}
    for k in ('feat_global_max', 'feat_local_max', 'logits'):
        out[k] = nb.V(torch.cat([p[k].v for p in parts]), torch.cat([p[k].e for p in parts]))
    if parts[0]['R'] is not None:
        out['R'] = (torch.cat([p['R'][0] for p in parts]), torch.cat([p['R'][1] for p in parts]))
    return out


def check_bound(tag, variant, sd, inp, P=300, S=1000):
    Pm = nb.to_device(nb.fold_params(sd, variant), DEV)
    args = [cu(inp[k]) for k in KEYS]
    bad = []
    for name in ENGINES:
        eng = engine(sd, variant, name, P, S)
        logits = eng.forward(*args)
        _, aux = eng.forward_with_aux(*args)
        R = aux['trans'] if synth.VARIANTS[variant]['use_point_stn'] else None
        ref = oracle(Pm, variant, args, name, R)
        ratios = {k: nb.worst(nb.excess(aux[k], ref[k])) for k in ('feat_global_max', 'feat_local_max')}
        ratios['logits'] = nb.worst(nb.excess(logits, ref['logits']))
        if 'R' in ref:
            R64, eR = ref['R']
            err = (R.double() - R64).abs()
            ratios['R'] = nb.worst(torch.where(err == 0, torch.zeros_like(err), err / eR))
        eng.close()
        # worst (query, channel) and its error-to-bound ratio per output
        print('%s %s: %s' % (tag, name, ', '.join('%s %.3g at %s' % (k, r, at) for k, (r, at) in ratios.items())))
        bad += [(name, k, r, at) for k, (r, at) in ratios.items() if not r <= 1.0]
    assert not bad, bad


@pytest.mark.parametrize('variant', VARIANTS)
def test_golden_inputs_within_the_bound(variant):
    sd, inp, _ = golden_model_case(variant)
    check_bound('golden ' + variant, variant, sd, inp)


def test_random_queries_within_the_bound():
    sd = calibrated_state_dict('vanilla', 21)
    check_bound('256 random', 'vanilla', sd, synth.make_model_inputs(256, seed=41))


@pytest.mark.parametrize('P,S', SHAPES)
def test_patch_and_subsample_sizes_within_the_bound(P, S):
    variant = VARIANTS[SHAPES.index((P, S)) % 3]
    sd = synth.make_state_dict(variant, seed=P + 3)
    check_bound('P %d S %d %s' % (P, S, variant), variant, sd, synth.make_model_inputs(16, P, S, seed=P * 7 + S), P, S)


def test_guard_band_diagnostics_land_in_each_querys_row():
    # with a guard band, `forward_with_aux` reports the recomputed features and rotation of every flagged query in that
    # query's own row: the recompute sees the flagged queries in list order, so its rows are scattered back like the logits
    sd = calibrated_state_dict('vanilla', 21)
    args = [cu(a) for a in (synth.make_model_inputs(300, seed=43)[k] for k in KEYS)]
    rows = lambda aux: torch.cat([aux['trans'].reshape(-1, 9), aux['feat_local_max'], aux['feat_global_max']], 1)
    fast = rows(engine(sd, 'vanilla', 'tc').forward_with_aux(*args)[1])
    precise = rows(engine(sd, 'vanilla', 'tc_precise').forward_with_aux(*args)[1])
    raw = engine(sd, 'vanilla', 'tc').forward(*args)
    band = float(raw[:, 1].abs().median())               # about half of the queries are recomputed
    eng = ops.Engine(sd, 1, 1, precision='tc', guard_band=band)
    got = rows(eng.forward_with_aux(*args)[1])
    flagged = raw[:, 1].abs() < band
    assert 0 < eng.last_guard_count() == int(flagged.sum()) < 300
    assert torch.equal(got[flagged], precise[flagged])
    assert torch.equal(got[~flagged], fast[~flagged])


def _rows_equal(tag, t):
    diff = (t != t[:1]).reshape(t.shape[0], -1)
    rows = torch.nonzero(diff.any(1)).reshape(-1)
    if rows.numel():
        r = int(rows[0])
        cols = torch.nonzero(diff[r]).reshape(-1)[:8].tolist()
        raise AssertionError('%s: %d rows differ from row 0; first row %d at columns %s' % (tag, rows.numel(), r, cols))


@pytest.mark.parametrize('P,S', SHAPES)
@pytest.mark.parametrize('variant', VARIANTS)
def test_every_slot_is_read_exactly_once(variant, P, S):
    inp = synth.make_model_inputs(1, P, S, seed=P * 11 + S)
    sd = synth.make_state_dict(variant, seed=13)
    B = max(P, S)
    j = np.arange(B)
    patch = inp['patch_pts_ps'][0][(np.arange(P)[None, :] + (j % P)[:, None]) % P]
    sub = inp['pts_sub_sample_ms'][0][(np.arange(S)[None, :] + (j % S)[:, None]) % S]
    args = [cu(patch), cu(sub), cu(np.repeat(inp['imp_surf_query_point_ms'], B, 0))]
    for name in ENGINES:
        eng = engine(sd, variant, name, P, S)
        # the fp32 engine runs calls of 64 to 1024 queries: each call is one chunk and every FC layer stays on the same GEMM kernel
        calls = [(0, B)] if name != 'fp32' or B <= 1024 else [(0, B // 2), (B // 2, B)]
        logits, aux = [], []
        for a, b in calls:
            part = [t[a:b] for t in args]
            logits.append(eng.forward(*part))
            _, x = eng.forward_with_aux(*part)
            aux.append(torch.cat([x['trans'].reshape(b - a, 9), x['feat_local_max'], x['feat_global_max']], 1))
        eng.close()
        _rows_equal('%s %s P %d S %d logits' % (name, variant, P, S), torch.cat(logits))
        _rows_equal('%s %s P %d S %d aux (R | local | global)' % (name, variant, P, S), torch.cat(aux))


@pytest.mark.parametrize('variant', VARIANTS)
def test_padding_is_a_duplicate_point(variant):
    sd = synth.make_state_dict(variant, seed=17)
    inp = synth.make_model_inputs(16, 75, 1000, seed=19)
    patch128 = np.concatenate([inp['patch_pts_ps'], inp['patch_pts_ps'][:, :53]], 1)
    sub, q = cu(inp['pts_sub_sample_ms']), cu(inp['imp_surf_query_point_ms'])
    for name in ENGINES:
        a = engine(sd, variant, name, 75, 1000).forward_with_aux(cu(inp['patch_pts_ps']), sub, q)[1]['feat_local_max']
        b = engine(sd, variant, name, 128, 1000).forward_with_aux(cu(patch128), sub, q)[1]['feat_local_max']
        assert torch.equal(a, b), (name, float((a - b).abs().max()))


@pytest.mark.parametrize('name', ['tc', 'tc_precise'])
def test_logits_do_not_depend_on_batch_position(name):
    N = 16385
    sd = calibrated_state_dict('vanilla', 21)
    inp = synth.make_model_inputs(N, seed=12)
    args = [cu(inp[k]) for k in KEYS]
    eng = engine(sd, 'vanilla', name)
    full = eng.forward(*args)
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    streams = [sm // 2, sm // 8]                     # query streams of the pass kernel: kSplit = 2, or 8 on the precise path
    sizes = sorted({1, 2, 8191, 8192, 8193} | {s + d for s in streams for d in (-1, 0, 1)})
    rng = np.random.RandomState(3)
    for B in sizes:
        for off in sorted({0, 1, N - B, (N - B) // 2, int(rng.randint(0, N - B + 1))}):
            out = eng.forward(*[a[off:off + B] for a in args])
            same = (out == full[off:off + B]).all(1)
            assert bool(same.all()), (B, off, int(torch.nonzero(~same)[0]))
    perm = torch.from_numpy(rng.permutation(N)).to(DEV)
    out = eng.forward(*[a[perm] for a in args])
    same = (out == full[perm]).all(1)
    assert bool(same.all()), ('permutation', int(torch.nonzero(~same)[0]))
    eng.close()
