"""GPU: the CTA-pair exchange of `pointnet_pass_kernel<false>` with many queries on every query stream.

The fp16 pass kernel runs each query stream on a cluster of two CTAs that split every query's tiles between them and
swap the big layer's A fragments through distributed shared memory; which CTA produces which tile changes with the
query's place in its stream (tests/pass_schedule.py models the schedule on the CPU).  Every (variant, P, S) below runs
B queries with B >= 8 x 66 and B around multiples of 66 and of 33, so that every stream of the `tc` engine runs at
least 8 queries, both warpgroups at least 4, whatever number of clusters fit on the device (B / 33 per stream at half
the clusters), and the split-precision recompute ('tc_precise', guard band 1e9: four CTAs per stream and no exchange)
runs B / 16 per stream on 132 SMs.  The shapes cover every variant, odd and even tile totals, one-tile segments, the
ABI's limits P = 8 / 1536 and S = 8 / 4096, and the production ablations P = 75 (small kNN) and P = 1200 (large kNN).

a. Batch position: every query's logits (`forward`) and `forward_with_aux` row (R, local and global max feature; the
   shared encoder's one max feature) are bit-identical in the full batch and in a permutation of it.  Every query's
   logits are also bit-identical alone in a batch of one (one stream, first query of warpgroup 0), and so are the aux
   rows of the sample below.  Each query's features are exact maxima over the same per-tile arithmetic whichever CTA
   produced a tile, so any difference is a schedule error; a failure names the first differing query, its stream and
   place in it, and the column.
b. Per element: the sample holds the first four and last two queries of stream 0 and of the last stream (both
   warpgroups, both halves of the `own` alternation) for the `tc` engine's stream count at all and at half of the
   clusters and for the recompute's; their rows of the full batch lie within oracle/net_bound.py's bound (LAMBDA times
   the error scale of the engine's arithmetic; tests/shared_encoder_oracle.py for the shared encoder).  With (a), that
   covers every query of the batch.
c. Two-segment launches (the vanilla network's QSTN over patch + centred sub-sample, every pass of the shared encoder):
   for an odd number of patch tiles the boundary between the segments falls inside a pair of tiles, and each CTA of a
   cluster, over the sampled queries, produces the last patch tile of that pair as well as receives it.
"""
import numpy as np
import pytest
import torch

from oracle import net_bound as nb
from points2surf_b200 import synth, ops
import pass_schedule as ps
import shared_encoder_oracle as sorc
from test_gpu_net_kernels import oracle as net_oracle
from test_gpu_shared_encoder import _oracle as shared_oracle

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
KEYS = ('patch_pts_ps', 'pts_sub_sample_ms', 'imp_surf_query_point_ms')
ENGINES = {'tc': 0.0, 'tc_precise': 1e9}          # guard band
# (variant, P, S): tiles per launch in the comment (two-segment launches as patch + sub-sample)
CASES = [
    ('vanilla', 8, 4096),        # QSTN 1 + 64 (boundary inside pair 0), local 1, global 64; P and S at their limits
    ('vanilla', 1536, 8),        # QSTN 24 + 1 (boundary between pairs, odd total), local 24, global 1
    ('vanilla', 129, 65),        # QSTN 3 + 2 (boundary inside pair 1), local 3, global 2
    ('vanilla', 75, 1000),       # small kNN: QSTN 2 + 16, local 2
    ('vanilla', 1200, 1000),     # large kNN: QSTN 19 + 16 (boundary inside pair 9), local 19
    ('max', 64, 65),             # local 1, global 2
    ('max', 1200, 8),            # local 19, global 1
    ('uniform', 65, 64),         # QSTN and global 1, local 2
    ('uniform', 1536, 1000),     # local 24, QSTN and global 16
    ('regression', 128, 4096),   # local 2, QSTN and global 64
    ('regression', 300, 1000),   # local 5, QSTN and global 16
    ('shared_encoder', 8, 64),   # every pass 1 + 1: one pair, split by the boundary
    ('shared_encoder', 300, 65),  # 5 + 2 (boundary inside pair 2)
    ('shared_encoder', 75, 1000),  # 2 + 16 (boundary between pairs)
    ('shared_encoder', 1200, 4096),  # 19 + 64 (boundary inside pair 9), odd total 83
]
BATCHES = (66 * 8 + 1, 66 * 10 - 1, 66 * 12, 33 * 17)
TWO_SEGMENT = {'vanilla', 'shared_encoder'}


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def engine(sd, variant, P, S, guard_band):
    v = synth.VARIANTS[variant]
    return ops.Engine(sd, v['use_point_stn'], v['shared_transformer'], points_per_patch=P, sub_sample_size=S,
                      precision='tc', guard_band=guard_band, output_dim=v.get('output_dim', 2),
                      single_transformer=v.get('single_transformer', 0))


def aux_rows(variant, aux):
    B = aux['trans'].shape[0]
    feats = [aux['feat_max']] if variant == 'shared_encoder' else [aux['feat_local_max'], aux['feat_global_max']]
    return torch.cat([aux['trans'].reshape(B, 9)] + feats, 1)


def stream_counts():
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    return {'tc': (sm // ps.KSPLIT, sm // (2 * ps.KSPLIT)), 'tc_precise': (sm // 8,)}


def sample(B):
    """First four and last two queries of stream 0 and of the last stream, for every stream count an engine may run."""
    out = set()
    for counts in stream_counts().values():
        for ns in counts:
            for stream in (0, ns - 1):
                nq = ps.queries_of_stream(B, stream, ns)
                out |= {ps.query_index(stream, qi, ns) for qi in (0, 1, 2, 3, nq - 2, nq - 1)}
    return sorted(out)


def bound_ratios(Pm, variant, args, name, logits, aux):
    """Worst error-to-bound ratio and its (query, channel) per output, as check_bound in test_gpu_net_kernels.py and
    test_gpu_shared_encoder.py computes them."""
    R = aux['trans']
    if variant == 'shared_encoder':
        ref = shared_oracle(Pm, args, name, R)
        feats = ('feat_max',)
    else:
        R = R if synth.VARIANTS[variant]['use_point_stn'] else None
        ref = net_oracle(Pm, variant, args, name, R)
        feats = ('feat_global_max', 'feat_local_max')
    ratios = {k: nb.worst(nb.excess(aux[k], ref[k])) for k in feats}
    ratios['logits'] = nb.worst(nb.excess(logits, ref['logits']))
    if 'R' in ref:
        R64, eR = ref['R']
        err = (R.double() - R64).abs()
        ratios['R'] = nb.worst(torch.where(err == 0, torch.zeros_like(err), err / eR))
    return ratios


def where(q, ns):
    return 'query %d (stream %d, qi %d of %d streams)' % (q, q % ns, q // ns, ns)


def assert_rows_equal(tag, got, want, queries, ns):
    diff = (got != want).reshape(got.shape[0], -1)
    rows = torch.nonzero(diff.any(1)).reshape(-1)
    if rows.numel():
        r = int(rows[0])
        col = int(torch.nonzero(diff[r])[0])
        raise AssertionError('%s: %d rows differ; first %s, column %d: %r vs %r'
                             % (tag, rows.numel(), where(int(queries[r]), ns), col, float(got[r, col]), float(want[r, col])))


@pytest.mark.parametrize('variant,P,S', CASES)
def test_pass_exchange(variant, P, S):
    B = BATCHES[CASES.index((variant, P, S)) % len(BATCHES)]
    seed = P * 13 + S
    sd = synth.make_state_dict(variant, seed=seed % 97)
    args = [cu(a) for a in (synth.make_model_inputs(B, P, S, seed=seed)[k] for k in KEYS)]
    picked = sample(B)
    perm = torch.from_numpy(np.random.RandomState(seed).permutation(B)).to(DEV)
    shared = variant == 'shared_encoder'
    Pm = nb.to_device(sorc.fold_params(sd) if shared else nb.fold_params(sd, variant), DEV)
    counts = stream_counts()
    pt, st = ps.seg_tiles(P), ps.seg_tiles(S)
    tiles = [pt + st] if shared else ([pt + st] if variant == 'vanilla' else []) + [pt, st]
    print('%s P %d S %d: B %d, tiles per launch %s, queries per stream %s, sample %s'
          % (variant, P, S, B, tiles, {n: [-(-B // ns) for ns in c] for n, c in counts.items()}, picked))

    if variant in TWO_SEGMENT and pt % 2:
        # c. the pair (pt - 1, pt) holds the last patch tile and the first sub-sample tile; over the sampled queries of
        # stream 0, every CTA of the cluster and both of its warpgroups produce the patch tile and receive it
        for part in range(ps.KSPLIT):
            for wg in range(ps.KWG):
                roles = set()
                for qi in range(wg, 4, ps.KWG):
                    tq = ps.step_tile(pt - 1, ps.own_tile(part, wg, qi))
                    roles.add(ps.is_mine(pt - 1, tq, pt + st) and tq == pt - 1)
                assert roles == {True, False}, (part, wg)

    bad, worst = [], {}
    for name, band in ENGINES.items():
        ns = counts[name][0]
        eng = engine(sd, variant, P, S, band)
        logits = eng.forward(*args)
        _, aux = eng.forward_with_aux(*args)
        rows = aux_rows(variant, aux)
        # a. permutation of the batch; every query alone (logits), the sampled ones also with their aux rows
        lp = eng.forward(*[a[perm] for a in args])
        rp = aux_rows(variant, eng.forward_with_aux(*[a[perm] for a in args])[1])
        assert_rows_equal('%s permuted logits' % name, lp, logits[perm], perm.cpu(), ns)
        assert_rows_equal('%s permuted aux' % name, rp, rows[perm], perm.cpu(), ns)
        la = torch.cat([eng.forward(*[a[q:q + 1] for a in args]) for q in range(B)])
        assert_rows_equal('%s alone logits' % name, la, logits, range(B), ns)
        ra = torch.cat([aux_rows(variant, eng.forward_with_aux(*[a[q:q + 1] for a in args])[1]) for q in picked])
        assert_rows_equal('%s alone aux' % name, ra, rows[picked], picked, ns)
        eng.close()
        # b. the sample's rows of the full batch against the float64 network
        idx = torch.tensor(picked, device=DEV)
        sa = [a[idx] for a in args]
        saux = {k: t[idx] for k, t in aux.items()}
        ratios = bound_ratios(Pm, variant, sa, name, logits[idx], saux)
        worst[name] = max(r for r, _ in ratios.values())
        print('  %s: %s' % (name, ', '.join('%s %.3g at %s' % (k, r, where(picked[at[0]], ns))
                                           for k, (r, at) in ratios.items())))
        bad += [(name, k, r, where(picked[at[0]], ns)) for k, (r, at) in ratios.items() if not r <= 1.0]
    print('  worst bound ratio %s' % {k: round(v, 4) for k, v in worst.items()})
    assert not bad, bad
