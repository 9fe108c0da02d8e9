"""Every sub-sample kernel against the exact law of the reference's draw.

Weighted: the cases of tests/subsample_cases.py put every geometry class on each of the three kernels (cells, cached and
uncached clocks), which the cloud size selects; the inclusion counts are tested per point against Binomial(T, pi_i) and per
distance bin by batch means, with pi from oracle/subsample_law.py, and the tiny clouds by Pearson chi-square over all sets.
Uniform: chi-square on ids and on pairs of adjacent slots inside and across Philox quads.
Ball query: inclusion k / count for every point of the ball and pairwise inclusion k (k-1) / (count (count-1)) on pairs of
ids that share a Philox quad, on each branch (count <= k, k < count <= 2048, count > 2048)."""
import numpy as np
import pytest
import torch
from scipy import stats

from oracle import p2s_oracle as orc
from oracle import subsample_law as law
from points2surf_b200 import ops, synth
import subsample_cases as sc

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
SEED = 20261016


@pytest.fixture(scope='module')
def law_counts():
    res = {}
    for name, c in sc.cases().items():
        cloud = torch.from_numpy(c['cloud']).to(DEV)
        N, S, T = len(c['cloud']), c['S'], c['T']
        per = T // sc.BATCHES
        q = torch.from_numpy(np.ascontiguousarray(np.repeat(c['query'][None], per, axis=0))).to(DEV)
        counts = torch.zeros((sc.BATCHES, N), dtype=torch.int64, device=DEV)
        sets = torch.zeros(1 << N if N <= 16 else 1, dtype=torch.int64, device=DEV)
        dup = 0
        for b in range(sc.BATCHES):
            ids = ops.subsample(cloud, q, S, False, SEED, query_index_base=b * per).long()
            counts[b] = torch.bincount(ids.view(-1), minlength=N)
            s = torch.sort(ids, dim=1).values
            dup += int((s[:, 1:] == s[:, :-1]).sum()) + int(((s < 0) | (s >= N)).sum())
            if N <= 16:
                sets += torch.bincount((1 << ids).sum(1), minlength=1 << N)
        res[name] = dict(counts=counts.cpu().numpy(), sets=sets.cpu().numpy(), dup=dup)
    return res


@pytest.mark.parametrize('name', sc.runs())
def test_weighted_kernel_realises_the_law(law_counts, name):
    c = sc.cases()[name]
    cloud, q, S, T = c['cloud'], c['query'], c['S'], c['T']
    N = len(cloud)
    got = law_counts[name]
    assert int(got['dup']) == 0                                  # S distinct ids in range in every trial
    w = law.weights(cloud, q)
    pi = law.inclusion_probabilities(w, S, device=DEV)
    counts = got['counts'].sum(0)
    zmax, p = sc.point_stats(counts, T, pi)
    bins = law.equal_mass_bins(pi, np.linalg.norm(cloud.astype(np.float64) - q.astype(np.float64), axis=1))
    t = sc.binned_t(got['counts'], T, pi, bins)
    tmax = float(np.nanmax(np.abs(np.where(np.isfinite(t), t, 0.0))))
    print('%s [%s]: T=%d max|z|=%.2f max|t|=%.2f (bound %.2f)' % (name, sc.kernel_for(N, S), T, zmax, tmax, sc.t_bound()))
    assert p > sc.ALPHA, (name, zmax, p)
    assert tmax < sc.t_bound(), (name, t)
    if N <= 16:
        full = law.set_law(w, S)
        keys = [sum(1 << i for i in s) for s in full]
        exp = np.array([full[s] for s in full]) * T
        obs = got['sets'][keys]
        assert obs.sum() == T
        chi2 = float(((obs - exp) ** 2 / exp).sum())
        print('  chi2 over %d sets = %.1f (bound %.1f)' % (len(keys), chi2, stats.chi2.isf(sc.ALPHA, len(keys) - 1)))
        assert chi2 < stats.chi2.isf(sc.ALPHA, len(keys) - 1)


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def test_uniform_subsample_ids_and_adjacent_pairs():
    N, S, T = 1000, 1000, 4096
    cloud = synth.make_cloud('sphere', N, seed=1)
    ids = ops.subsample(cu(cloud), cu(np.zeros((T, 3), np.float32)), S, True, seed=SEED).long()
    cnt = torch.bincount(ids.view(-1), minlength=N).cpu().numpy()
    chi2 = float(((cnt - T * S / N) ** 2 / (T * S / N)).sum())
    bound = stats.chi2.isf(sc.ALPHA / 3, N - 1)
    print('uniform ids: chi2 %.1f (bound %.1f)' % (chi2, bound))
    assert chi2 < bound
    # pairs of adjacent slots (j, j+1) in 16 x 16 id buckets: inside a Philox quad (j % 4 < 3) and across quads (j % 4 == 3)
    a, b = ids[:, :-1] * 16 // N, ids[:, 1:] * 16 // N
    j = torch.arange(S - 1, device=ids.device)
    for name, sel in (('inside', j % 4 < 3), ('across', j % 4 == 3)):
        pc = torch.bincount((a[:, sel] * 16 + b[:, sel]).reshape(-1), minlength=256).cpu().numpy()
        size = np.bincount(np.arange(N) * 16 // N, minlength=16)         # 62 or 63 ids per bucket
        e = pc.sum() * np.outer(size, size).ravel() / N ** 2
        chi2 = float(((pc - e) ** 2 / e).sum())
        bound = stats.chi2.isf(sc.ALPHA / 3, 255)
        print('uniform pairs %s quads: chi2 %.1f (bound %.1f)' % (name, chi2, bound))
        assert chi2 < bound


@pytest.mark.parametrize('branch', ['all', 'sort', 'histogram'])
def test_ball_subset_inclusion_and_pairs(branch):
    k = 32 if branch != 'histogram' else 300
    if branch == 'histogram':
        rng = np.random.RandomState(0)
        cloud = (rng.standard_normal((30000, 3)) * 0.05).clip(-0.9, 0.9).astype(np.float32)
        q, radius = np.zeros(3, np.float32), 0.1
    else:
        cloud = synth.make_cloud('sphere', 20000, seed=3)
        q, radius = cloud[0].copy(), (0.02 if branch == 'all' else 0.08)
    ball = np.array(sorted(orc.make_kdtree(cloud).query_ball_point(q, radius)))
    count = len(ball)
    assert {'all': count <= k, 'sort': k < count <= 2048, 'histogram': count > 2048}[branch], count
    T = sc.BATCHES * 64
    ids, _, _, counts = ops.ball_patch(cu(cloud), cu(np.repeat(q[None], T, axis=0)), k, radius, seed=SEED)
    assert (counts == count).all()
    ids = ids.long()
    if count <= k:
        assert (ids[:, :count].cpu().numpy() == ball[None]).all()
        return
    s = torch.sort(ids, dim=1).values
    assert not (s[:, 1:] == s[:, :-1]).any()
    inb = torch.zeros(len(cloud), dtype=torch.bool, device=DEV)
    inb[cu(ball)] = True
    assert inb[ids].all()
    cnt = torch.bincount(ids.view(-1), minlength=len(cloud)).cpu().numpy()[ball]
    zmax, p = sc.point_stats(cnt, T, np.full(count, k / count))
    # selected pairs that share a Philox quad (same id >> 2), per trial, against their expectation
    qsel = (s >> 2)
    same = (qsel[:, :, None] == qsel[:, None, :]).sum((1, 2)) - k                               # ordered pairs, i != j
    bq = np.bincount(ball >> 2)
    pairs_ball = float((bq * (bq - 1)).sum())
    want = pairs_ball * k * (k - 1) / (count * (count - 1))
    bm = same.double().view(sc.BATCHES, -1).mean(1).cpu().numpy()
    t = (bm.mean() - want) / (bm.std(ddof=1) / np.sqrt(sc.BATCHES))
    print('ball %s: count %d, T=%d max|z|=%.2f, quad pairs t=%.2f (bound %.2f)' % (branch, count, T, zmax, t, sc.t_bound(1)))
    assert p > sc.ALPHA, (zmax, p)
    assert abs(t) < sc.t_bound(1)
