"""The exact law of the distance-weighted sub-sample (oracle/subsample_law.py) against full enumeration, simulation and the
reference's own sampler, and the power of the GPU law tests (tests/test_gpu_subsample_law.py) against perturbed laws."""
import numpy as np
import pytest

from oracle import p2s_oracle as orc
from oracle import subsample_law as law
import subsample_cases as sc

TINY = [n for n in sc.runs() if n.startswith('tiny_')]


@pytest.mark.parametrize('N,S', [(5, 2), (8, 3), (8, 5), (9, 1), (9, 4), (9, 8)])
def test_integral_matches_enumeration(N, S):
    rng = np.random.RandomState(N * 10 + S)
    for w in (rng.uniform(0.05, 1.0, N), np.r_[np.full(N - 2, 0.05), 1.0, 0.5]):
        exact = law.set_inclusion(law.set_law(w, S), N)
        assert abs(sum(law.set_law(w, S).values()) - 1) < 1e-13
        assert np.abs(law.inclusion_probabilities(w, S) - exact).max() < 1e-12


def test_tiny_cases_match_enumeration():
    for name in TINY:
        c = sc.cases()[name]
        w = law.weights(c['cloud'], c['query'])
        exact = law.set_inclusion(law.set_law(w, c['S']), len(w))
        assert np.abs(law.inclusion_probabilities(w, c['S']) - exact).max() < 1e-12


@pytest.mark.parametrize('name', ['bench_band', 'bench_on_point', 'bench_outside', 'n_1p2s', 'n_s1', 'planar'])
def test_inclusion_sums_to_s(name):
    c = sc.cases()[name]
    pi = law.inclusion_probabilities(law.weights(c['cloud'], c['query']), c['S'])
    assert abs(pi.sum() - c['S']) < 1e-9 and pi.min() > 0 and pi.max() <= 1 + 1e-12


def test_equal_weights_single_draw_and_full_draw():
    assert np.abs(law.inclusion_probabilities(np.full(3000, 0.37), 700) - 700 / 3000).max() < 1e-12
    w = np.random.RandomState(1).uniform(0.05, 1.0, 2500)
    assert np.abs(law.inclusion_probabilities(w, 1) - w / w.sum()).max() < 1e-12
    assert (law.inclusion_probabilities(w, 2500) == 1).all()


def test_interpolation_matches_direct_evaluation(monkeypatch):
    w = np.random.RandomState(2).uniform(0.05, 1.0, 1000)
    interp = law.inclusion_probabilities(w, 200)
    monkeypatch.setattr(law, '_DIRECT', 10 ** 9)
    direct = law.inclusion_probabilities(w, 200)
    assert np.abs(interp - direct).max() < 1e-10


def _es_counts(w, S, T, seed, chunk=500):
    """Efraimidis-Spirakis in float64: the S smallest clocks E_i / w_i -> per-point counts and per-trial id sets."""
    rng = np.random.RandomState(seed)
    counts = np.zeros(len(w), np.int64)
    sets = []
    for b in range(0, T, chunk):
        clocks = rng.standard_exponential((min(chunk, T - b), len(w))) / w[None, :]
        ids = np.argpartition(clocks, S - 1, axis=1)[:, :S]
        counts += np.bincount(ids.ravel(), minlength=len(w))
        sets.append(ids)
    return counts, np.concatenate(sets)


def test_agrees_with_efraimidis_spirakis_simulation():
    rng = np.random.RandomState(4)
    w = rng.uniform(0.05, 1.0, 2000)
    T = 4000
    counts, _ = _es_counts(w, 500, T, seed=5)
    _, p = sc.point_stats(counts, T, law.inclusion_probabilities(w, 500))
    assert p > sc.ALPHA, p


def test_agrees_with_randomstate_choice():
    rng = np.random.RandomState(3)
    cloud = rng.uniform(-0.9, 0.9, (40, 3)).astype(np.float32)
    q = np.array([0.3, -0.2, 0.1], np.float32)
    prob = orc.sub_sample_probabilities(cloud, q)
    rs = np.random.RandomState(5)
    T = 6000
    counts = np.bincount(np.concatenate([rs.choice(40, size=10, replace=False, p=prob) for _ in range(T)]), minlength=40)
    _, p = sc.point_stats(counts, T, law.inclusion_probabilities(law.weights(cloud, q), 10))
    assert p > sc.ALPHA, p


def test_tiny_cases_expect_every_set_five_times():
    for name in TINY:
        c = sc.cases()[name]
        probs = np.array(list(law.set_law(law.weights(c['cloud'], c['query']), c['S']).values()))
        assert probs.min() * c['T'] >= 5, (name, probs.min() * c['T'])


@pytest.mark.parametrize('name', ['bench_band', 'bench_on_point', 'bench_outside'])
def test_binned_statistic_rejects_perturbed_laws(name):
    """Expected |t| of the GPU test's binned statistic at T = T_LAW if the kernel realised a perturbed law: d_max x 0.99, a
    0.048 clamp floor, uniform weights.  The per-trial variance of each bin total comes from an Efraimidis-Spirakis simulation
    of the true law."""
    c = sc.cases()[name]
    cloud, q, S, T = c['cloud'], c['query'], c['S'], c['T']
    w = law.weights(cloud, q)
    pi = law.inclusion_probabilities(w, S)
    bins = law.equal_mass_bins(pi, np.linalg.norm(cloud.astype(np.float64) - q.astype(np.float64), axis=1))
    _, sets = _es_counts(w, S, 2000, seed=6)
    var = np.bincount(bins[sets.ravel()] + sc.NBINS * np.repeat(np.arange(len(sets)), S),
                      minlength=sc.NBINS * len(sets)).reshape(len(sets), sc.NBINS).var(axis=0, ddof=1)
    want = np.bincount(bins, weights=pi, minlength=sc.NBINS)
    for alt in (law.weights(cloud, q, dmax_scale=0.99), law.weights(cloud, q, floor=0.048), np.ones(len(w))):
        alt_tot = np.bincount(bins, weights=law.inclusion_probabilities(alt, S), minlength=sc.NBINS)
        t = np.abs(alt_tot - want) * np.sqrt(T / var)
        assert t.max() >= 10, (name, t.max())
