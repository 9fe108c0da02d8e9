"""Inputs of the sub-sample law tests (tests/test_subsample_law_host.py, tests/test_gpu_subsample_law.py).

Each case is one cloud and one query, drawn T times: trial j is query index j, so every trial has its own Philox stream.  T is
64 batches of equal size; the binned test uses batch means because the points of one trial are dependent."""
import numpy as np

from points2surf_b200 import synth

BATCHES = 64
T_LAW = BATCHES * 512          # 32 768 trials: the d_max x 0.99 perturbation of the bench cloud gives an expected |t| >= 10
T_TINY = BATCHES * 2048        # 131 072 trials: every set of the tiny clouds is expected >= 5 times
NBINS = 20
SMEM_CLOUD_MAX = 40960         # csrc/assemble.cu kSmemCloudMax: largest cloud whose per-point shared-memory array fits
FAR_CAP = 864                  # csrc/assemble.cu subsample_cells_kernel: kFarCap far cells fit into the list


def kernel_for(N, S):
    """Which weighted kernel csrc/assemble.cu subsample() launches."""
    if N > SMEM_CLOUD_MAX:
        return 'clocks_uncached'
    return 'cells' if N >= 2 * S else 'clocks_cached'


def _volume(n, seed):
    return np.random.RandomState(seed).uniform(-0.9, 0.9, (n, 3)).astype(np.float32)


def _clustered(n, seed):
    rng = np.random.RandomState(seed)
    centres = rng.uniform(-0.7, 0.7, (20, 3))
    return (centres[rng.randint(0, 20, n)] + rng.standard_normal((n, 3)) * 0.02).astype(np.float32)


def _planar(n, seed):
    c = np.random.RandomState(seed).uniform(-0.9, 0.9, (n, 3)).astype(np.float32)
    c[:, 2] = 0.25
    return c


def _sphere(n, seed=0):
    return synth.make_cloud('sphere', n, seed=seed)


def _tiny(n, seed):
    return np.random.RandomState(seed).uniform(-0.9, 0.9, (n, 3)).astype(np.float32)


def _duplicates(n, seed):
    return np.repeat(_volume(n // 4, seed), 4, axis=0)      # every point four times: exact ties in distance and weight


def _case(cloud, q, S, T=T_LAW):
    return dict(cloud=cloud, query=np.asarray(q, np.float32), S=S, T=T)


def _geometries(suffix, n, seed):
    """Every geometry class at n points and S = 1000: band and on-point queries and a query outside the box on a sphere,
    a far query (every weight at the 0.05 floor), volume, clustered, planar and duplicated clouds."""
    sph = _sphere(n, seed)
    return {
        'band' + suffix: _case(sph, sph[0] * np.float32(0.97), 1000),
        'on_point' + suffix: _case(sph, sph[17], 1000),
        'outside' + suffix: _case(sph, [1.4, -1.25, 1.1], 1000),
        'far' + suffix: _case(_volume(n, seed + 1), [1e6, 3e5, 0.0], 1000),
        'volume' + suffix: _case(_volume(n, seed + 2), [0.2, -0.1, 0.3], 1000),
        'clustered' + suffix: _case(_clustered(n, seed + 3), [0.1, 0.1, -0.2], 1000),
        'planar' + suffix: _case(_planar(n, seed + 4), [0.1, 0.2, 0.5], 1000),
        'duplicates' + suffix: _case(_duplicates(n, seed + 5), [0.3, -0.2, 0.1], 1000),
    }


def cases():
    """name -> dict(cloud [N,3] f32, query [3] f32, S, T).  Every geometry class runs on each of the three weighted kernels:
    the cell kernel (N >= 2S), the cached clocks (S < N < 2S) and the uncached clocks (N > SMEM_CLOUD_MAX)."""
    bench = _sphere(10000)
    return {
        'bench_band': _case(bench, bench[0] * np.float32(0.97), 1000),
        'bench_on_point': _case(bench, bench[17], 1000),
        'bench_outside': _case(bench, [1.4, -1.25, 1.1], 1000),
        # the query is 10^6 cloud extents away: all 1728 cells are far cells (> FAR_CAP), so the far-cell list overflows
        # into the in-place scan.  Only such far queries were found to overflow it (a sphere centred on the query reaches
        # ~625 cells), and at that distance every weight is at the 0.05 floor: the law is uniform.
        'far_cells': _case(_volume(30000, 1), [1e6, 3e5, 0.0], 1000),
        'volume': _case(_volume(10000, 2), [0.2, -0.1, 0.3], 1000),
        'clustered': _case(_clustered(20000, 3), [0.1, 0.1, -0.2], 1000),
        'planar': _case(_planar(10000, 4), [0.1, 0.2, 0.5], 1000),
        'duplicates': _case(_duplicates(10000, 5), [0.3, -0.2, 0.1], 1000),
        **_geometries('_1p5s', 1500, 20),
        **_geometries('_50k', 50000, 30),
        # the size limits of each kernel, on both sides
        'n_2s': _case(_sphere(2000, 5), [0.3, 0.1, -0.4], 1000),
        'n_2s_1': _case(_sphere(1999, 15), [0.3, 0.1, -0.4], 1000),
        'n_38400': _case(_sphere(38400, 6), [0.5, -0.5, 0.2], 1000),
        'n_40960': _case(_sphere(40960, 7), [-0.2, 0.6, 0.1], 1000),
        'n_40960_s20481': _case(_sphere(40960, 16), [-0.2, 0.6, 0.1], 20481),
        'n_40961': _case(_sphere(40961, 17), [0.4, 0.1, -0.3], 1000),
        'n_s': _case(_sphere(1000, 8), [0.1, 0.2, 0.3], 1000),
        'n_s1': _case(_sphere(1001, 9), [0.1, 0.2, 0.3], 1000),
        'n_1p2s': _case(_sphere(1200, 10), [0.6, 0.2, 0.3], 1000),
        'n_1p9s': _case(_sphere(1900, 11), [-0.6, 0.2, 0.3], 1000),
        'n_50000': _case(_sphere(50000, 12), [0.3, 0.3, 0.3], 1000),
        's_1': _case(bench, bench[3] * np.float32(1.02), 1),
        's_1_50k': _case(_sphere(50000, 18), [0.2, -0.3, 0.3], 1),
        # the whole law of the set, on the cell kernel (N >= 2S) and the cached clocks (N < 2S)
        'tiny_8_3': _case(_tiny(8, 13), [0.2, 0.1, 0.0], 3, T_TINY),
        'tiny_8_4': _case(_tiny(8, 19), [0.2, 0.1, 0.0], 4, T_TINY),
        'tiny_8_5': _case(_tiny(8, 14), [0.2, 0.1, 0.0], 5, T_TINY),
        'tiny_7_4': _case(_tiny(7, 21), [0.2, 0.1, 0.0], 4, T_TINY),
    }


def runs():
    """The names of the law cases."""
    return list(cases())


ALPHA = 1e-6                   # false-alarm rate of each statistical test (Bonferroni over its points, bins or sets)


def point_stats(counts, T, pi):
    """Per-point inclusion counts against Binomial(T, pi_i) -> (largest |z|, smallest Bonferroni-corrected p-value)."""
    from scipy import stats
    pi = np.clip(pi, 0.0, 1.0)
    sd = np.sqrt(T * pi * (1 - pi))
    z = np.where(sd > 0, (counts - T * pi) / np.where(sd > 0, sd, 1), np.where(counts == np.round(T * pi), 0.0, np.inf))
    p = np.minimum(1.0, 2 * np.minimum(stats.binom.cdf(counts, T, pi), stats.binom.sf(counts - 1, T, pi)))
    p = np.where(sd > 0, p, np.where(np.isfinite(z), 1.0, 0.0))
    return float(np.abs(z).max()), float(p.min() * len(pi))


def binned_t(batch_counts, T, pi, bins, nbins=NBINS):
    """Bin totals per trial, by batch means over the BATCHES batches -> t statistic per bin."""
    per = T / batch_counts.shape[0]
    tot = np.stack([np.bincount(bins, weights=bc, minlength=nbins) for bc in batch_counts]) / per
    want = np.bincount(bins, weights=pi, minlength=nbins)
    sd = tot.std(axis=0, ddof=1)
    return (tot.mean(axis=0) - want) / np.where(sd > 0, sd, np.inf) * np.sqrt(batch_counts.shape[0])


def t_bound(nbins=NBINS):
    from scipy import stats
    return float(stats.t.isf(ALPHA / (2 * nbins), BATCHES - 1))
