"""kNN patches bit for bit: the ids are the first k of lexsort((id, d2_f64)) (orc.knn_bruteforce, cKDTree semantics with ties
broken by id), and the radius and patch are NumPy float32 on those ids.  Swept over k at the edges of the register sort,
the 1024- and 2048-candidate instantiations and the histogram candidate cap; over clouds with many exact ties; over query
orders that select the fast path (voxel order, repeated queries) or the histogram path (shuffled); and over coordinate scales
whose squared distances fall outside the histogram's unclamped range 2^-100 .. 2^27."""
import numpy as np
import pytest
import torch

from oracle import p2s_oracle as orc
from points2surf_b200 import ops, synth

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
KS = [1, 2, 63, 64, 65, 256, 300, 511, 512, 513, 1024, 1200, 1536]


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def check_exact(cloud, q, k):
    ids, patch, radius = (t.cpu().numpy() for t in ops.knn_patch(cu(cloud), cu(q), k))
    for i in range(len(q)):
        want, _ = orc.knn_bruteforce(cloud, q[i], k)
        assert np.array_equal(ids[i], want), (i, k)
        d = np.linalg.norm(np.repeat(q[i][None], k, axis=0) - cloud[want], axis=1)
        r = np.max(d)
        assert radius[i] == r, (i, k)
        assert np.array_equal(patch[i], ((cloud[want] - q[i][None]) / r).astype(np.float32)), (i, k)
    return ids


def torus():
    return synth.make_cloud('torus', 7000, seed=4)


def lattice():
    g = np.arange(-10, 10, dtype=np.float32) / np.float32(16)           # exact binary fractions: many equal distances
    return np.stack(np.meshgrid(g, g, g, indexing='ij'), -1).reshape(-1, 3)


def duplicates():
    c = torus()
    q = orc.query_grid(c, 32, 3)[100]
    order, _ = orc.knn_bruteforce(c, q, 700)
    c[order[250:350]] = c[order[300]]                                    # 100 copies straddle the 300-th, 512-th... ranks
    return c


CLOUDS = {'torus': torus, 'lattice': lattice, 'duplicates': duplicates}


def queries(cloud, order):
    if order == 'voxel':                                                 # consecutive voxel centres: fast path
        return orc.query_grid(cloud, 32, 3)[90:114]
    base = orc.query_grid(cloud, 32, 3)
    if order == 'shuffled':                                              # jumps between queries: histogram path
        return base[np.random.RandomState(1).permutation(len(base))[:24]]
    return np.repeat(base[[100, 300, 500]], 8, axis=0)                 # runs of one repeated query: fast path, step 0


@pytest.mark.parametrize('order', ['voxel', 'shuffled', 'repeated'])
@pytest.mark.parametrize('cloud', list(CLOUDS))
def test_knn_exact_over_k(cloud, order):
    c = CLOUDS[cloud]()
    q = queries(c, order)
    if cloud == 'lattice':
        q = (np.round(q * 32) / 32).astype(np.float32)                   # on lattice points and half-way between them
    for k in KS:
        ids = check_exact(c, q, k)
        if order == 'repeated':
            assert (ids.reshape(3, 8, k) == ids.reshape(3, 8, k)[:, :1]).all()


@pytest.mark.parametrize('scale', [2.0 ** 15, 2.0 ** -15, 2.0 ** 16, 2.0 ** 20, 2.0 ** -50])
@pytest.mark.parametrize('order', ['voxel', 'shuffled'])
def test_knn_exact_far_from_unit_scale(scale, order):
    # squared distances above 2^27 or below 2^-100 share the clamped histogram bins, which must still refine in key order
    c = torus()
    q = queries(c, order)
    s = np.float32(scale)
    for k in (300, 1200):
        check_exact(c * s, q * s, k)


def test_knn_more_exact_ties_than_the_candidate_buffer():
    c = torus()
    q = queries(c, 'shuffled')[:4]
    order, _ = orc.knn_bruteforce(c, q[0], 1700)
    c[order[100:1700]] = c[order[200]]                                   # 1 600 copies around the 300-th rank > kCap = 1024
    with pytest.raises(ops.P2SError):
        ops.knn_patch(cu(c), cu(q), 300)
    check_exact(torus(), q, 300)                                         # the error flag was cleared
