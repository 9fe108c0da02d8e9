"""GPU tests of the library scratch (include/p2s_b200.h, "Scratch memory"): launch counts of every driver, results that do
not depend on what ran before, CUDA graphs that survive later growth of the training GEMMs' scratch, and one thread
calling the drivers on two devices."""
import math
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

from points2surf_b200 import ops, synth, trafo
from points2surf_b200.train_ops import CudaPrims
from helpers import load_golden

pytestmark = pytest.mark.gpu


def _sphere_mesh(dev, res):
    x = torch.linspace(-1, 1, res, device=dev)
    X, Y, Z = torch.meshgrid(x, x, x, indexing='ij')
    return ops.marching_cubes((0.6 - torch.sqrt(X * X + Y * Y + Z * Z)).contiguous(), 0.0)


def _dirty(v, f):
    """a mesh that takes every branch of mesh_clean: duplicated vertices, a duplicate face, holes, flipped faces"""
    f = f.clone()
    f[::7] = f[::7].flip(1)
    f = torch.cat([f[:-3], f[:1]])
    v = torch.cat([v, v[:5]])
    return v, f


def _scan_poses(n):
    g = load_golden('scan.npz')
    rot = np.stack([trafo.quaternion_matrix(q)[:3, :3] for q in g['rotations_0']])[:n]
    return rot, g['locations_0'][:n]


def _inputs(dev, large):
    """fixed inputs of every driver, at two sizes"""
    n = 30000 if large else 3000
    cloud = torch.from_numpy(synth.make_cloud('sphere', n, seed=3)).to(dev)
    v, f = _sphere_mesh(dev, 96 if large else 24)
    g = torch.Generator().manual_seed(5)
    q = (torch.rand((20000 if large else 500, 3), generator=g) * 2.4 - 1.2).to(dev)
    res = 64 if large else 16
    lin = ops.query_grid(cloud, res, 3)
    sdf = 0.3 - ops.query_points(lin, res).norm(dim=1)
    nrm = cloud / cloud.norm(dim=1, keepdim=True)
    rot, loc = _scan_poses(4 if large else 1)
    return dict(cloud=cloud, v=v, f=f, q=q, res=res, lin=lin, sdf=sdf, nrm=nrm, rot=rot, loc=loc,
                queries=cloud[:(2000 if large else 100)])


DRIVERS = {
    'query_grid': lambda x: ops.query_grid(x['cloud'], x['res'], 3),
    'sdf_to_volume': lambda x: ops.sdf_to_volume(x['lin'], x['sdf'], x['res'], 5, 13.0),
    'marching_cubes': lambda x: _sphere_mesh(x['v'].device, 2 * x['res']),
    'mesh_sample': lambda x: ops.mesh_sample(x['v'], x['f'], 10000, seed=1, return_face_ids=True),
    'nn_distance': lambda x: ops.nn_distance(x['q'], x['cloud']),
    'chamfer_hausdorff': lambda x: ops.chamfer_hausdorff(x['q'], x['cloud']),
    'mesh_signed_distance': lambda x: ops.mesh_signed_distance(x['v'], x['f'], x['q'], True, True),
    'mesh_closest_point': lambda x: ops.mesh_closest_point(x['v'], x['f'], x['q']),
    'mesh_clean': lambda x: ops.mesh_clean(*_dirty(x['v'], x['f'])),
    'poisson_solve': lambda x: ops.poisson_solve(x['cloud'], x['nrm'], depth=6),
    'range_scan': lambda x: ops.range_scan(x['v'], x['f'], x['rot'], x['loc'], noise_sigma=0.01, seed=2),
    'knn_patch': lambda x: ops.knn_patch(x['cloud'], x['queries'], 300),
    'ball_patch': lambda x: ops.ball_patch(x['cloud'], x['queries'], 300, 0.1, seed=4),
    'subsample_weighted': lambda x: ops.subsample(x['cloud'][:20000], x['queries'], 1000, False, seed=6),
}

# launches of one call on the small inputs (ops.launch_count(): every kernel, CUB counted per call site)
LAUNCHES = {'query_grid': 8, 'sdf_to_volume': 6, 'marching_cubes': 16, 'mesh_sample': 3, 'nn_distance': 3,
            'chamfer_hausdorff': 6, 'mesh_signed_distance': 3, 'mesh_closest_point': 3, 'mesh_clean': 50,
            'poisson_solve': 555, 'range_scan': 8, 'knn_patch': 1, 'ball_patch': 1, 'subsample_weighted': 7}


def _flat(r):
    if isinstance(r, dict):
        return [r[k] for k in sorted(r) if k != 'stage_ms']
    if isinstance(r, (tuple, list)):
        return [y for z in r for y in _flat(z)]
    return [r]


def _assert_same(a, b, name):
    a, b = _flat(a), _flat(b)
    assert len(a) == len(b), name
    for x, y in zip(a, b):
        if isinstance(x, torch.Tensor):
            assert x.shape == y.shape and torch.equal(x.cpu(), y.cpu()), name
        elif isinstance(x, float) and math.isnan(x):
            assert math.isnan(y), name
        else:
            assert x == y, name


def _run(name, x):
    r = DRIVERS[name](x)
    if name == 'chamfer_hausdorff':
        # the sums are float atomics (order varies from run to run); the maxima are exact
        r = {k: v for k, v in r.items() if k != 'chamfer'}
    torch.cuda.synchronize()
    return r


def _in_new_thread(fn):
    """runs fn on a new thread, whose library scratch starts empty whatever earlier tests ran (scratch is per thread)"""
    with ThreadPoolExecutor(1) as ex:
        return ex.submit(fn).result()


def launch_counts(dev='cuda:0'):
    x = _inputs(dev, False)
    out = {}
    for name in DRIVERS:
        _run(name, x)
        before = ops.launch_count()
        _run(name, x)
        out[name] = ops.launch_count() - before
    return out


def test_launch_counts():
    got = launch_counts()
    assert got == LAUNCHES


def test_reuse_after_other_sizes():
    _in_new_thread(_reuse_after_other_sizes)


def _reuse_after_other_sizes():
    small, large = _inputs('cuda:0', False), _inputs('cuda:0', True)
    for name in DRIVERS:
        ref_small = _run(name, small)
        ref_large = _run(name, large)
        _assert_same(_run(name, small), ref_small, name)
        _assert_same(_run(name, large), ref_large, name)


def test_graph_survives_scratch_growth():
    _in_new_thread(_graph_survives_scratch_growth)


def _graph_survives_scratch_growth():
    prims = CudaPrims()
    g = torch.Generator().manual_seed(7)
    rnd = lambda *s: torch.randn(*s, generator=g).cuda()
    # gemm_nt takes the tensor-core path at M >= 128; gemm_tn at M >= 4096, and with >= 2 tiles per SM pair it runs
    # one split, so its atomics add to zero exactly once and the result is bitwise reproducible
    M, N, K = 512, 256, 128
    Mt, Nt, Kt = 4096, 2048, 4096
    A, W, b = rnd(M, K), rnd(N, K), rnd(N)
    At, Bt = rnd(Mt, Nt), rnd(Mt, Kt)
    prims.gemm_nt(A, W, b)
    prims.gemm_nt(A, W)
    prims.gemm_tn(At, Bt)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out_nt = prims.gemm_nt(A, W, b)
        out_nt0 = prims.gemm_nt(A, W)
        out_tn = prims.gemm_tn(At, Bt)
    # eager calls at larger shapes grow the scratch the graph holds
    prims.gemm_nt(rnd(8 * M, K), W, b)
    prims.gemm_tn(rnd(Mt, 2 * Nt), rnd(Mt, Kt))
    torch.cuda.synchronize()
    for _ in range(2):
        A.copy_(rnd(M, K))
        At.copy_(rnd(Mt, Nt))
        Bt.copy_(rnd(Mt, Kt))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out_nt, prims.gemm_nt(A, W, b))
        assert torch.equal(out_nt0, prims.gemm_nt(A, W))
        assert torch.equal(out_tn, prims.gemm_tn(At, Bt))
    # a first call of a larger shape inside a capture is refused before it launches anything
    big = rnd(64 * M, K)
    with pytest.raises(ops.P2SError, match='eager call of the same size first'):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            prims.gemm_nt(big, W, b)
    torch.cuda.synchronize()
    assert torch.equal(prims.gemm_nt(A, W, b), out_nt)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs two GPUs')
def test_two_devices_one_thread():
    x0, x1 = _inputs('cuda:0', True), _inputs('cuda:1', True)
    for name in DRIVERS:
        ref = _run(name, x0)
        _assert_same(_run(name, x1), ref, name)
        _assert_same(_run(name, x0), ref, name)
