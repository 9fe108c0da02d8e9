"""GPU tests of the exact mesh queries (csrc/meshsdf.cu: p2s_mesh_signed_distance_dev, p2s_mesh_closest_point_dev) at
every coordinate scale, across the query chunks and the face slabs, on sliver faces, and of the solid voxelisation
(csrc/inside.cu) at the production resolution and up to res 1024.

- Scale law.  Multiplying the mesh and the queries by 2^k is exact in fp32, and every float64 operation of the recompute
  and of the winding number then scales exactly, so the header's contract implies d(2^k M, 2^k q) = 2^k d(M, q) bit for
  bit, the same face and winding number, 2^k times the closest point, and the sign by the header's rule.
- Chunks (2^18 queries per launch) and slabs (face ranges that depend on F alone): bitwise independent of the query
  split; a sample that holds both sides of every chunk boundary within a float64-derived bound of tests/mesh_query_torch.py;
  the lowest face index wins ties inside a slab, across slabs and across a slab boundary.
- Solid voxelisation: bit for bit against oracle/inside_oracle.py at res 256, 512, 993 and 1024 (above 256 the oracle's
  crossings are turned into flags on the device), with vertices at |x|, |y| = 16 - 2^-20 and faces below the fixed-point
  step, and against the winding-number parity at res 256."""
import numpy as np
import pytest
import torch

import inside_cases as ic
import mesh_query_torch as mqt
from oracle import inside_oracle as io
from points2surf_b200 import ops
from test_gpu_mesh_sdf import _fixture, _mc_mesh, _stress_points, cu

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
CHUNK = 1 << 18          # queries per launch of meshsdf.cu (kChunk)
SCALES = [-60, -40, -31, -20, 0, 20, 31, 33, 36]
FLT_MIN = np.float32(2.0 ** -126)


# ------------------------------------------------------------------ the cases
def _decoy(order):
    """The query 0.05 above the big triangle A; a small triangle B 0.10 away.  An fp32 prefilter that under- or
    overflows on A picks B."""
    v = np.array([[-1, -1, 0], [2, -1, 0], [-1, 2, 0], [0, 0, 0.15], [0.01, 0, 0.15], [0, 0.01, 0.15]], np.float32)
    f = np.array([[3, 4, 5], [0, 1, 2]] if order == 'b_first' else [[0, 1, 2], [3, 4, 5]], np.int32)
    q = np.array([[0, 0, 0.05], [0.3, 0.2, -0.05], [0.5, 0.5, 0.01], [-0.9, -0.9, 0.002], [0.005, 0.002, 0.12]],
                 np.float32)
    return v, f, q


def _fan(n=64):
    """n faces around the apex at the origin, the rim a float32 circle at height 0.05: on the axis every face is nearly
    equally close"""
    t = 2 * np.pi * np.arange(n) / n
    rim = np.stack([np.cos(t), np.sin(t), np.full(n, 0.05)], 1)
    v = np.concatenate([[[0, 0, 0]], rim]).astype(np.float32)
    f = np.array([[0, 1 + i, 1 + (i + 1) % n] for i in range(n)], np.int32)
    z = np.array([0.0, 1e-6, -1e-6, 0.01, -0.01, 0.05, 0.3, -0.3, 2.0, -7.0], np.float32)
    q = np.concatenate([np.stack([np.zeros_like(z), np.zeros_like(z), z], 1),
                        np.stack([np.full_like(z, 1e-4), np.full_like(z, -2e-4), z], 1)]).astype(np.float32)
    return v, f, q


def _scale_case(name):
    if name in ('decoy_b_first', 'decoy_a_first'):
        return _decoy(name[6:])
    if name == 'fan':
        return _fan()
    if name == 'abc0':
        fx = _fixture(0)
        v, f = fx['verts'], fx['faces']
    else:
        v, f = _mc_mesh('sphere', 32)
    return v, f, _stress_points(v, f, np.random.RandomState(len(f)))


def _scaled(x, k):
    """x * 2^k in fp32, asserted exact and normal (no coordinate becomes subnormal)"""
    y = (x.astype(np.float64) * 2.0 ** k).astype(np.float32)
    assert np.array_equal((y.astype(np.float64) * 2.0 ** -k).astype(np.float32), x)
    assert ((y == 0) | (np.abs(y) >= FLT_MIN)).all()
    return y


def _both(v, f, q):
    d, face, w = (t.cpu().numpy() for t in ops.mesh_signed_distance(cu(v), cu(f), cu(q), True, True))
    cp, du, fu = (t.cpu().numpy() for t in ops.mesh_closest_point(cu(v), cu(f), cu(q)))
    return d, face, w, cp, du, fu


def _times_2k(x, k):
    """x * 2^k for fp32 results: exact where the product is normal; where it is subnormal, within half its spacing"""
    return x.astype(np.float64) * 2.0 ** k


def _assert_scaled(got, want0, k, what):
    want = _times_2k(want0, k)
    g = got.astype(np.float64)
    normal = (want == 0) | (np.abs(want) >= FLT_MIN)
    bad = ~((g == want) | (~normal & (np.abs(g - want) <= 2.0 ** -150)))
    assert not bad.any(), (what, k, int(bad.sum()), g[bad][:4], want[bad][:4])


def _dist_bound(d, q, vmax):
    """|d_kernel - d_f64|: the fp32 rounding of the result (2^-24 |d|, doubled) plus the float64 error of both
    formulations, a few ulp of the coordinate scale (bounded by 2^-44 (|q|_inf + vmax))"""
    return 2.0 ** -23 * np.abs(d) + 2.0 ** -44 * (np.abs(q).max(1) + vmax)


def _check_against_reference(v, f, q, d, face, w, cp):
    """the kernel's results on unit-scale inputs against the float64 device reference: distance and point within the
    bound, the face up to float64 ties (its reference distance within the float64 part of the bound of the minimum)"""
    r = {k: t.cpu().numpy() for k, t in mqt.mesh_query(cu(v), cu(f), cu(q)).items()}
    vmax = float(np.abs(v).max())
    bound = _dist_bound(r['d'], q, vmax)
    assert (np.abs(np.abs(d) - r['d']) <= bound).all(), float((np.abs(np.abs(d) - r['d']) / bound).max())
    tie = 2.0 ** -44 * (np.abs(q).max(1) + vmax)
    df = np.sqrt(mqt.face_dist2(cu(v), cu(f), cu(q), cu(face.astype(np.int64))).cpu().numpy())
    assert (df - r['d'] <= tie).all(), float((df - r['d']).max())
    decided = np.abs(r['w'] - 0.5) > 1e-3
    assert np.array_equal(np.signbit(d[decided]), np.signbit(r['signed'][decided]))
    off = r['d'] > 1e-6
    assert np.abs(w[off] - r['w'][off]).max() <= 1e-4
    pt = mqt.closest_on_faces(cu(v), cu(f), cu(q), cu(face.astype(np.int64))).cpu().numpy()   # on the kernel's face
    cbound = 2.0 ** -23 * np.abs(pt).max(1) + 2.0 ** -44 * (np.abs(q).max(1) + vmax)
    assert (np.abs(cp - pt).max(1) <= cbound).all()
    print('%d queries, %d faces: worst |d - d_f64| / bound %.3f, worst point error / bound %.3f' % (
        len(q), len(f), float((np.abs(np.abs(d) - r['d']) / bound).max()), float((np.abs(cp - pt).max(1) / cbound).max())))
    return r


# ------------------------------------------------------------------ scale law
@pytest.mark.parametrize('name', ['abc0', 'sphere', 'decoy_b_first', 'decoy_a_first', 'fan'])
def test_scale_law(name):
    v, f, q = _scale_case(name)
    d0, face0, w0, cp0, du0, fu0 = _both(v, f, q)
    _check_against_reference(v, f, q, d0, face0, w0, cp0)
    if name.startswith('decoy'):   # A, 0.05 below the first query, not the small B 0.10 away
        assert face0[0] == (1 if name == 'decoy_b_first' else 0) and abs(float(d0[0])) == np.float32(0.05)
    failed = {}
    for k in SCALES:
        vk, qk = _scaled(v, k), _scaled(q, k)
        d, face, w, cp, du, fu = _both(vk, f, qk)
        try:
            assert np.array_equal(face, face0), ('face', np.nonzero(face != face0)[0][:8])
            assert np.array_equal(fu, face) and np.array_equal(du, np.abs(d))
            _assert_scaled(np.abs(d), np.abs(d0), k, 'distance')
            _assert_scaled(cp, cp0, k, 'closest point')
            assert np.array_equal(w, w0), 'winding'
            # the sign by the header's rule: inside (w > 0.5) or on the surface (|d| <= 1e-8) is positive
            pos = (w.astype(np.float64) > 0.5) | (np.abs(d) <= 1e-8)
            decided = np.abs(w.astype(np.float64) - 0.5) > 1e-6
            assert np.array_equal(~np.signbit(d[decided]), pos[decided]), 'sign'
        except AssertionError as e:
            failed[k] = '%s (NaN distances: %d, first query d = %r vs %r)' % (
                str(e).splitlines()[0][:200], int(np.isnan(d).sum()), float(d[0]), float(d0[0]) * 2.0 ** k)
    assert not failed, '\n'.join('k = %d: %s' % kv for kv in failed.items())


# ------------------------------------------------------------------ chunks
def _chunk_queries(v, f, n, seed):
    rng = np.random.RandomState(seed)
    fi = rng.randint(0, len(f), n // 2)
    a, b, c = v[f[fi, 0]], v[f[fi, 1]], v[f[fi, 2]]
    r = rng.uniform(0, 1, (len(fi), 2))
    r[r.sum(1) > 1] = 1 - r[r.sum(1) > 1]
    near = a + r[:, :1] * (b - a) + r[:, 1:] * (c - a) + rng.normal(0, 0.01, (len(fi), 3))
    return np.concatenate([near, rng.uniform(-1, 1, (n - len(fi), 3))]).astype(np.float32)


def _sample_around_chunk_boundaries(Q, rng, n=4096):
    edges = np.concatenate([np.arange(max(0, b - 64), min(Q, b + 64)) for b in range(CHUNK, Q, CHUNK)] + [[0, Q - 1]])
    rest = rng.choice(Q, max(0, n - len(edges)), replace=False)
    return np.unique(np.concatenate([edges, rest]))


def _check_chunks(v, f, q, seed):
    Q = len(q)
    vc, fc, qc = cu(v), cu(f), cu(q)
    full = [t.cpu().numpy() for t in ops.mesh_signed_distance(vc, fc, qc, True, True)]
    cfull = [t.cpu().numpy() for t in ops.mesh_closest_point(vc, fc, qc)]
    step = 100003
    parts = [[t.cpu().numpy() for t in ops.mesh_signed_distance(vc, fc, qc[a:a + step], True, True)]
             for a in range(0, Q, step)]
    cparts = [[t.cpu().numpy() for t in ops.mesh_closest_point(vc, fc, qc[a:a + step])] for a in range(0, Q, step)]
    for k in range(3):
        assert full[k].tobytes() == np.concatenate([p[k] for p in parts]).tobytes()
        assert cfull[k].tobytes() == np.concatenate([p[k] for p in cparts]).tobytes()
    sel = _sample_around_chunk_boundaries(Q, np.random.RandomState(seed))
    d, face, w = (x[sel] for x in full)
    _check_against_reference(v, f, q[sel], d, face, w, cfull[0][sel])


@pytest.mark.parametrize('Q', [CHUNK - 1, CHUNK, CHUNK + 1, 2 * CHUNK + 5])
def test_chunks_are_bitwise_split_independent_and_exact(Q):
    fx = _fixture(1)
    v, f = fx['verts'], fx['faces']
    _check_chunks(v, f, _chunk_queries(v, f, Q, Q), Q)


def _scan_grid(i, res=256):
    import os
    from points2surf_b200 import trafo
    v, f = ic.abc(i)
    g = np.load(os.path.join(ic.GOLDEN, 'scan.npz'))
    rot = np.stack([trafo.quaternion_matrix(x)[:3, :3] for x in g['rotations_%d' % i]])
    pts = ops.range_scan(cu(v), cu(f), rot, g['locations_%d' % i], noise_sigma=float(g['sigma_%d' % i]), seed=7)[0]
    return ops.query_points(ops.query_grid(cu(pts.cpu().numpy().astype(np.float32)), res, 3), res).cpu().numpy()


def test_production_size_grid_call():
    """the full res-256 candidate grid of the first abc_minimal scan (573 606 queries, three launches)"""
    v, f = ic.abc(0)
    q = _scan_grid(0)
    assert len(q) > 2 * CHUNK
    _check_chunks(v, f, q, 3)


# ------------------------------------------------------------------ slabs
def _slab_len(F):
    return max(128, -(-(-(-F // 32)) // 128) * 128)


def _slab_mesh(F, rng):
    """F faces: the triangle T in the plane z = 0.5 and its mirror image R in z = -0.5 on both sides of a slab boundary,
    a copy of T in the last slab, and small far-away filler faces.  Queries in the plane z = 0 see T and R at exactly
    the same float64 (and fp32) distance."""
    t = np.array([[-0.3, -0.2, 0.5], [0.4, -0.1, 0.5], [0.0, 0.4, 0.5]], np.float32)
    n_fill = F   # more than needed
    centre = rng.normal(size=(n_fill, 3))
    centre = 40 * centre / np.linalg.norm(centre, axis=1, keepdims=True)
    fill = (centre[:, None] + rng.uniform(-0.5, 0.5, (n_fill, 3, 3))).astype(np.float32)
    L = _slab_len(F)
    b = (F // L) * L if F > L else F // 2
    if b == F:
        b -= L
    if F == 1:
        slots = {0: 'T'}
    elif F == 2:
        slots = {0: 'R', 1: 'T'}
    else:
        slots = {b - 1: 'R', b: 'T', F - 1: 'D'}
    tris, k = [None] * F, 0
    for i in range(F):
        if i in slots:
            tris[i] = t * np.array([1, 1, -1], np.float32) if slots[i] == 'R' else t
        else:
            tris[i] = fill[k]
            k += 1
    v = np.stack(tris).reshape(-1, 3).astype(np.float32)
    faces = np.arange(3 * F, dtype=np.int32).reshape(F, 3)
    return v, faces, min(slots)


@pytest.mark.parametrize('F', [1, 2, 127, 128, 129, 4095, 4096, 4097, 131073])
def test_slab_ties_take_the_lowest_face(F):
    rng = np.random.RandomState(F)
    v, f, want = _slab_mesh(F, rng)
    r = rng.uniform(0, 1, (2000, 2))
    r[r.sum(1) > 1] = 1 - r[r.sum(1) > 1]
    t = v[3 * want:3 * want + 3].astype(np.float64)
    q = t[0] + r[:, :1] * (t[1] - t[0]) + r[:, 1:] * (t[2] - t[0])
    q = np.concatenate([q, rng.uniform(-2, 2, (500, 3)) * [1, 1, 0]])
    q[:, 2] = 0.0
    q = q.astype(np.float32)
    d, face, w, cp, du, fu = _both(v, f, q)
    assert (face == want).all() and (fu == want).all(), np.unique(face)
    _check_against_reference(v, f, q, d, face, w, cp)


def test_duplicated_faces_across_slabs_of_a_200k_face_torus():
    from test_gpu_mesh_clean import _mc
    v, f = _mc('torus', 300)
    assert len(f) >= 200000
    L = _slab_len(len(f) + 2)
    j, b = 17, 5 * L                                 # face j in slab 0; face b - 1 ends slab 4
    f2 = np.concatenate([f[:b], f[b - 1:b], f[b:], f[j:j + 1]]).astype(np.int32)   # copies at b and at the end
    assert _slab_len(len(f2)) == L and f2[b].tolist() == f2[b - 1].tolist() and f2[-1].tolist() == f2[j].tolist()
    rng = np.random.RandomState(0)
    a_, b_, c_ = (v[f2[[j, b - 1], k]].astype(np.float64) for k in range(3))
    n = np.cross(b_ - a_, c_ - a_)
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    ctr = (a_ + b_ + c_) / 3
    h = np.array([0.0, 1e-4, -1e-4, 1e-3, -1e-3])
    q_target = (ctr[:, None] + h[None, :, None] * n[:, None]).reshape(-1, 3)
    q = np.concatenate([q_target, _chunk_queries(v, f, 3000, 1)]).astype(np.float32)
    d, face, w, cp, du, fu = _both(v, f2, q)
    assert face[:5].tolist() == [j] * 5 and face[5:10].tolist() == [b - 1] * 5
    assert fu[:10].tolist() == face[:10].tolist()
    _check_against_reference(v, f2, q, d, face, w, cp)


# ------------------------------------------------------------------ sliver boundary
def test_faces_at_the_sliver_threshold():
    """|n|^2 against 2^-10 * longest edge^4: faces just above (fp32 path) and just below (always float64), queries near
    their planes, on them and far out along them"""
    faces, verts = [], []
    rng = np.random.RandomState(5)
    rot = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    for i, hh in enumerate([2.0 ** -5 * (1 + 2.0 ** -20), 2.0 ** -5 * (1 - 2.0 ** -20), 2.0 ** -5 * 1.01,
                            2.0 ** -5 * 0.99]):
        tri = np.array([[0, 0, 0], [1, 0, 0], [0.5, hh, 0]]) + [0, 0, 0.01 * i]
        if i >= 2:
            tri = tri @ rot.T
        verts.append(tri)
        faces.append(np.arange(3) + 3 * i)
    v = np.concatenate(verts).astype(np.float32)
    f = np.array(faces, np.int32)
    q = np.concatenate([
        rng.uniform(-0.2, 1.2, (600, 3)) * [1, 0.05, 0.05],
        rng.uniform(-100, 100, (300, 3)) * [1, 1e-3, 1e-4],
        rng.uniform(0, 1, (300, 3)) * [1, 0.03, 0] + [0, 0, 0.005],
        (rng.uniform(-0.2, 1.2, (300, 3)) * [1, 0.05, 0.05]) @ rot.T,
        rng.normal(size=(100, 3)) * 50]).astype(np.float32)
    d, face, w, cp, du, fu = _both(v, f, q)
    _check_against_reference(v, f, q, d, face, w, cp)
    for k in (-40, 33):
        dk, facek = ops.mesh_signed_distance(cu(_scaled(v, k)), cu(f), cu(_scaled(q, k)), True)
        assert np.array_equal(facek.cpu().numpy(), face)
        _assert_scaled(np.abs(dk.cpu().numpy()), np.abs(d), k, 'distance')


# ------------------------------------------------------------------ solid voxelisation
def _inside_cases():
    out = dict(ic.closed_cases())
    v, f = ic.icosphere(level=3)
    out['open_sphere'] = (v, f[1:])
    return out


@pytest.mark.parametrize('name', ['sphere', 'torus', 'abc0', 'abc1', 'abc2', 'box', 'octahedron', 'open_sphere'])
def test_inside_equals_oracle_bit_for_bit_at_res256(name):
    v, f = _inside_cases()[name]
    got = ops.mesh_inside_grid(cu(v), cu(f), 256).cpu().numpy().astype(np.uint8)
    want, _ = io.inside_grid(v, f, 256)
    assert np.array_equal(got, want), int((got != want).sum())


def _flags_from_crossings(v, f, res, got):
    """compare the kernel's flags with oracle crossings() turned into flags on the device, a slab of x at a time"""
    col, zh = io.crossings(v, f, res)
    c = torch.from_numpy(io.centres(res).astype(np.float64)).to(DEV)
    col, zh = torch.from_numpy(col).to(DEV), torch.from_numpy(zh).to(DEV)
    k0 = torch.searchsorted(c, zh, right=False)              # voxel centres below the crossing
    slab = 64
    for x0 in range(0, res, slab):
        lo, hi = x0 * res, min(res, x0 + slab) * res
        m = (col >= lo) & (col < hi)
        cnt = torch.zeros((hi - lo, res + 1), dtype=torch.int32, device=DEV)
        cnt.index_put_((col[m] - lo, k0[m]), torch.ones_like(k0[m], dtype=torch.int32), accumulate=True)
        above = cnt.flip(1).cumsum(1).flip(1)[:, 1:]        # crossings with k0 > k flip voxel k
        want = (above % 2).bool().view(-1, res, res)
        assert torch.equal(got[x0:x0 + slab], want), (x0, int((got[x0:x0 + slab] != want).sum()))
    return int(col.numel())


@pytest.mark.parametrize('res', [512, 993, 1024])
@pytest.mark.parametrize('name', ['sphere', 'torus', 'abc0', 'abc1', 'octahedron', 'open_sphere'])
def test_inside_at_high_resolution(name, res):
    v, f = _inside_cases()[name]
    got = ops.mesh_inside_grid(cu(v), cu(f), res)
    n = _flags_from_crossings(v, f, res, got)
    assert n > 0 and (name == 'open_sphere' or int(got.sum()) > 0)


def _range_edge_meshes():
    """a closed octahedron whose equator spans the whole grid with |x|, |y| = 16 - 2^-20 (edge functions within a factor
    2 of 2^63), and closed tetrahedra smaller than the 2^-26 fixed-point step and a few steps wide, at a column centre"""
    m = np.float32(16 - 2.0 ** -20)
    assert float(m) == 16 - 2.0 ** -20
    big = np.array([[m, 0, 0.1], [-m, 0, 0.1], [0, m, 0.1], [0, -m, 0.1], [0, 0, 0.9], [0, 0, -0.7]], np.float32)
    fo = ic.octahedron()[1]
    res = 256
    cx = float(io.centres(res)[128])   # 2^-8: fp32 resolves 2^-31 there, the fixed point 2^-26
    meshes = {'octahedron_16': (big, fo)}
    for name, s in (('tetra_sub_step', 2.0 ** -28), ('tetra_few_steps', 3 * 2.0 ** -26)):
        t = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0.3, 0.3, 1]]) * s + [cx - s / 3, cx - s / 3, 0.2]
        tf = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int32)
        meshes[name] = (t.astype(np.float32), tf)
    both = [meshes['octahedron_16'], meshes['tetra_few_steps']]
    meshes['octahedron_16_and_tetra'] = (np.concatenate([both[0][0], both[1][0]]),
                                         np.concatenate([both[0][1], both[1][1] + len(both[0][0])]).astype(np.int32))
    return meshes


@pytest.mark.parametrize('name', ['octahedron_16', 'tetra_sub_step', 'tetra_few_steps', 'octahedron_16_and_tetra'])
def test_inside_at_the_coordinate_limits(name):
    v, f = _range_edge_meshes()[name]
    for res in (256, 1024):
        got = ops.mesh_inside_grid(cu(v), cu(f), res)
        if res == 256:
            want, cross = io.inside_grid(v, f, res)
            assert np.array_equal(got.cpu().numpy().astype(np.uint8), want) and (cross % 2 == 0).all()
        else:
            _flags_from_crossings(v, f, res, got)
    if name == 'octahedron_16':
        assert bool(got[:, :, 600].all()) and not bool(got[:, :, -1].any())


@pytest.mark.parametrize('name', ['abc0', 'abc2'])
def test_inside_agrees_with_winding_number_parity_at_res256(name):
    res = 256
    v, f = ic.closed_cases()[name]
    inside = ops.mesh_inside_grid(cu(v), cu(f), res).reshape(-1)
    q = ops.query_points(torch.arange(res ** 3, dtype=torch.int32, device=DEV), res)
    d, w = ops.mesh_signed_distance(cu(v), cu(f), q, return_winding=True)
    far = d.abs() > 1e-5
    wr = torch.round(w)
    assert float((w - wr).abs()[far].max()) < 1e-2
    assert int(((wr.remainder(2) == 1) != inside)[far].sum()) == 0
    simple = far & ((wr == 0) | (wr == 1))
    assert int(((d > 0) != inside)[simple].sum()) == 0
    assert int(simple.sum()) > 0.99 * res ** 3
