"""GPU: every training-step primitive of csrc/train_ops.cu other than the GEMMs, per element against the float64 bounds of
tests/train_prims_bound.py, at the shapes training uses and where the launch geometry changes: rows B*n for
B in {1, 2, 32, 1024} and n in {300, 1000}, the FC BatchNorms' M = B, M = 1 and M < 8, the 64-row floor / in-between /
4096-row cap of col_reduce_grid, channel counts that are not multiples of 32 or 128 (the tx choice of rowwise_grid).
Columns mix |mean| / std from 0 to 10^4, constant columns, scales 2^-30 .. 2^17, zero and negative gamma.  Each case
prints its worst excess (error / bound, <= 1 passes) and where it occurs.

Peak device memory is about 12 GB, counted from the tensor sizes of the fused BatchNorm + max-pool case on
z = [1024 * 1000, 1024]: 4.2 GB for z, 4.2 GB for dz, and a few float64 [1024000, 64] temporaries of the reference, which
is built 64 columns at a time.  The file runs in about 20 s on an H100 80GB HBM3 (700 W)."""
import numpy as np
import pytest
import torch

import train_prims_bound as tb
from points2surf_b200.ops import P2SError, _ptr, _stream
from points2surf_b200.train_ops import CudaPrims

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
EPS = 1e-5
MOM = 0.1


@pytest.fixture(scope='module')
def prims():
    return CudaPrims()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def worst(got, exact, bound):
    """-> (max |got - exact| / bound, index of the worst element); a non-finite got counts as infinite."""
    got = got.double()
    exact, bound = exact.double().to(got.device), bound.double().to(got.device)
    err = (got - exact).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    r = torch.where(torch.isfinite(got), r, torch.full_like(r, float('inf')))
    if r.numel() == 0:
        return 0.0, ()
    i = int(torch.argmax(r))
    return float(r.reshape(-1)[i]), tuple(int(v) for v in np.unravel_index(i, tuple(r.shape)))


def report(case, res):
    print(case + ': ' + ', '.join('%s %.3g at %s' % (k, v[0], v[1]) for k, v in res.items()))
    bad = {k: v for k, v in res.items() if not v[0] <= 1.0}
    assert not bad, (case, bad)


def columns(M, C, seed):
    """fp32 [M, C]: column c has mean ratio(c) * scale(c) and std scale(c); ratio cycles over 0, 1, 10, 100, 10^3, 10^4,
    -10^3; scale spans 2^-30 .. 2^17; column C // 2 is constant (var = 0)."""
    z = torch.randn(M, C, device=DEV, generator=_gen(seed))
    ratios = torch.tensor([0.0, 1.0, 10.0, 100.0, 1e3, 1e4, -1e3], device=DEV)[torch.arange(C, device=DEV) % 7]
    scale = 2.0 ** torch.linspace(-30, 17, C, device=DEV).round()
    z.add_(ratios).mul_(scale)
    if C > 1:
        z[:, C // 2] = 1000.3
    return z


def params(C, seed):
    g = _gen(seed)
    gamma = torch.randn(C, device=DEV, generator=g)
    gamma[::7] = 0.0
    beta = torch.randn(C, device=DEV, generator=g)
    return gamma, beta


def stats_blocked(z, cb=64):
    """col_stats_exact column block by column block (the float64 copy of a block only)."""
    parts = [tb.col_stats_exact(z[:, c0:c0 + cb], EPS) for c0 in range(0, z.shape[1], cb)]
    return {k: (torch.cat([p[k] for p in parts]) if k != 'M' else z.shape[0]) for k in parts[0]}


INV_EPS = float(np.float32(1.0 / np.sqrt(np.float64(np.float32(EPS)))))


def check_stats(case, st, mean, invstd, const_col=None, extra=None):
    res = {'mean': worst(mean, st['mean'], tb.mean_bound(st)),
           'invstd': worst(invstd, st['invstd'], st['invstd'] * tb.invstd_rel_bound(st, EPS))}
    res.update(extra or {})
    report(case, res)
    if const_col is not None:
        assert float(invstd[const_col]) == INV_EPS


# (M, C): B*n rows, the FC BatchNorms' M = B, M = 1, M < 8, and the three col_reduce_grid regimes (132 SMs: the 64-row
# floor up to M = 528 * 64 for C <= 64, rows in between, the 4096 cap once M > 33 * 4096 at C = 1024)
BN_SHAPES = [(300, 64), (1000, 128), (600, 3), (2000, 33), (9600, 256), (32000, 512), (64000, 4), (307200, 64),
             (1024000, 128), (300000, 64), (140000, 1024), (1, 64), (2, 1024), (5, 4), (7, 33), (32, 512), (1024, 256),
             (1024, 1024)]


@pytest.mark.parametrize('M,C', BN_SHAPES)
def test_batchnorm_forward_backward_bounds(prims, M, C):
    z = columns(M, C, seed=M + C)
    gamma, beta = params(C, 1)
    st = stats_blocked(z)
    rm = torch.randn(C, device=DEV, generator=_gen(2))
    rv = torch.rand(C, device=DEV, generator=_gen(3)) + 0.5
    rm2, rv2, brm, brv = tb.running_exact_and_bound(st, rm, rv, MOM)
    y, mean, invstd = prims.bn_forward(z, gamma, beta, False, rm, rv, EPS, MOM)
    ye, by = tb.bn_apply_own(z, mean, invstd, gamma, beta, False)
    yt, byt = tb.bn_apply_true(z, st, gamma, beta, False, EPS)
    check_stats('bn M=%d C=%d' % (M, C), st, mean, invstd, C // 2 if C > 1 else None,
                {'running_mean': worst(rm, rm2, brm), 'running_var': worst(rv, rv2, brv),
                 'y(own stats)': worst(y, ye, by), 'y(f64 stats)': worst(y, yt, byt)})
    assert torch.equal(y, tb.bn_apply_emulate(z, mean, invstd, gamma, beta, False))
    del ye, by, yt, byt
    yr, mean_r, invstd_r = prims.bn_forward(z, gamma, beta, True, None, None, EPS, MOM)
    assert torch.equal(yr, tb.bn_apply_emulate(z, mean_r, invstd_r, gamma, beta, True))
    dy = torch.randn(M, C, device=DEV, generator=_gen(4))
    for relu in (False, True):
        mask = (yr > 0).float() if relu else None
        dz, dg, db = prims.bn_backward(dy, z, yr if relu else None, mean_r, invstd_r, gamma)
        g = dy * mask if relu else dy
        dze, dge, dbe, bdz, bdg, bdb = tb.bn_backward_exact(g, z, mean_r, invstd_r, gamma)
        report('bn backward M=%d C=%d relu=%d' % (M, C, relu),
               {'dz': worst(dz, dze, bdz), 'dgamma': worst(dg, dge, bdg), 'dbeta': worst(db, dbe, bdb)})
        del dze, bdz
    S = dy.double().sum(0)
    report('col_sum M=%d C=%d' % (M, C),
           {'sum': worst(prims.col_sum(dy), S, tb.U * S.abs() + tb.gamma64(M + 1) * dy.double().abs().sum(0))})


@pytest.mark.parametrize('k', [0, 4, 8, 12])
def test_batchnorm_output_is_shift_invariant(prims, k):
    # z on a grid of multiples of 2^-10 in (-4, 4): z + 2^k is exact in fp32 for k <= 12, so y(z + t) and y(z) have the
    # same float64 value and may differ only by the two bounds
    M, C = 70000, 64
    z = (torch.randint(-4095, 4096, (M, C), device=DEV, generator=_gen(5)).float() * 2.0 ** -10)
    z[:, 1] = 0.75
    zt = z + 2.0 ** k
    assert torch.equal(zt - 2.0 ** k, z)
    gamma, beta = params(C, 6)
    y0, _, _ = prims.bn_forward(z, gamma, beta, False)
    yk, mk, ik = prims.bn_forward(zt, gamma, beta, False)
    st0, stk = tb.col_stats_exact(z, EPS), tb.col_stats_exact(zt, EPS)
    ye, b0 = tb.bn_apply_true(z, st0, gamma, beta, False, EPS)
    _, bk = tb.bn_apply_true(zt, stk, gamma, beta, False, EPS)
    check_stats('shift 2^%d' % k, stk, mk, ik, 1,
                {'y(z + t) vs y(z)': worst(yk, y0.double(), b0 + bk), 'y(z + t)': worst(yk, ye, bk)})


def _first_max(v, dim):
    """(max, first index of it) along dim, NaN propagating (the first NaN wins)."""
    n = v.shape[dim]
    idx = torch.arange(n, device=v.device).reshape([-1 if d == dim else 1 for d in range(v.dim())])
    nan = torch.isnan(v)
    has_nan = nan.any(dim)
    mx = torch.where(nan, torch.full_like(v, -float('inf')), v).amax(dim)
    first_nan = torch.where(nan, idx, n).amin(dim)
    first_max = torch.where(v == mx.unsqueeze(dim), idx, n).amin(dim)
    out = torch.where(has_nan, torch.full_like(mx, float('nan')), mx)
    return out, torch.where(has_nan, first_nan, first_max)


# (B, npts, C, relu): the conv3 shapes of training, odd channel counts, npts = 1, and z = [1024 * 1000, 1024]
FUSED = [(1, 300, 1024, True), (2, 1000, 64, False), (32, 300, 33, True), (32, 1000, 128, False), (1024, 300, 256, True),
         (3, 1, 4, True), (5, 7, 3, False), (1024, 1000, 1024, True)]


@pytest.mark.parametrize('B,n,C,relu', FUSED)
def test_fused_batchnorm_maxpool_bounds(prims, B, n, C, relu):
    M = B * n
    z = columns(M, C, seed=B + n + C)
    gamma, beta = params(C, 7)
    out, arg, mean, invstd = prims.bn_maxpool_forward(z, B, n, gamma, beta, relu)
    st = stats_blocked(z)
    check_stats('fused B=%d n=%d C=%d' % (B, n, C), st, mean, invstd, C // 2 if C > 1 else None)
    del st
    dout = torch.randn(B, C, device=DEV, generator=_gen(8))
    dz, dg, db = prims.bn_maxpool_backward(dout, arg, out, z, mean, invstd, gamma, relu, B, n)
    g = dout * (out > 0).float() if relu else dout
    res = {}
    cb = 64
    for c0 in range(0, C, cb):
        sl = slice(c0, c0 + cb)
        zb = z[:, sl]
        y = tb.bn_apply_emulate(zb, mean[sl], invstd[sl], gamma[sl], beta[sl], relu)
        o, a = _first_max(y.view(B, n, -1), 1)
        assert torch.equal(out[:, sl], o) and torch.equal(arg[:, sl].long(), a), 'max-pool at columns %d..' % c0
        del y
        gd = torch.zeros(B, n, zb.shape[1], device=DEV).scatter_(1, a.unsqueeze(1), g[:, sl].unsqueeze(1))
        dze, dge, dbe, bdz, bdg, bdb = tb.bn_backward_exact(gd.view(M, -1), zb, mean[sl], invstd[sl], gamma[sl])
        for k, (got, ex, bd) in {'dz': (dz[:, sl], dze, bdz), 'dgamma': (dg[sl], dge, bdg), 'dbeta': (db[sl], dbe, bdb)}.items():
            r, i = worst(got, ex, bd)
            if k not in res or r > res[k][0]:
                res[k] = (r, (i[0], i[-1] + c0))
        del gd, dze, bdz
    report('fused backward B=%d n=%d C=%d relu=%d' % (B, n, C, relu), res)
    if M * C <= 1 << 26:       # the unfused pair gives the same bits (same fmaf, same first-maximum rule)
        y = prims.bn_apply(z, mean, invstd, gamma, beta, relu)
        o2, a2 = prims.maxpool_fwd(y, B, n)
        assert torch.equal(out, o2) and torch.equal(arg, a2)


def _fused_fwd_raw(prims, z, B, n, relu):
    """bn_maxpool_fwd with mean 0, invstd 1, gamma 1, beta 0: y = fmaf(1, z - 0, 0) = z."""
    C_ = z.shape[1]
    one, zero = torch.ones(C_, device=DEV), torch.zeros(C_, device=DEV)
    out = torch.empty(B, C_, device=DEV)
    arg = torch.empty(B, C_, dtype=torch.int32, device=DEV)
    rc = prims.lib.p2s_op_bn_maxpool_fwd(_ptr(z), B, n, C_, _ptr(zero), _ptr(one), _ptr(one), _ptr(zero), 1 if relu else 0,
                                         _ptr(out), _ptr(arg), _stream())
    assert rc == 0
    return out, arg


@pytest.mark.parametrize('n', [1, 2, 300])
def test_maxpool_ties_infinities_and_nan(prims, n):
    B, C_ = 4, 40
    y = torch.randn(B, n, C_, device=DEV, generator=_gen(9)).round()     # many ties
    y[0, :, 0] = -float('inf')
    y[1, :, 1] = 2.0
    y[2, n // 2, 2] = float('nan')                                       # NaN in the middle, at the end, at row 0
    y[2, n - 1, 3] = float('nan')
    y[3, 0, 4] = float('nan')
    y[3, :, 5] = float('nan')
    y[1, n - 1, 6] = float('inf')
    y = y.reshape(B * n, C_)
    o_ref, a_ref = _first_max(y.view(B, n, C_), 1)
    o1, a1 = prims.maxpool_fwd(y, B, n)
    o2, a2 = _fused_fwd_raw(prims, y, B, n, False)
    for o, a in ((o1, a1), (o2, a2)):
        assert torch.equal(torch.isnan(o), torch.isnan(o_ref))
        assert torch.equal(torch.nan_to_num(o), torch.nan_to_num(o_ref))
        assert torch.equal(a.long(), a_ref)
    tv = torch.max(y.view(B, n, C_), 1)[0]                                # NaN propagates like torch.max
    assert torch.equal(torch.isnan(tv), torch.isnan(o1))
    # with the ReLU both paths map NaN to 0 (fmaxf) before the max: they still agree bit for bit
    o3, a3 = prims.maxpool_fwd(torch.clamp_min(y.nan_to_num(0.0, posinf=float('inf'), neginf=-float('inf')), 0.0), B, n)
    o4, a4 = _fused_fwd_raw(prims, y, B, n, True)
    assert torch.equal(o3, o4) and torch.equal(a3, a4)


def test_batch_limit_of_the_grid(prims):
    n, C_ = 2, 3
    for B, ok in ((65535, True), (65536, False)):
        z = torch.randn(B * n, C_, device=DEV, generator=_gen(10))
        gamma, beta = torch.ones(C_, device=DEV), torch.zeros(C_, device=DEV)
        dout = torch.randn(B, C_, device=DEV, generator=_gen(11))
        arg = torch.zeros(B, C_, dtype=torch.int32, device=DEV)
        calls = [lambda: prims.maxpool_bwd(dout, arg, n),
                 lambda: prims.bn_maxpool_forward(z, B, n, gamma, beta, True),
                 lambda: prims.bn_maxpool_backward(dout, arg, dout, z, torch.zeros(C_, device=DEV),
                                                   torch.ones(C_, device=DEV), gamma, True, B, n)]
        for f in calls:
            if ok:
                f()
            else:
                with pytest.raises(P2SError):
                    f()
    zb = z[:65535 * n]
    out, arg, mean, invstd = prims.bn_maxpool_forward(zb, 65535, n, gamma, beta, False)
    o, a = _first_max(tb.bn_apply_emulate(zb, mean, invstd, gamma, beta, False).view(65535, n, C_), 1)
    assert torch.equal(out, o) and torch.equal(arg.long(), a)


def _loss_inputs(B, seed):
    g = _gen(seed)
    pred = torch.randn(B, 2, device=DEV, generator=g) * 3
    tmag = torch.rand(B, device=DEV, generator=g) * 0.1
    rad = torch.rand(B, device=DEV, generator=g) * 0.3 + 0.05
    tsign = (torch.rand(B, device=DEV, generator=g) < 0.5).float()
    special = torch.tensor([0.0, 80.0, -80.0, 1e4, -1e4, 20.0, -20.0, 1e-8], device=DEV)
    k = min(B, len(special))
    pred[:k, 0] = special[:k]
    pred[-k:, 1] = special[:k]
    tmag[B // 2:B // 2 + min(B - B // 2, 4)] = 0.0
    rad[:min(B, 3)] = torch.tensor([1e-30, 1e-6, 1e-3], device=DEV)[:min(B, 3)]
    return pred, tmag, rad, tsign


@pytest.mark.parametrize('B', [1, 255, 256, 257, 1024, 100000])
def test_losses_per_element(prims, B):
    pred, tmag, rad, tsign = _loss_inputs(B, 12 + B)
    for fixed in (False, True):
        L, dp = prims.loss(pred, tmag, rad, tsign, 1.0, 0.7, fixed_radius=fixed)
        Le, bL, dpe, bdp = tb.loss_exact(pred, tmag, rad, tsign, 1.0, 0.7, fixed)
        Ld, dpd = prims.loss_distance(pred[:, :1].contiguous(), tmag, rad, 0.9, fixed_radius=fixed)
        Lde, bLd, dpde, bdpd = tb.loss_distance_exact(pred[:, :1], tmag, rad, 0.9, fixed)
        report('loss B=%d fixed_radius=%d' % (B, fixed),
               {'loss': worst(L, Le, bL), 'dpred': worst(dp, dpe, bdp),
                'loss_distance': worst(Ld, Lde, bLd), 'dpred_distance': worst(dpd, dpde, bdpd)})
        if B == 1:          # B = 1: the loss is the per-query term itself
            assert worst(L, Le, bL)[0] <= 1


def test_quaternion_forward_backward_bounds(prims):
    g = _gen(13)
    q4 = torch.cat([torch.randn(4096, 4, device=DEV, generator=g) * 0.3,                       # general
                    torch.randn(4096, 4, device=DEV, generator=g) * 1e-4,                      # near the identity
                    torch.tensor([[-1.0, 0, 0, 0]], device=DEV) + torch.randn(4096, 4, device=DEV, generator=g) * 1e-3])
    dR = torch.randn(q4.shape[0], 9, device=DEV, generator=g)
    R = prims.quat_to_rot(q4)
    dq = prims.quat_to_rot_bwd(q4, dR)
    Re, bR = tb.quat_to_rot_exact(q4)
    dqe, bdq = tb.quat_to_rot_bwd_exact(q4, dR)
    report('quaternion', {'R': worst(R.reshape(-1, 9), Re, bR), 'dq': worst(dq, dqe, bdq)})
    # q = 0: the same non-finite pattern as torch autograd on utils.batch_quat_to_rotmat
    from oracle.p2s_oracle import quat_to_rotmat
    qz = torch.tensor([[-1.0, 0, 0, 0], [-1.0, 0, 0, 0]])
    dRz = torch.randn(2, 9, generator=torch.Generator().manual_seed(0))
    qt = qz.clone().requires_grad_(True)
    with torch.enable_grad():
        Rt = quat_to_rotmat(qt + torch.tensor([1.0, 0, 0, 0]))
        Rt.backward(dRz.view(2, 3, 3))
    Rk = prims.quat_to_rot(qz.to(DEV)).cpu().reshape(2, 9)
    dqk = prims.quat_to_rot_bwd(qz.to(DEV), dRz.to(DEV)).cpu()
    for a, b in ((Rk, Rt.detach().reshape(2, 9)), (dqk, qt.grad)):
        assert torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(torch.isinf(a), torch.isinf(b))


def test_elementwise_ops_bit_exact(prims):
    g = _gen(14)
    n = 1000003
    par, grad = torch.randn(n, device=DEV, generator=g), torch.randn(n, device=DEV, generator=g)
    buf = torch.zeros(n, device=DEV)
    lr, mom = torch.tensor(0.0123, device=DEV), torch.tensor(0.9, device=DEV)
    p0 = par.clone()
    prims.sgd_(par, grad, buf, float(lr), float(mom), True)
    assert torch.equal(buf, grad) and torch.equal(par, tb.fma32(-lr.expand(n), grad, p0))
    p1, b1 = par.clone(), buf.clone()
    grad2 = torch.randn(n, device=DEV, generator=g)
    prims.sgd_(par, grad2, buf, float(lr), float(mom), False)
    b2 = tb.fma32(mom.expand(n), b1, grad2)
    assert torch.equal(buf, b2) and torch.equal(par, tb.fma32(-lr.expand(n), b2, p1))
    y0, x = torch.randn(n, device=DEV, generator=g), torch.randn(n, device=DEV, generator=g)
    y = y0.clone()
    prims.axpy_(y, x, 0.37)
    assert torch.equal(y, tb.fma32(torch.tensor(0.37, device=DEV).expand(n), x, y0))
    xr, v = torch.randn(1025, 33, device=DEV, generator=g), torch.randn(33, device=DEV, generator=g)
    assert torch.equal(prims.add_row_(xr.clone(), v), xr + v)
    pts, q = torch.randn(7, 1001, 3, device=DEV, generator=g), torch.randn(7, 3, device=DEV, generator=g)
    assert torch.equal(prims.center(pts, q), pts - q.unsqueeze(1))
    for shape in ((33, 1000), (1, 1), (7, 129, 65)):
        t = torch.randn(*shape, device=DEV, generator=g)
        assert torch.equal(prims.transpose(t), t.transpose(-1, -2))


@pytest.mark.parametrize('M,C', [(1, 3), (2000, 33), (307200, 64)])
def test_raw_column_sums_of_the_c_abi(prims, M, C):
    # p2s_op_col_stats keeps its unshifted sums (sum x, sum x^2), f64 from the first term; p2s_op_bn_finalize on them
    # gives the same mean as p2s_op_bn_stats within the mean bound (its variance cancels, which is why BatchNorm does
    # not use it)
    z = columns(M, C, seed=20 + M)
    s = torch.empty(2, C, dtype=torch.float64, device=DEV)
    assert prims.lib.p2s_op_col_stats(_ptr(z), M, C, _ptr(s[0]), _ptr(s[1]), _stream()) == 0
    zd = z.double()
    S1, S2 = zd.sum(0), (zd * zd).sum(0)
    b1, b2 = tb.gamma64(M + 8) * zd.abs().sum(0), tb.gamma64(M + 8) * S2
    mean, inv = torch.empty(C, device=DEV), torch.empty(C, device=DEV)
    assert prims.lib.p2s_op_bn_finalize(_ptr(s[0]), _ptr(s[1]), M, C, EPS, MOM, _ptr(mean), _ptr(inv), None, None,
                                        _stream()) == 0
    st = tb.col_stats_exact(z, EPS)
    report('col_stats M=%d C=%d' % (M, C), {'sum x': worst(s[0], S1, b1), 'sum x^2': worst(s[1], S2, b2),
                                            'mean': worst(mean, st['mean'], tb.mean_bound(st))})
