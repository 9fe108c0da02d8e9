"""CPU: the float64 bounds of tests/train_prims_bound.py hold for emulations of the intended fp32 arithmetic of the
training-step primitives, are tight enough to catch a dropped term, and the fp32 FMA emulation rounds once.  The
BatchNorm statistics case is the regression test of the shifted f64 column sums: the previous reduction order (fp32
partials of E[z] and E[z^2] over up to 512 rows per thread) breaks the invstd bound once |mean| / std reaches 100; the
shipped order meets it up to 10^4."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import train_prims_bound as tb

EPS = 1e-5


def _f32(x):
    return torch.as_tensor(np.asarray(x, np.float32))


def test_fma32_rounds_once():
    rng = np.random.RandomState(0)
    a = rng.randn(4000).astype(np.float32)
    b = rng.randn(4000).astype(np.float32)
    c = (rng.randn(4000) * 2.0 ** rng.randint(-40, 20, 4000)).astype(np.float32)
    # products that sit exactly on an fp32 midpoint, plus a tiny c: a double-rounding emulation gets these wrong
    a[:1000] = np.float32(1 + 2.0 ** -12)
    b[:1000] = np.float32(1 + 2.0 ** -12)                  # a b = 1 + 2^-11 + 2^-24: midpoint between two fp32
    c[:500] = np.float32(2.0 ** -60)
    c[500:1000] = np.float32(-(2.0 ** -60))
    r = tb.fma32(_f32(a), _f32(b), _f32(c)).numpy()
    for i in range(len(a)):
        ex = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        ri = r[i]
        lo, hi = np.nextafter(ri, np.float32(-np.inf)), np.nextafter(ri, np.float32(np.inf))
        e, el, eh = abs(ex - Fraction(float(ri))), abs(ex - Fraction(float(lo))), abs(ex - Fraction(float(hi)))
        assert e <= el and e <= eh, i
        if e == el or e == eh:
            assert int(np.array(ri).view(np.int32)) % 2 == 0, i


@pytest.mark.parametrize('ratio', [0.0, 1.0, 10.0, 100.0, 1e3, 1e4])
@pytest.mark.parametrize('M,rpb', [(1024, 64), (65536, 4096), (3000, 569)])
def test_batchnorm_statistics_order(M, rpb, ratio):
    z = (ratio + np.random.RandomState(int(ratio) + M).randn(M)).astype(np.float32)
    st = tb.col_stats_exact(_f32(z).reshape(-1, 1), EPS)
    rel = float(tb.invstd_rel_bound(st, EPS)[0])
    mean_b = float(tb.mean_bound(st)[0])
    mean_n, inv_n = tb.col_stats_new_order(z, rpb, EPS)
    inv_e, mean_e = float(st['invstd'][0]), float(st['mean'][0])
    new_ratio = abs(float(inv_n) - inv_e) / (inv_e * rel)
    assert new_ratio <= 1.0, new_ratio
    assert abs(float(mean_n) - mean_e) <= mean_b
    mean_o, inv_o = tb.col_stats_old_order(z, rpb, EPS)
    old_ratio = abs(float(inv_o) - inv_e) / (inv_e * rel)
    print('M %d rpb %d mean/std %g: invstd excess shipped %.3g, previous order %.3g' % (M, rpb, ratio, new_ratio, old_ratio))
    if ratio >= 100:
        assert old_ratio > 1.0, old_ratio


def test_col_reduce_grid_regimes():
    # the three regimes the GPU tests exercise (132 SMs): the 64-row floor, in between, the 4096-row cap
    assert tb.col_reduce_grid(1000, 64) == 64
    assert 64 < tb.col_reduce_grid(300000, 64) < 4096
    assert tb.col_reduce_grid(1024 * 1000, 1024) == 4096
    assert tb.col_reduce_grid(70000, 128) == 266


def _stats_cols(M, C, seed):
    g = torch.Generator().manual_seed(seed)
    ratios = torch.tensor([0.0, 1.0, 10.0, 100.0, 1e3, 1e4, -1e3, 0.0])[torch.arange(C) % 8]
    scale = 2.0 ** torch.linspace(-30, 17, C).round()
    z = (torch.randn(M, C, generator=g) + ratios) * scale
    z[:, C // 2] = 3.25                                     # a constant column: var = 0, invstd = eps^-1/2
    return z.float()


def _emulate_stats(z):
    means, invs = [], []
    for c in range(z.shape[1]):
        m, i = tb.col_stats_new_order(z[:, c].numpy(), tb.col_reduce_grid(z.shape[0], z.shape[1]), EPS)
        means.append(m)
        invs.append(i)
    return _f32(means), _f32(invs)


@pytest.mark.parametrize('M,C', [(1, 3), (5, 4), (300, 33), (2000, 8)])
def test_bn_forward_bounds_hold_for_the_emulation(M, C):
    z = _stats_cols(M, C, M)
    st = tb.col_stats_exact(z, EPS)
    mean, inv = _emulate_stats(z)
    assert tb.excess(mean, st['mean'], tb.mean_bound(st)) <= 1
    assert tb.excess(inv, st['invstd'], st['invstd'] * tb.invstd_rel_bound(st, EPS)) <= 1
    assert float(inv[C // 2]) == float(np.float32(1 / np.sqrt(np.float64(np.float32(EPS)))))
    g = torch.Generator().manual_seed(1)
    gamma_ = torch.randn(C, generator=g)
    gamma_[0], gamma_[1 % C] = 0.0, -1.5
    beta = torch.randn(C, generator=g)
    for relu in (False, True):
        y = tb.bn_apply_emulate(z, mean, inv, gamma_, beta, relu)
        ye, b = tb.bn_apply_own(z, mean, inv, gamma_, beta, relu)
        assert tb.excess(y, ye, b) <= 1
        yt, bt = tb.bn_apply_true(z, st, gamma_, beta, relu, EPS)
        assert tb.excess(y, yt, bt) <= 1
    rm, rv = torch.randn(C, generator=g), torch.rand(C, generator=g) + 0.5
    rm2, rv2, brm, brv = tb.running_exact_and_bound(st, rm, rv, 0.1)
    m = np.float32(0.1)
    f = M / (M - 1) if M > 1 else 1.0
    var_k = (st['var'] * f).float()
    rm_k = (np.float32(1) - m) * rm + m * mean
    rv_k = (np.float32(1) - m) * rv + m * var_k
    assert tb.excess(rm_k, rm2, brm) <= 1 and tb.excess(rv_k, rv2, brv) <= 1


def _bn_backward_emulate(dy, z, mask, mean, inv, gamma_, fused_fma):
    """bn_backward in the kernel's fp32 arithmetic (f64 sums), with or without the contraction of g - m1 - xh m2."""
    g = dy * mask if mask is not None else dy
    xh = (z - mean) * inv
    M = z.shape[0]
    s1 = g.double().sum(0)
    s2 = (g.double() * xh.double()).sum(0)
    m1, m2 = (s1 / M).float(), (s2 / M).float()
    gi = gamma_ * inv
    if fused_fma:
        r = tb.fma32(-xh, m2.expand_as(xh), (g - m1))
    else:
        r = (g - m1) - xh * m2
    return gi * r, s2.float(), s1.float()


@pytest.mark.parametrize('M,C', [(2, 3), (7, 4), (500, 33), (4000, 8)])
def test_bn_backward_bounds_hold_and_catch_a_dropped_term(M, C):
    z = _stats_cols(M, C, 7 + M)
    mean, inv = _emulate_stats(z)
    g = torch.Generator().manual_seed(2)
    dy = torch.randn(M, C, generator=g)
    gamma_ = torch.randn(C, generator=g)
    beta = torch.randn(C, generator=g)
    y = tb.bn_apply_emulate(z, mean, inv, gamma_, beta, True)
    for mask in (None, (y > 0).float()):
        gm = dy * mask if mask is not None else dy
        dz_e, dg_e, db_e, bdz, bdg, bdb = tb.bn_backward_exact(gm, z, mean, inv, gamma_)
        for fused in (False, True):
            dz, dg, db = _bn_backward_emulate(dy, z, mask, mean, inv, gamma_, fused)
            assert tb.excess(dz, dz_e, bdz) <= 1
            assert tb.excess(dg, dg_e, bdg) <= 1
            assert tb.excess(db, db_e, bdb) <= 1
    # a kernel that forgot the xhat * m2 term would not pass
    xh = (z - mean) * inv
    wrong = (gamma_ * inv) * (dy - (dy.double().sum(0) / M).float())
    dz_e, _, _, bdz, _, _ = tb.bn_backward_exact(dy, z, mean, inv, gamma_)
    if M > 4:
        assert tb.excess(wrong, dz_e, bdz) > 1
    assert xh.shape == z.shape


def test_loss_bounds_hold_for_fp32_arithmetic():
    g = torch.Generator().manual_seed(3)
    B = 2000
    pred = torch.randn(B, 2, generator=g) * 3
    pred[:20, 0] = 0.0
    pred[20:40, 1] = torch.tensor([80.0, -80.0, 1e4, -1e4] * 5)
    pred[40:60, 0] = torch.tensor([80.0, -80.0, 1e4, -1e4] * 5)
    tmag = torch.rand(B, generator=g) * 0.1
    tmag[60:80] = 0.0
    rad = torch.rand(B, generator=g) * 0.3 + 0.05
    rad[80:100] = 1e-30
    tsign = (torch.rand(B, generator=g) < 0.5).float()
    for fixed in (False, True):
        t = tmag if fixed else tmag / rad
        a, b = torch.tanh(pred[:, 0].abs()), torch.tanh(t.abs())
        d = a - b
        invB = np.float32(1) / np.float32(B)
        sg = torch.sign(pred[:, 0])
        dp0 = np.float32(2) * d * invB * (1 - a * a) * sg
        p1 = pred[:, 1]
        l1 = torch.clamp_min(p1, 0) - p1 * tsign + torch.log1p(torch.exp(-p1.abs()))
        dp1 = (1 / (1 + torch.exp(-p1)) - tsign) * invB * np.float32(0.7)
        L = torch.stack([(d * d).double().sum() / B, 0.7 * l1.double().sum() / B])
        Le, bL, dpe, bdp = tb.loss_exact(pred, tmag, rad, tsign, 1.0, 0.7, fixed)
        assert tb.excess(L, Le, bL) <= 1
        assert tb.excess(torch.stack([dp0, dp1], 1), dpe, bdp) <= 1
        ld = torch.tanh(pred[:, 0]) - torch.tanh(t)
        dpd = np.float32(2) * ld * invB * (1 - torch.tanh(pred[:, 0]) ** 2)
        Le, bL, dpe, bdp = tb.loss_distance_exact(pred[:, :1], tmag, rad, 1.0, fixed)
        assert tb.excess((ld * ld).double().sum().reshape(1) / B, Le, bL) <= 1
        assert tb.excess(dpd.reshape(-1, 1), dpe, bdp) <= 1


def _quat_fwd_fp32(q4):
    q = tb.quat_fp32(q4)
    s = 2.0 / (q * q).sum(1, keepdim=True)
    A, _ = tb._A_and_abs(q)
    return torch.eye(3).reshape(1, 9) + A * s


def test_quaternion_bounds_hold_for_fp32_arithmetic():
    g = torch.Generator().manual_seed(4)
    q4 = torch.cat([torch.randn(500, 4, generator=g) * 0.3, torch.randn(100, 4, generator=g) * 1e-4,
                    torch.tensor([[-1.0, 0, 0, 0]]).repeat(100, 1) + torch.randn(100, 4, generator=g) * 1e-3])
    dR = torch.randn(q4.shape[0], 9, generator=g)
    Re, bR = tb.quat_to_rot_exact(q4)
    assert tb.excess(_quat_fwd_fp32(q4), Re, bR) <= 1
    q = q4.clone().requires_grad_(True)
    with torch.enable_grad():
        _quat_fwd_fp32(q).backward(dR)
    dqe, bdq = tb.quat_to_rot_bwd_exact(q4, dR)
    # autograd in fp32 is another fp32 evaluation order of the same formula: it meets the bound too
    assert tb.excess(q.grad, dqe, bdq) <= 1
