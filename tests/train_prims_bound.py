"""Float64 error bounds of the training-step primitives of csrc/train_ops.cu other than the GEMMs (those are held to
oracle/split_gemm.py), and bit-exact emulations of the ones that round only once per element.

Every bound takes the kernel's fp32 inputs, promotes them exactly to float64 as the truth, and is stated per element with
u = 2^-24 (fp32 unit roundoff), u64 = 2^-53, gamma_n = n u / (1 - n u) and gamma64_n the same with u64 (Higham, Accuracy and
Stability of Numerical Algorithms, 2nd ed., eq. 3.5: any summation order, with or without FMA).  `excess(got, exact, bound)`
(split_gemm.excess) is max |got - exact| / bound; <= 1 meets it.

Column statistics (col_reduce_kernel<0> + bn_finalize_kernel), column c of z [M, C], shift z0 = z[0, c]:
  every term d = z - z0 is formed in f64 (exact), d and d^2 are summed in f64 from the first term; the longest fp32 sum the
  implementation admits is L = 0, so the fp32 gamma_L of a blocked fp32 sum becomes gamma64_M.
  * mean:   |mean - mu| <= u |mu| + gamma64_{M+3} (mean|d| + |mu|)          (u |mu|: the mean is stored in fp32)
  * var:    |var_k - var| <= 4 gamma64_{M+3} S2 / M,  S2 = sum d^2  (s1^2 <= M s2, so the cancellation is relative to
            S2 / M = var + (mu - z0)^2: the spread about the shift, not the mean)
  * invstd = fp32(1 / sqrt(var + eps)): relative error <= C_INVSTD u + |dvar| / (2 (var + eps)); C_INVSTD = 2: one u for the
            final rounding to fp32, one u of slack for the f64 sqrt / division / eps conversion (each <= u64).  This does not
            depend on |mu| / sigma.  An fp32 partial sum of E[z^2] (the old kernel) has an error ~ gamma_L (mu / sigma)^2.
  * running mean (1 - m) rm + m mean and running var (1 - m) rv + m var M / (M - 1) (M > 1; var when M == 1), fp32 update:
            <= 3 u ((1 - m)|rm| + m|mu|) + m |dmean| + u |rm'|, and the same with var M/(M-1) and its bound.
bn_apply (y = fmaf(fp32(gamma invstd), fp32(z - mean), beta), ReLU after):
  * bit-exact: equals `fma32` of the same fp32 operands (a single rounding);
  * against the kernel's own (mean, invstd):   3 u |gamma invstd (z - mean)| + u |y|
  * against the float64 statistics: + |gamma| invstd (|dmean| + |z - mu| rel_invstd).  |dmean| carries u |mu|: a mean
    stored in fp32 moves every y by up to u |mu| gamma invstd, which no fp32 BatchNorm avoids.
bn_backward (col_reduce_kernel<1> + bn_bwd_apply_kernel), g = dy (masked by y > 0 with the ReLU), xh = (z - mean) invstd
with the kernel's own mean / invstd, A1 = sum |g|, A2 = sum |g xh|, S1 = sum g, S2 = sum g xh:
  * dbeta  = fp32(s1): u |S1| + gamma64_{M+1} A1
  * dgamma = fp32(s2): u |S2| + 2.1 u A2 + gamma64_{M+2} A2       (2.1 u: the two fp32 roundings of xh)
  * dz = fp32(gamma invstd) (g - m1 - xh m2), m1 = fp32(s1 / M), m2 = fp32(s2 / M):
            |gamma invstd| (8 u T + 2.2 u |xh| A2 / M + 2 gamma64_{M+2} A1 / M),  T = |g| + |S1| / M + |xh| |S2| / M
    (8 u: the roundings of m1, m2, xh, the two subtractions, the product xh m2, gamma invstd and the final product).
  The fused bn_maxpool backward is the same with the sparse g of the max-pool (nonzero only at the arg rows).
loss / loss_distance (one CTA; fp32 per query, f64 block sum).  CUDA math library maximum errors (CUDA C++ Programming
Guide, "Mathematical Functions", single precision, default flags, no fast math): tanhf 2 ulp, expf 2 ulp, log1pf 1 ulp;
x / y and 1 / x are correctly rounded (-prec-div=true).  An ulp of x is <= 2 u |x| for a normal x, so k ulp <= 2 k u |x|;
TINY = 2^-146 covers a subnormal result.  With a = tanhf(|p0|) (signed p for the distance loss), b = tanhf(|t / r|),
d = a - b, F = 1 - a^2:
  * da = 4 u a + TINY, db = 4 u b + (1 - b^2) u |t / r| + TINY (the division), dd = da + db + u |d|
  * per query, magnitude term d^2:  2 |d| dd + dd^2 + u (|d| + dd)^2
  * per query, sign term max(p1, 0) - p1 s + log1p(exp(-|p1|)) (first two exact for s in {0, 1}), e = exp(-|p1|):
            4 u e / (1 + e) + 2 u log1p(e) + u |term| + TINY
  * loss_out = w / B sum: (w / B) sum of the per-query bounds + gamma64_{B+4} |loss|
  * dpred0 = w 2 d (1/B) F sign(p0): |2 w / B| (|F| dd + |d| dF + 5 u |d F|), dF = 2 |a| da + u a^2 + u |F|
  * dpred1 = w (sigmoid(p1) - s) / B:  |w / B| (dsig + 4.1 u |sig - s|), dsig = 4 u sig (1 - sig) + 2.1 u sig + TINY
quat_to_rot / quat_to_rot_bwd, q = fp32(q4 + (1, 0, 0, 0)) (the fp32 quaternion the model forms), s = 2 / |q|^2,
R = I + s A(q), A the quadratic form of utils.batch_quat_to_rotmat; Aabs_ij = sum of |monomials| of A_ij:
  * R_ij: s (gamma_3 Aabs_ij + gamma_7 |A_ij|) + u |R_ij|
  * dq_k = -s^2 q_k GA + s D_k, GA = sum g_ij A_ij, D_k = sum g_ij dA_ij/dq_k (every dA_ij/dq_k is one monomial):
            s^2 |q_k| (gamma_13 |GA| + gamma_11 GAabs) + s (gamma_6 |D_k| + gamma_8 Dabs_k) + u |dq_k|,
            GAabs = sum |g_ij| Aabs_ij, Dabs_k = sum |g_ij| |dA_ij/dq_k|  (|q|^-2 enters through s).
sgd_, axpy_, add_row_, center, transpose: bit-exact against the same fp32 formula (`fma32` where the kernel has fmaf)."""
import math

import numpy as np
import torch

from oracle.split_gemm import excess  # noqa: F401  (re-exported: the one excess() of the bounds)

U = 2.0 ** -24
U64 = 2.0 ** -53
TINY = 2.0 ** -146
C_INVSTD = 2.0
SM_COUNT_H100 = 132


def gamma(n):
    return n * U / (1.0 - n * U)


def gamma64(n):
    return n * U64 / (1.0 - n * U64)


# ---------------------------------------------------------------------------------------------- exact fp32 FMA
def fma32(a, b, c):
    """fp32 fma(a, b, c) with one rounding, bit for bit, for fp32 tensors on any device.  a b is exact in f64; the f64 sum
    is rounded to odd (the sticky bit is kept in the last place when the sum was inexact), after which rounding to fp32 is
    correct: round-to-odd at p >= 2 q + 2 bits followed by round-to-nearest at q bits is round-to-nearest at q bits."""
    p = a.double() * b.double()
    cc = c.double()
    s = p + cc
    bb = s - p
    err = (p - (s - bb)) + (cc - bb)                       # TwoSum: s + err == p + c exactly
    even = (s.view(torch.int64) & 1) == 0
    fix = (err != 0) & even & torch.isfinite(s)
    s = torch.where(fix, torch.nextafter(s, torch.where(err > 0, torch.full_like(s, math.inf), torch.full_like(s, -math.inf))), s)
    return s.float()


# ---------------------------------------------------------------------------------------------- column statistics
def col_stats_exact(z, eps):
    """float64 truth of the column statistics of fp32 z [M, C] -> dict(mean, var, invstd, S2, absd) (float64 [C]);
    S2 = sum (z - z0)^2 and absd = mean |z - z0| are the spread terms of the bound."""
    zd = z.double()
    M = z.shape[0]
    mu = zd.mean(0)
    var = ((zd - mu) ** 2).mean(0)
    d = zd - zd[0]
    return dict(mean=mu, var=var, invstd=1.0 / torch.sqrt(var + float(np.float32(eps))),
                S2=(d * d).sum(0), absd=d.abs().mean(0), M=M)


def mean_bound(st):
    M = st['M']
    return U * st['mean'].abs() + gamma64(M + 3) * (st['absd'] + st['mean'].abs())


def var_bound(st):
    return 4 * gamma64(st['M'] + 3) * st['S2'] / st['M']


def invstd_rel_bound(st, eps):
    return C_INVSTD * U + var_bound(st) / (2 * (st['var'] + float(np.float32(eps))))


def running_exact_and_bound(st, rm, rv, momentum):
    """-> (rm', rv', bound rm', bound rv') in float64 for the fp32 update of bn_finalize_kernel."""
    m = float(np.float32(momentum))
    M = st['M']
    rm, rv = rm.double(), rv.double()
    f = M / (M - 1) if M > 1 else 1.0
    vu = st['var'] * f
    rm2 = (1 - m) * rm + m * st['mean']
    rv2 = (1 - m) * rv + m * vu
    brm = 3 * U * ((1 - m) * rm.abs() + m * st['mean'].abs()) + m * mean_bound(st) + U * rm2.abs()
    brv = 3 * U * ((1 - m) * rv.abs() + m * vu) + m * f * var_bound(st) + U * rv2.abs() + 2 * U64 * m * vu
    return rm2, rv2, brm, brv


# ---------------------------------------------------------------------------------------------- BatchNorm apply
def bn_apply_emulate(z, mean, invstd, gamma_, beta, relu):
    """bn_apply_kernel bit for bit: fmaf(fp32(gamma invstd), fp32(z - mean), beta), then fmaxf(., 0)."""
    y = fma32((gamma_ * invstd).expand_as(z), z - mean, beta.expand_as(z))
    return torch.clamp_min(y, 0.0) if relu else y


def bn_apply_own(z, mean, invstd, gamma_, beta, relu):
    """-> (exact y from the kernel's own fp32 mean / invstd, bound)."""
    t = gamma_.double() * invstd.double() * (z.double() - mean.double())
    y = t + beta.double()
    b = 3 * U * t.abs() + U * y.abs()
    return (torch.clamp_min(y, 0.0) if relu else y), b


def bn_apply_true(z, st, gamma_, beta, relu, eps):
    """-> (exact y from the float64 statistics, bound for the kernel's y)."""
    g = gamma_.double()
    zc = z.double() - st['mean']
    t = g * st['invstd'] * zc
    y = t + beta.double()
    rel = invstd_rel_bound(st, eps)
    b = 3.1 * U * t.abs() + U * y.abs() + g.abs() * st['invstd'] * (1 + rel) * (mean_bound(st) + zc.abs() * rel)
    return (torch.clamp_min(y, 0.0) if relu else y), b


# ---------------------------------------------------------------------------------------------- BatchNorm backward
def bn_backward_exact(g, z, mean, invstd, gamma_, M=None):
    """g = masked dy (float, any device), z: fp32 [rows, C]; mean / invstd / gamma: the kernel's fp32 inputs.
    M = number of rows of the BatchNorm (the fused backward passes its sparse g over B*npts rows as a dense tensor).
    -> (dz, dgamma, dbeta exact; their bounds), float64."""
    M = g.shape[0] if M is None else M
    gd = g.double()
    xh = (z.double() - mean.double()) * invstd.double()
    gx = gd * xh
    S1, S2 = gd.sum(0), gx.sum(0)
    A1, A2 = gd.abs().sum(0), gx.abs().sum(0)
    gi = gamma_.double() * invstd.double()
    r = gd - S1 / M - xh * (S2 / M)
    dz = gi * r
    T = gd.abs() + S1.abs() / M + xh.abs() * S2.abs() / M
    bdz = gi.abs() * (8 * U * T + 2.2 * U * xh.abs() * A2 / M + 2 * gamma64(M + 2) * A1 / M)
    bdb = U * S1.abs() + gamma64(M + 1) * A1
    bdg = U * S2.abs() + 2.1 * U * A2 + gamma64(M + 2) * A2
    return dz, S2, S1, bdz, bdg, bdb


# ---------------------------------------------------------------------------------------------- losses
def _tanh_err(x):
    """|tanhf(x) - tanh(x)| bound for fp32 x (2 ulp)."""
    return 4 * U * torch.tanh(x).abs() + TINY


def loss_exact(pred, target_mag, radius, target_sign, w_mag, w_sign, fixed_radius):
    """loss_kernel: -> (loss [2] exact, their bounds [2], dpred [B,2] exact, its bound), float64."""
    p = pred.double()
    p0, p1 = p[:, 0], p[:, 1]
    t = target_mag.double() if fixed_radius else target_mag.double() / radius.double()
    B = p.shape[0]
    a, b = torch.tanh(p0.abs()), torch.tanh(t.abs())
    d = a - b
    da = _tanh_err(p0.abs())
    db = _tanh_err(t.abs()) + (0 if fixed_radius else (1 - b * b) * U * t.abs())
    dd = da + db + U * d.abs()
    e0 = 2 * d.abs() * dd + dd * dd + U * (d.abs() + dd) ** 2
    s = target_sign.double()
    e = torch.exp(-p1.abs())
    l1 = torch.clamp_min(p1, 0) - p1 * s + torch.log1p(e)
    e1 = 4 * U * e / (1 + e) + 2 * U * torch.log1p(e) + U * l1.abs() + TINY
    wm, ws = float(np.float32(w_mag)), float(np.float32(w_sign))
    L = torch.stack([wm * (d * d).sum() / B, ws * l1.sum() / B])
    bL = torch.stack([abs(wm) / B * e0.sum(), abs(ws) / B * e1.sum()]) + gamma64(B + 4) * L.abs()
    F = 1 - a * a
    dF = 2 * a.abs() * da + U * a * a + U * F.abs()
    dp0 = 2 * wm * d * F * torch.sign(p0) / B
    bdp0 = abs(2 * wm / B) * (F.abs() * dd + d.abs() * dF + 5 * U * (d * F).abs())
    sig = torch.sigmoid(p1)
    dsig = 4 * U * sig * (1 - sig) + 2.1 * U * sig + TINY
    dp1 = ws * (sig - s) / B
    bdp1 = abs(ws / B) * (dsig + 4.1 * U * (sig - s).abs())
    return L, bL, torch.stack([dp0, dp1], 1), torch.stack([bdp0, bdp1], 1)


def loss_distance_exact(pred, target, radius, w, fixed_radius):
    """loss_distance_kernel: -> (loss [1], bound [1], dpred [B,1], bound), float64."""
    p = pred.double().reshape(-1)
    t = target.double().reshape(-1) if fixed_radius else target.double().reshape(-1) / radius.double().reshape(-1)
    B = p.shape[0]
    a, b = torch.tanh(p), torch.tanh(t)
    d = a - b
    da = _tanh_err(p)
    db = _tanh_err(t) + (0 if fixed_radius else (1 - b * b) * U * t.abs())
    dd = da + db + U * d.abs()
    e0 = 2 * d.abs() * dd + dd * dd + U * (d.abs() + dd) ** 2
    wf = float(np.float32(w))
    L = (wf * (d * d).sum() / B).reshape(1)
    bL = (abs(wf) / B * e0.sum()).reshape(1) + gamma64(B + 4) * L.abs()
    F = 1 - a * a
    dF = 2 * a.abs() * da + U * a * a + U * F.abs()
    dp = 2 * wf * d * F / B
    bdp = abs(2 * wf / B) * (F.abs() * dd + d.abs() * dF + 5 * U * (d * F).abs())
    return L, bL, dp.reshape(-1, 1), bdp.reshape(-1, 1)


# ---------------------------------------------------------------------------------------------- quaternions
# A(q) as monomials: A_ij = sum_t coef * q_m q_n (row-major 3x3), utils.batch_quat_to_rotmat
_A_TERMS = [
    [(-1, 2, 2), (-1, 3, 3)], [(1, 1, 2), (-1, 3, 0)], [(1, 1, 3), (1, 2, 0)],
    [(1, 1, 2), (1, 3, 0)], [(-1, 1, 1), (-1, 3, 3)], [(1, 2, 3), (-1, 1, 0)],
    [(1, 1, 3), (-1, 2, 0)], [(1, 2, 3), (1, 1, 0)], [(-1, 1, 1), (-1, 2, 2)],
]


def quat_fp32(q4):
    """The fp32 quaternion the model forms: q4 + (1, 0, 0, 0) in fp32."""
    return q4.float() + q4.new_tensor([1.0, 0.0, 0.0, 0.0]).float()


def _A_and_abs(q):
    A = torch.stack([sum(c * q[:, m] * q[:, n] for c, m, n in ts) for ts in _A_TERMS], 1)
    Aabs = torch.stack([sum((q[:, m] * q[:, n]).abs() for c, m, n in ts) for ts in _A_TERMS], 1)
    return A, Aabs


def _dA(q):
    """dA_ij/dq_k as [B, 4, 9] (each entry one monomial, or zero)."""
    out = q.new_zeros(q.shape[0], 4, 9)
    for ij, ts in enumerate(_A_TERMS):
        for c, m, n in ts:
            out[:, m, ij] += c * q[:, n]
            out[:, n, ij] += c * q[:, m]
    return out


def quat_to_rot_exact(q4):
    """-> (R [B,9] exact, bound), float64."""
    q = quat_fp32(q4).double()
    s = 2.0 / (q * q).sum(1, keepdim=True)
    A, Aabs = _A_and_abs(q)
    R = s * A + torch.eye(3, dtype=torch.float64, device=q.device).reshape(1, 9)
    b = s * (gamma(3) * Aabs + gamma(7) * A.abs()) + U * R.abs()
    return R, b


def quat_to_rot_bwd_exact(q4, dR):
    """-> (dq [B,4] exact, bound), float64."""
    q = quat_fp32(q4).double()
    g = dR.double().reshape(-1, 9)
    s = 2.0 / (q * q).sum(1, keepdim=True)
    A, Aabs = _A_and_abs(q)
    J = _dA(q)                                              # [B,4,9]
    GA = (g * A).sum(1, keepdim=True)
    GAabs = (g.abs() * Aabs).sum(1, keepdim=True)
    D = (J * g.unsqueeze(1)).sum(2)
    Dabs = (J.abs() * g.abs().unsqueeze(1)).sum(2)
    dq = -s * s * q * GA + s * D
    b = s * s * q.abs() * (gamma(13) * GA.abs() + gamma(11) * GAabs) + s * (gamma(6) * D.abs() + gamma(8) * Dabs) + U * dq.abs()
    return dq, b


# ---------------------------------------------------------------------------------------------- reduction orders
def col_reduce_grid(M, C, sm_count=SM_COUNT_H100):
    """rows_per_block of col_reduce_grid (train_ops.cu) on a device with `sm_count` SMs."""
    cx = -(-C // 32)
    want = max(1, -(-8 * sm_count // cx))
    rpb = max(64, -(-M // want))
    rpb = min(rpb, 4096)
    return max(rpb, -(-M // 65535))


def _fma32_np(a, b, c):
    return fma32(torch.from_numpy(a), torch.from_numpy(b), torch.from_numpy(c)).numpy()


def _blocked(z, rpb):
    """z fp32 [M] (one column) -> [blocks, 8, steps] view of the rows each thread of col_reduce_kernel walks (thread ty of
    block k takes rows k rpb + ty, + 8, ...), zero-padded, and the matching validity mask."""
    M = z.shape[0]
    nb = -(-M // rpb)
    steps = -(-rpb // 8)
    zp = np.zeros(nb * steps * 8, dtype=z.dtype)
    valid = np.zeros(nb * steps * 8, dtype=bool)
    rows = np.arange(M)
    blk, off = rows // rpb, rows % rpb
    pos = blk * (steps * 8) + (off % 8) * steps + off // 8
    zp[pos] = z
    valid[pos] = True
    return zp.reshape(nb, 8, steps), valid.reshape(nb, 8, steps)


def _finish(d1, d2, M, eps, shift):
    """Block merge (8 f64 adds per block), cross-block f64 sum, bn_finalize -> (mean, invstd) as fp32."""
    s1 = s2 = 0.0
    for k in range(d1.shape[0]):
        b1 = b2 = 0.0
        for j in range(8):
            b1 += float(d1[k, j])
            b2 += float(d2[k, j])
        s1 += b1
        s2 += b2
    md = s1 / M
    var = max(s2 / M - md * md, 0.0)
    return np.float32(shift + md), np.float32(1.0 / math.sqrt(var + float(np.float32(eps))))


def col_stats_old_order(z, rpb, eps=1e-5):
    """The previous col_reduce_kernel<0> on one fp32 column: fp32 partials a1 += v, a2 = fmaf(v, v, a2) over each thread's
    rows (up to rpb / 8), f64 block merge and cross-block sum of sum z, sum z^2, var = E[z^2] - E[z]^2."""
    zp, valid = _blocked(np.asarray(z, np.float32), rpb)
    a1 = np.zeros(zp.shape[:2], np.float32)
    a2 = np.zeros(zp.shape[:2], np.float32)
    for t in range(zp.shape[2]):
        v = np.where(valid[:, :, t], zp[:, :, t], np.float32(0))
        a1 = (a1 + v).astype(np.float32)
        a2 = _fma32_np(v, v, a2)
    return _finish(a1.astype(np.float64), a2.astype(np.float64), len(z), eps, 0.0)


def col_stats_new_order(z, rpb, eps=1e-5):
    """The shipped col_reduce_kernel<0> + bn_finalize on one fp32 column: d = z - z[0] in f64, f64 sums from the first
    term, mean = z0 + s1 / M, var = s2 / M - (s1 / M)^2."""
    z = np.asarray(z, np.float32)
    zp, valid = _blocked(z, rpb)
    x0 = float(z[0])
    a1 = np.zeros(zp.shape[:2])
    a2 = np.zeros(zp.shape[:2])
    for t in range(zp.shape[2]):
        d = np.where(valid[:, :, t], zp[:, :, t].astype(np.float64) - x0, 0.0)
        a1 = a1 + d
        a2 = a2 + d * d          # fma(d, d, a2) in f64: d*d + a2 rounded once; the plain form rounds twice, u64 apart
    return _finish(a1, a2, len(z), eps, x0)
