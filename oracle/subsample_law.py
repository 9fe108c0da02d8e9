"""The exact law of the distance-weighted sub-sample (source/base/utils.py:196-219), in float64.

The reference draws S of N points with RandomState.choice(replace=False, p), p ~ w: successive sampling.  Its inclusion
probabilities are those of exponential clocks (Efraimidis-Spirakis): point i is drawn when its clock E_i / w_i is among the
S smallest, so

    pi_i = int_0^inf w_i exp(-w_i t) P(K_-i(t) <= S - 1) dt,

where K_-i(t) counts the other points whose clocks fall below t, a Poisson-binomial variable with p_j(t) = 1 - exp(-w_j t).
The law of the full count K(t) is built once per quadrature node by a product tree of FFT convolutions; K_-i(t) is K(t) with
one Bernoulli(p_i(t)) deconvolved, so pi_i depends on w_i and K alone.  It is evaluated at the distinct weights, or at
Chebyshev nodes in w followed by barycentric interpolation when there are many of them.

`set_law` gives the probability of every S-subset for tiny N (the sum over orderings of the successive-draw products), which
the integral is checked against.
"""
import math

import numpy as np
import torch

from oracle import p2s_oracle as orc

_TAIL = 1e-18           # Bernstein bound below which a tail of K(t) is treated as empty
_PANELS, _GL = 16, 16   # composite Gauss-Legendre in log t over the band where P(K_-i(t) <= S - 1) is neither 0 nor 1
_DIRECT = 128           # at most this many distinct weights: evaluate at each; more: Chebyshev interpolation
_CHEB = 64


def weights(pts, query, dmax_scale=1.0, floor=0.05):
    """The reference's float32 weights as float64.  `dmax_scale` and `floor` perturb the law (for power analysis)."""
    if dmax_scale == 1.0 and floor == 0.05:
        return orc.sub_sample_weights(pts, query).astype(np.float64)
    dist = np.linalg.norm(np.broadcast_to(query, pts.shape) - pts, axis=1)
    prob = 1.0 - 1.5 * (dist / (np.max(dist) * np.float32(dmax_scale)))
    return np.clip(prob, np.float32(floor), 1.0).astype(np.float64)


def _pb_law(p):
    """Poisson-binomial law: p [B, n] float64 -> [B, n + 1], by a product tree of FFT convolutions."""
    B, n = p.shape
    m = 1 << max(0, (n - 1).bit_length())
    pp = torch.zeros((B, m), dtype=torch.float64, device=p.device)
    pp[:, :n] = p
    poly = torch.stack([1.0 - pp, pp], dim=-1)              # [B, leaves, 2]
    while poly.shape[1] > 1:
        a, b = poly[:, 0::2], poly[:, 1::2]
        L = a.shape[-1]
        f = 2 * L
        poly = torch.fft.irfft(torch.fft.rfft(a, f) * torch.fft.rfft(b, f), f)[..., :2 * L - 1]
    return poly[:, 0, :n + 1]


def _le_without_one(P, p, S):
    """P(K' <= S - 1) for K = K' + Bernoulli(p): P [B, N+1] law of K, p [E, B] -> [E, B].
    p <= 1/2: forward deconvolution, P(K' <= S-1) = sum_{j<S} P_j (1 - (-p/(1-p))^(S-j));
    p >  1/2: backward, P(K' >= S) = sum_{j>S} P_j (1 - (-(1-p)/p)^(j-S)).  Both recurrences damp their errors."""
    N = P.shape[1] - 1
    live = (P.abs() > 1e-15).any(dim=0).nonzero()
    lo, hi = int(live.min()), int(live.max())               # outside [lo, hi] the law is below the FFT noise
    below = P[:, :S].sum(dim=1)                              # P(K <= S - 1)
    lo = min(lo, S)
    j = torch.arange(lo, S, device=P.device, dtype=torch.float64)
    rho = (p / (1.0 - p)).clamp(max=1.0)
    e = S - j                                                # exponents 1 .. S - lo
    sign = torch.where(e.remainder(2) == 0, 1.0, -1.0)
    pw = sign * torch.exp(e * torch.log(rho.clamp(min=1e-300))[..., None])
    fwd = below[None, :] - (P[None, :, lo:S] * pw).sum(-1)
    hi = min(hi, N)
    if hi > S:
        j2 = torch.arange(S + 1, hi + 1, device=P.device, dtype=torch.float64)
        sig = ((1.0 - p) / p.clamp(min=1e-300)).clamp(max=1.0)
        e2 = j2 - S
        sign2 = torch.where(e2.remainder(2) == 0, 1.0, -1.0)
        pw2 = sign2 * torch.exp(e2 * torch.log(sig.clamp(min=1e-300))[..., None])
        bwd = 1.0 - (P[None, :, S + 1:hi + 1] * (1.0 - pw2)).sum(-1)
    else:
        bwd = torch.ones_like(fwd)
    return torch.where(p <= 0.5, fwd, bwd)


def _bernstein(a, v):
    """Bernstein bound on P(K - E K >= a) (or <= -a) for a sum of independent Bernoullis with variance v."""
    with np.errstate(divide='ignore', invalid='ignore'):
        return np.where(a > 0, np.exp(-a * a / (2.0 * (v + a / 3.0))), 1.0)


def inclusion_probabilities(w, S, device='cpu', chunk=32):
    """pi_i of successive sampling of S points with p ~ w (float64 [N], all > 0)."""
    w = np.asarray(w, dtype=np.float64)
    N = len(w)
    assert 1 <= S <= N and (w > 0).all()
    if S == N:
        return np.ones(N)
    uw, inv, cnt = np.unique(w, return_inverse=True, return_counts=True)
    # band of t where P(K_-i(t) <= S - 1) is not 0 or 1 up to _TAIL (K - 1 <= K_-i <= K)
    ts = np.logspace(np.log10(1e-12 / uw[-1]), np.log10(41.0 / uw[0]), 4000)
    pt = -np.expm1(-np.outer(ts, uw))
    mu, var = pt @ cnt, (pt * (1 - pt)) @ cnt
    a_lo, a_hi = S - mu, mu - S
    ok_lo = (a_lo > 0) & (_bernstein(np.maximum(a_lo, 0), var) < _TAIL)
    ok_hi = (a_hi > 0) & (_bernstein(np.maximum(a_hi, 0), var) < _TAIL)
    t_a = ts[ok_lo].max() if ok_lo.any() else ts[0]
    t_b = ts[ok_hi].min() if ok_hi.any() else ts[-1]
    x, gw = np.polynomial.legendre.leggauss(_GL)
    edges = np.linspace(np.log(t_a), np.log(t_b), _PANELS + 1)
    u = ((edges[:-1, None] + edges[1:, None]) / 2 + (edges[1:, None] - edges[:-1, None]) / 2 * x[None, :]).ravel()
    qw = ((edges[1:, None] - edges[:-1, None]) / 2 * gw[None, :]).ravel()
    t = np.exp(u)
    if len(uw) <= _DIRECT:
        we = uw
    else:
        k = np.arange(_CHEB)
        we = (uw[0] + uw[-1]) / 2 + (uw[-1] - uw[0]) / 2 * np.cos(np.pi * (2 * k + 1) / (2 * _CHEB))
    dev = torch.device(device)
    wt = torch.from_numpy(w).to(dev)
    wet = torch.from_numpy(we).to(dev)
    acc = torch.from_numpy(-np.expm1(-we * t_a)).to(dev)     # t < t_a: P(K_-i <= S - 1) = 1
    for b0 in range(0, len(t), chunk):
        tb = torch.from_numpy(t[b0:b0 + chunk]).to(dev)
        P = _pb_law(-torch.expm1(-tb[:, None] * wt[None, :]))
        pe = -torch.expm1(-wet[:, None] * tb[None, :])        # [E, B]
        F = _le_without_one(P, pe, S)
        g = wet[:, None] * torch.exp(-wet[:, None] * tb[None, :]) * tb[None, :] * F
        acc = acc + (g * torch.from_numpy(qw[b0:b0 + chunk]).to(dev)[None, :]).sum(1)
    pe_ = acc.cpu().numpy()
    if len(uw) <= _DIRECT:
        return pe_[inv]
    # barycentric interpolation on Chebyshev points of the first kind
    k = np.arange(_CHEB)
    bw = (-1.0) ** k * np.sin(np.pi * (2 * k + 1) / (2 * _CHEB))
    diff = uw[:, None] - we[None, :]
    exact = diff == 0
    diff[exact] = 1.0
    c = bw[None, :] / diff
    out = (c @ pe_) / c.sum(1)
    hit = exact.any(1)
    out[hit] = pe_[exact[hit].argmax(1)]
    return out[inv]


def set_law(w, S):
    """Probability of every S-subset under successive sampling (tiny N): {sorted id tuple: probability}.
    P(first m draws form A) = sum_{i in A} P(first m-1 draws form A - i) * w_i / (W - w(A - i)), summed over subsets."""
    w = [float(v) for v in w]
    N, W = len(w), math.fsum(w)
    assert N <= 16 and 1 <= S <= N
    prob = {0: 1.0}
    for _ in range(S):
        nxt = {}
        for mask, pr in prob.items():
            rest = W - math.fsum(w[i] for i in range(N) if mask >> i & 1)
            for i in range(N):
                if not mask >> i & 1:
                    nxt[mask | 1 << i] = nxt.get(mask | 1 << i, 0.0) + pr * w[i] / rest
        prob = nxt
    return {tuple(i for i in range(N) if m >> i & 1): p for m, p in prob.items()}


def set_inclusion(law, N):
    pi = np.zeros(N)
    for s, p in law.items():
        pi[list(s)] += p
    return pi


def equal_mass_bins(pi, d, nbins=20):
    """Bin index per point: points ordered by distance d to the query, cut into `nbins` groups of about equal sum(pi)."""
    order = np.argsort(d, kind='stable')
    cum = np.cumsum(pi[order]) - pi[order] / 2
    b = np.minimum((cum / cum[-1] * nbins).astype(np.int64), nbins - 1) if cum[-1] > 0 else np.zeros(len(d), np.int64)
    out = np.empty(len(d), np.int64)
    out[order] = b
    return out
