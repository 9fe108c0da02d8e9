"""Float64 model of the split-precision operand arithmetic of the training GEMMs (csrc/fc_tc.cu, csrc/gemm_tn_tc.cu),
and the per-element error bound those GEMMs are held to.

Every fp32 operand x is split into two fp16 numbers, hi = fp16(x) and lo = fp16(x - hi), and a product is evaluated as
lo_a hi_b + hi_a lo_b + hi_a hi_b.  That keeps ~22 bits of x only while hi and lo are fp16 normal numbers
(2^-3 <~ |x| <= 65504).  `scaled=False` models the split applied to the raw operands; `scaled=True` models the shipped
kernels, which first multiply every row (gemm_nt) or column (gemm_tn) of an operand by 2^split_exp(its max |x|) and
undo the two scales on the result.  The products and their sums are formed in float64, so the model shows the error of
the operand split alone; accumulation rounding is what the bound's first term allows for.

Bound, for C = sum_k a_k b_k over a reduction of length K, every element:

    |C - C_f64| <= gamma_K sum_k |a_k| |b_k| + C2 K max_k |a_k| max_k |b_k|

gamma_K = K u / (1 - K u) with u = 2^-24 is the classical bound for an fp32 dot product of length K evaluated in any order
with rounding to nearest, with or without FMA (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., eq. 3.5).
It is what the plain fp32 FMA kernels satisfy by construction.  The second term is a floor: an implementation may lose
the parts of the operands that lie more than ~2^-40 below the largest element of their row or column."""
import numpy as np
import torch

U32 = 2.0 ** -24
C2 = 2.0 ** -40


def gamma(K):
    """gamma_K = K u / (1 - K u) for fp32 (u = 2^-24)."""
    return K * U32 / (1.0 - K * U32)


def split(x):
    """fp32 tensor -> (hi, lo) as float64 tensors holding fp16 values, as split_half2 / pack_fc_kernel compute them:
    hi = fp16(x), lo = fp16(fp32(x - hi))."""
    x = x.float()
    hi = x.half()
    lo = (x - hi.float()).half()
    return hi.double(), lo.double()


def split_exp(amax):
    """Scale exponent s of a row / column with largest magnitude `amax` (float32 array): amax 2^s lies in
    [2^15, 65504]; 0 for zero or non-finite maxima (model.cuh, split_exp)."""
    amax = np.asarray(amax, dtype=np.float32)
    f, e = np.frexp(amax.astype(np.float64))
    s = np.where(f * 65536.0 > 65504.0, 15 - e, 16 - e)
    return np.where((amax > 0) & np.isfinite(amax), s, 0).astype(np.int64)


def _scale_rows(x, s):
    return (x.double() * torch.pow(2.0, torch.from_numpy(s).double()).unsqueeze(1)).float()


def gemm_nt(A, W, scaled=True):
    """C[m][n] = sum_k A[m][k] W[n][k] under the split arithmetic (float64 result)."""
    A, W = A.detach().cpu().float(), W.detach().cpu().float()
    if scaled:
        sa = split_exp(A.abs().amax(1).numpy() if A.shape[1] else np.zeros(A.shape[0], np.float32))
        sw = split_exp(W.abs().amax(1).numpy() if W.shape[1] else np.zeros(W.shape[0], np.float32))
        A, W = _scale_rows(A, sa), _scale_rows(W, sw)
    ah, al = split(A)
    wh, wl = split(W)
    C = al @ wh.t() + ah @ wl.t() + ah @ wh.t()
    if scaled:
        C = C * torch.pow(2.0, -torch.from_numpy(sa[:, None] + sw[None, :]).double())
    return C


def gemm_tn(A, B, scaled=True):
    """C[n][k] = sum_m A[m][n] B[m][k] under the split arithmetic; the scales are per column of A and of B."""
    return gemm_nt(A.t(), B.t(), scaled)


def bound_nt(A, W, extra=None):
    """Per-element bound for sum_k A[m][k] W[n][k] (float64 [M, N]).  `extra` is an fp32 term added to the product (the
    running gradient of the accumulate form, or a bias): it joins the sum as one more term."""
    A, W = A.detach().double(), W.detach().double()
    K = A.shape[1]
    absum = A.abs() @ W.abs().t()
    if extra is not None:
        absum = absum + extra.detach().double().abs()
        K += 1
    ma = A.abs().amax(1) if A.shape[1] else A.new_zeros(A.shape[0])
    mw = W.abs().amax(1) if W.shape[1] else W.new_zeros(W.shape[0])
    return gamma(K) * absum + C2 * A.shape[1] * ma[:, None] * mw[None, :]


def excess(C, exact, bound):
    """max over elements of |C - exact| / bound: <= 1 meets the bound.  A zero bound demands an exact zero error; a
    non-finite C counts as infinite."""
    C, exact, bound = C.detach().double(), exact.detach().double().to(C.device), bound.to(C.device)
    err = (C - exact).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    r = torch.where(torch.isfinite(C), r, torch.full_like(r, float('inf')))
    return float(r.max()) if r.numel() else 0.0
