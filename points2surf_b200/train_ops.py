"""Tensor-level wrappers of the training-step primitives (include/p2s_b200.h `p2s_op_*`, csrc/train_ops.cu).
`CudaPrims` is the only backend of points2surf_b200.train; every call goes through the C ABI on CUDA tensors."""
import ctypes as C

import torch

from . import _lib
from ._lib import check
from .ops import _dev, _ptr, _stream, P2SError


def _f(t, name):
    return _dev(t, torch.float32, name)


class CudaPrims:
    """Stateless op set; tensors in, tensors out, all fp32 CUDA (f64 reductions are converted on the device)."""

    name = 'cuda'

    def __init__(self):
        self.lib = _lib.load()

    # ---- GEMMs
    def gemm_nt(self, A, W, bias=None, relu=False):
        """A [M,K] or [Z,M,K]; W [N,K] or [Z,N,K]  ->  act(A W^T + bias) [M,N] or [Z,M,N]."""
        A, W = _f(A, 'A'), _f(W, 'W')
        batched = A.dim() == 3
        Z = A.shape[0] if batched else 1
        M, K = A.shape[-2], A.shape[-1]
        N = W.shape[-2]
        if W.shape[-1] != K:
            raise P2SError('gemm_nt: K mismatch %s x %s' % (tuple(A.shape), tuple(W.shape)))
        out = torch.empty((Z, M, N) if batched else (M, N), dtype=torch.float32, device=A.device)
        w_stride = N * K if W.dim() == 3 else 0
        b = _f(bias, 'bias') if bias is not None else None
        with torch.cuda.device(A.device):
            check(self.lib.p2s_op_gemm_nt(_ptr(A), M * K, K, _ptr(W), w_stride, _ptr(b) if b is not None else None, _ptr(out),
                                          M * N, N, M, N, K, Z, 1 if relu else 0, _stream()))
        return out

    def gemm_tn(self, A, B, out=None):
        """A [M,N], B [M,K] (or batched [Z,M,*]) -> A^T B [N,K] (or [Z,N,K]); with `out` the product is ADDED to it."""
        A, B = _f(A, 'A'), _f(B, 'B')
        batched = A.dim() == 3
        Z = A.shape[0] if batched else 1
        M, N = A.shape[-2], A.shape[-1]
        K = B.shape[-1]
        if B.shape[-2] != M:
            raise P2SError('gemm_tn: M mismatch')
        acc = out is not None
        if acc:
            if not out.is_contiguous() or out.numel() != Z * N * K or out.dtype != torch.float32 or not out.is_cuda:
                raise P2SError('gemm_tn: bad `out`')
        else:
            out = torch.empty((Z, N, K) if batched else (N, K), dtype=torch.float32, device=A.device)
        with torch.cuda.device(A.device):
            check(self.lib.p2s_op_gemm_tn(_ptr(A), M * N, N, _ptr(B), M * K, K, _ptr(out), N * K, K, M, N, K, Z, 1 if acc else 0,
                                          _stream()))
        return out

    def transpose(self, x):
        x = _f(x, 'x')
        Z = x.shape[0] if x.dim() == 3 else 1
        r, c = x.shape[-2], x.shape[-1]
        out = torch.empty(((Z, c, r) if x.dim() == 3 else (c, r)), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            check(self.lib.p2s_op_transpose(_ptr(x), _ptr(out), r, c, Z, _stream()))
        return out

    # ---- BatchNorm1d (training mode)
    def bn_forward(self, z, gamma, beta, relu, running_mean=None, running_var=None, eps=1e-5, momentum=0.1):
        z = _f(z, 'z')
        M, Cc = z.shape
        s = torch.empty((2, Cc), dtype=torch.float64, device=z.device)
        mean = torch.empty(Cc, dtype=torch.float32, device=z.device)
        invstd = torch.empty_like(mean)
        y = torch.empty_like(z)
        with torch.cuda.device(z.device):
            check(self.lib.p2s_op_col_stats(_ptr(z), M, Cc, _ptr(s[0]), _ptr(s[1]), _stream()))
            check(self.lib.p2s_op_bn_finalize(_ptr(s[0]), _ptr(s[1]), M, Cc, float(eps), float(momentum), _ptr(mean), _ptr(invstd),
                                              _ptr(running_mean) if running_mean is not None else None,
                                              _ptr(running_var) if running_var is not None else None, _stream()))
            check(self.lib.p2s_op_bn_apply(_ptr(z), M, Cc, _ptr(mean), _ptr(invstd), _ptr(_f(gamma, 'gamma')), _ptr(_f(beta, 'beta')),
                                           1 if relu else 0, _ptr(y), _stream()))
        return y, mean, invstd

    def bn_apply(self, z, mean, invstd, gamma, beta, relu):
        """act(gamma (z - mean) invstd + beta) with given statistics (eval-mode BatchNorm: running mean / rsqrt(var + eps))."""
        z = _f(z, 'z')
        M, Cc = z.shape
        y = torch.empty_like(z)
        with torch.cuda.device(z.device):
            check(self.lib.p2s_op_bn_apply(_ptr(z), M, Cc, _ptr(_f(mean, 'mean')), _ptr(_f(invstd, 'invstd')), _ptr(_f(gamma, 'gamma')),
                                           _ptr(_f(beta, 'beta')), 1 if relu else 0, _ptr(y), _stream()))
        return y

    def bn_backward(self, dy, z, y_mask, mean, invstd, gamma):
        """-> dz, dgamma, dbeta.  y_mask = forward output when a ReLU follows the BatchNorm, else None."""
        dy, z = _f(dy, 'dy'), _f(z, 'z')
        M, Cc = z.shape
        s = torch.empty((2, Cc), dtype=torch.float64, device=z.device)
        dz = torch.empty_like(z)
        with torch.cuda.device(z.device):
            check(self.lib.p2s_op_bn_backward(_ptr(dy), _ptr(z), _ptr(_f(y_mask, 'y')) if y_mask is not None else None, M, Cc,
                                              _ptr(mean), _ptr(invstd), _ptr(_f(gamma, 'gamma')), _ptr(s[0]), _ptr(s[1]), _ptr(dz),
                                              _stream()))
        return dz, s[1].float(), s[0].float()

    def bn_maxpool_forward(self, z, B, npts, gamma, beta, relu, running_mean=None, running_var=None, eps=1e-5, momentum=0.1):
        """max over the points of act(BN_train(z)) without materialising it -> out [B,C], arg [B,C], mean, invstd."""
        z = _f(z, 'z')
        M, Cc = z.shape
        s = torch.empty((2, Cc), dtype=torch.float64, device=z.device)
        mean = torch.empty(Cc, dtype=torch.float32, device=z.device)
        invstd = torch.empty_like(mean)
        out = torch.empty((B, Cc), dtype=torch.float32, device=z.device)
        arg = torch.empty((B, Cc), dtype=torch.int32, device=z.device)
        with torch.cuda.device(z.device):
            check(self.lib.p2s_op_col_stats(_ptr(z), M, Cc, _ptr(s[0]), _ptr(s[1]), _stream()))
            check(self.lib.p2s_op_bn_finalize(_ptr(s[0]), _ptr(s[1]), M, Cc, float(eps), float(momentum), _ptr(mean), _ptr(invstd),
                                              _ptr(running_mean) if running_mean is not None else None,
                                              _ptr(running_var) if running_var is not None else None, _stream()))
            check(self.lib.p2s_op_bn_maxpool_fwd(_ptr(z), B, npts, Cc, _ptr(mean), _ptr(invstd), _ptr(_f(gamma, 'gamma')),
                                                 _ptr(_f(beta, 'beta')), 1 if relu else 0, _ptr(out), _ptr(arg), _stream()))
        return out, arg, mean, invstd

    def bn_maxpool_backward(self, dout, arg, out, z, mean, invstd, gamma, relu, B, npts):
        """-> dz [B*npts, C], dgamma, dbeta."""
        z = _f(z, 'z')
        Cc = z.shape[1]
        s = torch.empty((2, Cc), dtype=torch.float64, device=z.device)
        dz = torch.empty_like(z)
        with torch.cuda.device(z.device):
            check(self.lib.p2s_op_bn_maxpool_bwd(_ptr(_f(dout, 'dout')), _ptr(_dev(arg, torch.int32, 'arg')), _ptr(_f(out, 'out')), _ptr(z),
                                                 B, npts, Cc, _ptr(mean), _ptr(invstd), _ptr(_f(gamma, 'gamma')), 1 if relu else 0,
                                                 _ptr(s[0]), _ptr(s[1]), _ptr(dz), _stream()))
        return dz, s[1].float(), s[0].float()

    def col_sum(self, x):
        x = _f(x, 'x')
        M, Cc = x.shape
        s = torch.empty(Cc, dtype=torch.float64, device=x.device)
        with torch.cuda.device(x.device):
            check(self.lib.p2s_op_col_sum(_ptr(x), M, Cc, _ptr(s), _stream()))
        return s.float()

    # ---- symmetric max
    def maxpool_fwd(self, y, B, npts):
        y = _f(y, 'y')
        Cc = y.shape[-1]
        out = torch.empty((B, Cc), dtype=torch.float32, device=y.device)
        arg = torch.empty((B, Cc), dtype=torch.int32, device=y.device)
        with torch.cuda.device(y.device):
            check(self.lib.p2s_op_maxpool_fwd(_ptr(y), B, npts, Cc, _ptr(out), _ptr(arg), _stream()))
        return out, arg

    def maxpool_bwd(self, dout, arg, npts):
        dout = _f(dout, 'dout')
        B, Cc = dout.shape
        dy = torch.empty((B * npts, Cc), dtype=torch.float32, device=dout.device)
        with torch.cuda.device(dout.device):
            check(self.lib.p2s_op_maxpool_bwd(_ptr(dout), _ptr(_dev(arg, torch.int32, 'arg')), B, npts, Cc, _ptr(dy), _stream()))
        return dy

    # ---- loss, rotations, small element-wise ops
    def loss(self, pred, target_mag, radius, target_sign, w_mag, w_sign, fixed_radius=False, need_grad=True):
        pred = _f(pred, 'pred')
        B = pred.shape[0]
        out = torch.empty(2, dtype=torch.float64, device=pred.device)
        dpred = torch.empty_like(pred) if need_grad else None
        with torch.cuda.device(pred.device):
            check(self.lib.p2s_op_loss(_ptr(pred), _ptr(_f(target_mag, 'target_mag')), _ptr(_f(radius, 'radius')),
                                       _ptr(_f(target_sign, 'target_sign')), B, float(w_mag), float(w_sign), 1 if fixed_radius else 0,
                                       _ptr(out), _ptr(dpred) if need_grad else None, _stream()))
        return out, dpred

    def loss_distance(self, pred, target, radius, w, fixed_radius=False, need_grad=True):
        """Regression loss of the one-output head: -> (f64 [1] = [w * mse(tanh p, tanh(t / r))], dpred [B,1] or None)."""
        pred = _f(pred, 'pred')
        B = pred.shape[0]
        if pred.numel() != B:
            raise P2SError('loss_distance: pred must have one column, got %s' % (tuple(pred.shape),))
        out = torch.empty(1, dtype=torch.float64, device=pred.device)
        dpred = torch.empty_like(pred) if need_grad else None
        with torch.cuda.device(pred.device):
            check(self.lib.p2s_op_loss_distance(_ptr(pred), _ptr(_f(target, 'target')),
                                                None if fixed_radius else _ptr(_f(radius, 'radius')), B, float(w),
                                                1 if fixed_radius else 0, _ptr(out), _ptr(dpred) if need_grad else None,
                                                _stream()))
        return out, dpred

    def quat_to_rot(self, q):
        q = _f(q, 'q')
        R = torch.empty((q.shape[0], 3, 3), dtype=torch.float32, device=q.device)
        with torch.cuda.device(q.device):
            check(self.lib.p2s_op_quat_to_rot(_ptr(q), _ptr(R), q.shape[0], _stream()))
        return R

    def quat_to_rot_bwd(self, q, dR):
        q, dR = _f(q, 'q'), _f(dR, 'dR')
        dq = torch.empty_like(q)
        with torch.cuda.device(q.device):
            check(self.lib.p2s_op_quat_to_rot_bwd(_ptr(q), _ptr(dR), q.shape[0], _ptr(dq), _stream()))
        return dq

    def add_row_(self, x, v):
        x = _f(x, 'x')
        with torch.cuda.device(x.device):
            check(self.lib.p2s_op_add_row(_ptr(x), _ptr(_f(v, 'v')), x.shape[0], x.shape[1], _stream()))
        return x

    def center(self, pts, q):
        pts = _f(pts, 'pts')
        out = torch.empty_like(pts)
        with torch.cuda.device(pts.device):
            check(self.lib.p2s_op_center(_ptr(pts), _ptr(_f(q, 'q')), pts.shape[0], pts.shape[1], _ptr(out), _stream()))
        return out

    def axpy_(self, y, x, a=1.0):
        y = _f(y, 'y')
        with torch.cuda.device(y.device):
            check(self.lib.p2s_op_axpy(_ptr(y), _ptr(_f(x, 'x')), float(a), y.numel(), _stream()))
        return y

    def sgd_(self, param, grad, buf, lr, momentum, first):
        with torch.cuda.device(param.device):
            check(self.lib.p2s_op_sgd(_ptr(_f(param, 'param')), _ptr(_f(grad, 'grad')), _ptr(_f(buf, 'buf')), param.numel(), float(lr),
                                      float(momentum), 1 if first else 0, _stream()))
