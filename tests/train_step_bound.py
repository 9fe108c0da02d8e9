"""Float64 restatement of one training iteration of points2surf_b200.train.TrainStep, conditioned on the step's own
ReLU, max-pool and |p0| decisions, with a per-element error scale for the fp32 step next to every value.

Why conditioning.  An unconditioned float64 step and an fp32 step take different max-pool arg-maxes and ReLU masks
wherever two candidates are within rounding of each other, and after ~40 layers those flips move whole tensors by a
few percent, which is why the older tests compare relative L2 norms.  Here the float64 step is handed the fp32 step's
decisions: every ReLU multiplies by the step's mask (`tape.y_mask > 0`), every max over points gathers the step's `arg`
(and, after the fused BN + max-pool with ReLU of the STN conv3s, multiplies by `out > 0`: the kernel sends no gradient
where the pooled value is 0, train_ops.cu bn_maxpool_bwd), and the magnitude loss uses the sign of the step's p0,
including 0 (train_ops.cu loss_kernel `sg`).  The bias of a layer in front of a train-mode BatchNorm gets a gradient
of exactly 0, as TrainStep keeps it.  What is left between the two steps is rounding, and that is bounded per element.
The rest is the reference's math (oracle/train_oracle.py, pinned to the unmodified reference): BatchNorm with batch
statistics, running mean and unbiased running var, the quaternion, both losses and SGD with momentum.  With its own
decisions the value part equals TrainStep(dtype=float64, prims=TorchPrims()) to 1e-11 of each tensor's largest element
(tests/test_train_step_bound_host.py).

Each step starts from the state the fp32 step held before it (parameters, momentum buffers, running statistics,
promoted exactly), so differences never compound across steps.

Error scale.  Values are net_bound.V (v, e): first-order propagation, the terms of one sum added in quadrature, local
rounding bounds added in quadrature to the propagated part, and the check |x - v| <= LAMBDA e with net_bound's
LAMBDA = 4 (Hoeffding's argument: oracle/net_bound.py docstring).  e = None marks an exact value (parameters, inputs).
u = 2^-24, u64 = 2^-53; |.| and squares are element-wise.

* GEMMs (`_mm`), net_bound's linear-step rule, with |a| + e_a and |b| + e_b in the operand terms:
      e^2 = e_a^2 b^2 + a^2 e_b^2 + rho^2 |a|^2|b|^2 + n (u (1 + 2^-9))^2 (|a|^2|b|^2 + bias^2 + v^2) + floor^2
  - 'split' (the tensor-core kernels, fc_tc.cu launch_gemm_nt_tc :403-425, gemm_tn_tc.cu :161-177): rho = 3 2^-22,
    n = 3 K (three MMAs per k-step), u = 2^-23 (truncating accumulation), floor = split_gemm's 2^-40 K max|a| max|b|
    with the maxima over the reduction (the power-of-two scales are per row of A and W, per column of dZ and X).
  - 'fp32' (the FMA kernels, train_ops.cu launch_gemm_nt / op_gemm_tn): rho = 0, n = K, u = 2^-24, no floor.
  - Which kernel a call takes is restated from its shape: gemm_nt_tc_ok (fc_tc.cu:398-402: one batch, N % 4 == 0,
    64 <= N <= 4096, K % 32 == 0, M >= 128) and gemm_tn_tc_ok (gemm_tn_tc.cu:153-157: one batch, M >= 4096, N, K >= 64,
    N % 4 == K % 4 == 0); P2S_TRAIN_GEMM_FP32=1 sends every call to the FMA kernels.  A call that fails only the
    alignment test runs on the FMA kernel, whose bound the split rule contains.
  - gemm_tn adds its partial sums with fp32 atomics (train_ops.cu:74, gemm_tn_tc.cu:144-145) into the zeroed gradient:
    n grows by M / 1024 + 2, the most reduction splits either kernel makes plus the store.
  - A bias joins the sum as one more term (n + 1).
* BatchNorm forward over the M rows of column c (train_ops.cu col_reduce_kernel<0>, bn_finalize_kernel,
  bn_apply_kernel), zc = z - mu, s = 1 / sqrt(var + eps), xh = zc s:
      e_mu = sum e_z / M (linear: the rows' errors share a common-mode part, which the mean keeps; a quadrature mean
      put the fp32 step's running mean at 1.24 times the check), e_var^2 = (2 / M)^2 sum zc^2 e_z^2 (a common shift
      leaves the variance alone),
      e_xh^2 = s^2 (e_z^2 + sum e_z^2 / M^2) + (xh s^2 e_var / 2)^2,
      e_y^2 = gamma^2 e_xh^2 + local^2,  local = train_prims_bound.bn_apply_true's bound (fp32 statistics + apply).
  Running statistics (bn_finalize_kernel): e_rm^2 = (m e_mu)^2 + brm^2, e_rv^2 = (m M / (M - 1) e_var)^2 + brv^2 with
  brm, brv from train_prims_bound.running_exact_and_bound.  ReLU multiplies v and e by the step's mask; the max over
  points gathers v and e at the step's arg (bn_maxpool_fwd computes the same y only at the arg rows).
* BatchNorm backward (col_reduce_kernel<1>, bn_bwd_apply_kernel; the fused max-pool form with the sparse g of the
  arg rows), g = dy mask, S1 = sum g, S2 = sum g xh:
      dz = gamma s (g - S1 / M - xh S2 / M)
      e_dz^2 = (gamma s)^2 (e_g^2 + sum e_g^2 / M^2 + xh^2 sum xh^2 e_g^2 / M^2 + e_xh^2 (S2 / M)^2
               + xh^2 sum g^2 e_xh^2 / M^2) + (dz s^2 e_var / 2)^2 + bdz^2
      e_dgamma^2 = sum (xh^2 e_g^2 + g^2 e_xh^2) + bdg^2,   e_dbeta^2 = sum e_g^2 + bdb^2
  with bdz, bdg, bdb the local bounds of train_prims_bound.bn_backward_exact (its docstring gives their derivation).
  Two parts of e_dz are shared by every row of a column: c1 = |gamma s| (sqrt(sum e_g^2) + bdb) / M, the error of
  m1 = S1 / M, and xh c2 with c2 = |gamma s| (sqrt(sum (xh^2 e_g^2 + g^2 e_xh^2)) + bdg) / M, the error of m2 = S2 / M.
  The weight gradient dW = dz^T x sums them over the rows coherently, so it adds
      (c1 sum_rows |x|)^2 + (c2 sum_rows |xh| |x|)^2
  to the GEMM rule (in quadrature alone, the fp32 steps' conv3 weight gradients reached 1.7 to 2.5 times the check at
  132 000 rows).  For the same reason the running variance takes e_var linearly, 2 / M sum |zc| e_z.
* col_sum of dz (the bias of a layer without BatchNorm: fc3, fc4): e^2 = sum e_dz^2 + (u |S| + gamma64_M sum |dz|)^2.
* axpy_ (train_ops.cu:427-430 axpy_kernel, one fmaf) of two values with errors: e^2 = e_1^2 + e_2^2 + (u |v|)^2.
  Into a zeroed gradient it is exact and adds nothing.
* T = fc3 + I (add_row_kernel, train_ops.cu:411-414): e^2 = e^2 + (u |T|)^2.  center (center_kernel): e = u |v|.
* Quaternion (quat_to_rot_kernel, quat_to_rot_bwd_kernel), q = q4 + (1, 0, 0, 0) with e_q0^2 = e_q40^2 + (u |q0|)^2,
  R = I + s A(q), s = 2 / |q|^2, dR/dq_k = s dA/dq_k - s^2 q_k A:
      e_R^2 = sum_k (dR/dq_k e_qk)^2 + bR^2,
      e_dq^2 = sum_ij (dR_ij/dq_k)^2 e_gij^2 + sum_l (d dq_k / dq_l e_ql)^2 + bdq^2
  with bR, bdq from train_prims_bound.quat_to_rot_exact / quat_to_rot_bwd_exact and the second derivatives by autograd.
* Losses (loss_kernel, loss_distance_kernel): the local bounds of train_prims_bound.loss_exact / loss_distance_exact,
  plus the response to the logits' error: dL0/dp0 = dpred0, dL1/dp1 = dpred1, d dpred0 / dp0 = 2 w / B (F^2 - 2 a d F)
  (a = tanh(sign p0), F = 1 - a^2, d = a - tanh|t|; the same with a = tanh p for the distance loss), d dpred1 / dp1 =
  w / B sig (1 - sig).
* SGD (sgd_kernel: buf = fmaf(mu, buf, g), p = fmaf(-lr, buf, p)), lr and mu as the kernel receives them (fp32):
      e_buf^2 = e_g^2 + (u (|mu buf_old| + |buf|))^2,   e_p^2 = (lr e_buf)^2 + (u (|lr buf| + |p'|))^2
  (two roundings each, so that the torch stand-in's separate multiply and add are covered too).
"""
import numpy as np
import torch

from oracle import net_bound as nb
from oracle.net_bound import LAMBDA, V  # noqa: F401  (re-exported with the check below)
from oracle.split_gemm import C2
import train_prims_bound as tpb

U = 2.0 ** -24
UTC = 2.0 ** -23
RHO_SPLIT = 3 * 2.0 ** -22
EPS, BN_MOM = 1e-5, 0.1


def f32(x):
    return float(np.float32(x))


class Arith:
    """Which GEMM kernel a call reaches: fp32_only models P2S_TRAIN_GEMM_FP32=1 (or the torch stand-in on the CPU)."""

    def __init__(self, fp32_only):
        self.fp32_only = bool(fp32_only)

    def nt(self, M, N, K, Z):
        tc = (not self.fp32_only and Z == 1 and N % 4 == 0 and 64 <= N <= 4096 and K % 32 == 0 and K >= 32 and M >= 128)
        return ('split' if tc else 'fp32'), 0

    def tn(self, M, N, K, Z):
        tc = not self.fp32_only and Z == 1 and M >= 4096 and N >= 64 and K >= 64 and N % 4 == 0 and K % 4 == 0
        return ('split' if tc else 'fp32'), M // 1024 + 2


def _sq(x):
    return x * x


def _mm(a, b, arith, bias=None):
    """a.v [..., M, K] @ b.v [..., K, N] (+ bias [N]) with the GEMM rule of the docstring; a.e / b.e may be None."""
    kind, extra = arith
    K = a.v.shape[-1]
    aa = a.v.abs() if a.e is None else a.v.abs() + a.e
    ab = b.v.abs() if b.e is None else b.v.abs() + b.e
    v = a.v @ b.v
    mag2 = _sq(aa) @ _sq(ab)
    var = torch.zeros_like(v)
    if a.e is not None:
        var += _sq(a.e) @ _sq(b.v)
    if b.e is not None:
        var += _sq(aa) @ _sq(b.e)
    if kind == 'split':
        rho, n, u = RHO_SPLIT, 3 * K + extra, UTC
    else:
        rho, n, u = 0.0, K + extra, U
    if bias is not None:
        v += bias
        mag2 += _sq(bias)
        n += 1
    var += rho * rho * mag2 + n * (u * (1 + 2.0 ** -9)) ** 2 * (mag2 + _sq(v))
    del mag2
    if kind == 'split':
        ma, mb = aa.amax(-1, keepdim=True), ab.amax(-2, keepdim=True)
        var += _sq(C2 * K * ma * mb)
    return V(v, var.sqrt_())


def _T(x):
    return V(x.v.transpose(-1, -2), None if x.e is None else x.e.transpose(-1, -2))


def _view(x, *shape):
    return V(x.v.reshape(*shape), None if x.e is None else x.e.reshape(*shape))


def _add(x, y):
    """axpy_ of two values with errors: one fp32 rounding."""
    v = x.v + y.v
    return V(v, (_sq(x.e) + _sq(y.e) + _sq(U * v.abs())).sqrt())


class _Rec:
    __slots__ = ('name', 'bn', 'x', 'xh', 'st', 'mask', 'pool', 'M')


class BoundStep:
    """One conditioned float64 step.  `state`: dict(params, mom, buffers, steps_done) of fp32 tensors (the step's state
    before the iteration); `dec`: `decisions(...)`.  cfg keys: use_point_stn, shared, P, S, net, output_dim, lr,
    momentum, loss_weights, fixed_radius; bn_eps / bn_momentum (EPS / BN_MOM, or their fp32 values for the fp32 step)."""

    def __init__(self, cfg, arith, state, dec, device):
        self.c, self.ar, self.dec, self.dev = cfg, arith, dec, device
        self.params = {k: t.detach().to(device, torch.float64) for k, t in state['params'].items()}
        self.mom = {k: t.detach().to(device, torch.float64) for k, t in state['mom'].items()}
        self.buf = {k: t.detach().to(device, torch.float64) for k, t in state['buffers'].items()
                    if not k.endswith('num_batches_tracked')}
        self.first = state['steps_done'] == 0
        self.grads, self.out_buf = {}, {}

    # ------------------------------------------------------------------ units
    def _bn_fwd(self, z, bn, rec):
        c = self.c
        M = z.v.shape[0]
        eps = c['bn_eps']
        gamma, beta = self.params[bn + '.weight'], self.params[bn + '.bias']
        st = tpb.col_stats_exact(z.v, eps)
        st['var'] = st['var'].clone()
        mu, var = st['mean'], st['var']
        s = 1.0 / torch.sqrt(var + eps)
        zc = z.v - mu
        # the rows' errors share a common-mode part (the upstream statistics shift a whole column), which the running
        # mean keeps (linear sum e_mu) and the variance, a sum of zc^2 with sum zc = 0, cancels (quadrature); inside
        # xh the mean enters per row like any other term of the sum (quadrature e_mu_q)
        e_mu = z.e.sum(0) / M
        e_mu_q = _sq(z.e).sum(0).sqrt() / M
        e_var = 2.0 / M * (_sq(zc) * _sq(z.e)).sum(0).sqrt()
        e_var_lin = 2.0 / M * (zc.abs() * z.e).sum(0)         # the running variance keeps the common-mode scale part
        xh = zc * s
        e_xh = (_sq(s) * (_sq(z.e) + _sq(e_mu_q)) + _sq(0.5 * xh * _sq(s) * e_var)).sqrt()
        st['invstd'] = s
        rec.xh, rec.st, rec.M = V(xh, e_xh), dict(st, e_mu=e_mu, e_var=e_var), M
        # running statistics
        m = c['bn_momentum']
        f = M / (M - 1) if M > 1 else 1.0
        rm, rv = self.buf[bn + '.running_mean'], self.buf[bn + '.running_var']
        _, _, brm, brv = tpb.running_exact_and_bound(st, rm, rv, m)
        rm2 = (1 - m) * rm + m * mu
        rv2 = (1 - m) * rv + m * var * f
        self.out_buf[bn + '.running_mean'] = V(rm2, (_sq(m * e_mu) + _sq(brm)).sqrt())
        self.out_buf[bn + '.running_var'] = V(rv2, (_sq(m * f * e_var_lin) + _sq(brv)).sqrt())
        return gamma, beta, st

    def _apply(self, xh, z, gamma, beta, st):
        """y = gamma xh + beta on (a gather of) the rows, with its error scale."""
        y = gamma * xh.v + beta
        _, loc = tpb.bn_apply_true(z, st, gamma, beta, False, self.c['bn_eps'])
        return V(y, (_sq(gamma) * _sq(xh.e) + _sq(loc)).sqrt())

    def _lin(self, tape, x, name, bn, relu):
        W, b = self.params[name + '.weight'], self.params[name + '.bias']
        M, K = x.v.shape
        z = _mm(x, V(W.t(), None), self.ar.nt(M, W.shape[0], K, 1), bias=b)
        r = _Rec()
        r.name, r.bn, r.x, r.pool, r.mask = name, bn, x, None, None
        tape.append(r)
        if bn is None:
            r.xh = None
            return z
        gamma, beta, st = self._bn_fwd(z, bn, r)
        y = self._apply(r.xh, z.v, gamma, beta, st)
        if relu:
            r.mask = self.dec[name].to(y.v.dtype)
            y = V(y.v * r.mask, y.e * r.mask)
        return y

    def _lin_pool(self, tape, x, name, bn, relu, B, n):
        W, b = self.params[name + '.weight'], self.params[name + '.bias']
        M, K = x.v.shape
        z = _mm(x, V(W.t(), None), self.ar.nt(M, W.shape[0], K, 1), bias=b)
        r = _Rec()
        r.name, r.bn, r.x, r.mask = name, bn, x, None
        tape.append(r)
        gamma, beta, st = self._bn_fwd(z, bn, r)
        del z
        arg, pos = self.dec[name]
        C = arg.shape[1]
        idx = arg.unsqueeze(1)

        def g(t):
            return t.view(B, n, C).gather(1, idx).squeeze(1)

        xg = V(g(r.xh.v), g(r.xh.e))
        zg = xg.v / st['invstd'] + st['mean']              # z at the arg rows (for the local bound only)
        out = self._apply(xg, zg, gamma, beta, st)
        if relu:
            pm = pos.to(out.v.dtype)
            out = V(out.v * pm, out.e * pm)
        r.pool = (arg, pos, B, n)
        return out

    def _bn_bwd(self, r, g, eg):
        """Dense masked dy (g, eg) [M, C] -> dz V, dgamma V, dbeta V."""
        M, st = r.M, r.st
        xh, exh = r.xh.v, r.xh.e
        s = st['invstd']
        gamma = self.params[r.bn + '.weight']
        gi = gamma * s
        S1, S2 = g.sum(0), (g * xh).sum(0)
        A1, A2 = g.abs().sum(0), (g * xh).abs().sum(0)
        dz = gi * (g - S1 / M - xh * (S2 / M))
        eg2 = _sq(eg)
        E1, E2, E3 = eg2.sum(0), (_sq(xh) * eg2).sum(0), (_sq(g) * _sq(exh)).sum(0)
        T = g.abs() + S1.abs() / M + xh.abs() * S2.abs() / M
        bdz = gi.abs() * (8 * U * T + 2.2 * U * xh.abs() * A2 / M + 2 * tpb.gamma64(M + 2) * A1 / M)
        var = _sq(gi) * (eg2 + E1 / M ** 2 + _sq(xh) * E2 / M ** 2 + _sq(exh) * _sq(S2 / M) + _sq(xh) * E3 / M ** 2)
        var += _sq(dz * 0.5 * _sq(s) * st['e_var']) + _sq(bdz)
        del T, bdz
        bdb = U * S1.abs() + tpb.gamma64(M + 1) * A1
        bdg = U * S2.abs() + 2.1 * U * A2 + tpb.gamma64(M + 2) * A2
        dgamma = V(S2, (E2 + E3 + _sq(bdg)).sqrt())
        dbeta = V(S1, (E1 + _sq(bdb)).sqrt())
        dz = V(dz, var.sqrt_())
        # the parts of dz's error every row shares: the errors of m1 = S1 / M (the same for all rows) and of m2 = S2 / M
        # (times xh); a reduction over the rows adds them linearly (see _lin_bwd)
        dz.common = (gi.abs() * (E1.sqrt() + bdb) / M, gi.abs() * ((E2 + E3).sqrt() + bdg) / M, xh)
        return dz, dgamma, dbeta

    def _lin_bwd(self, r, dy, need_dx=True):
        name = r.name
        if r.pool is not None:
            arg, pos, B, n = r.pool
            C = arg.shape[1]
            dv, de = dy.v, dy.e
            if pos is not None:
                pm = pos.to(dv.dtype)
                dv, de = dv * pm, de * pm
            g = torch.zeros(B, n, C, dtype=dv.dtype, device=dv.device)
            g.scatter_(1, arg.unsqueeze(1), dv.unsqueeze(1))
            eg = torch.zeros_like(g)
            eg.scatter_(1, arg.unsqueeze(1), de.unsqueeze(1))
            dz, dgam, dbet = self._bn_bwd(r, g.view(B * n, C), eg.view(B * n, C))
            del g, eg
        elif r.bn is not None:
            m = r.mask if r.mask is not None else 1.0
            dz, dgam, dbet = self._bn_bwd(r, dy.v * m, dy.e * m)
        else:
            dz = dy
        if r.bn is not None:
            self.grads[r.bn + '.weight'], self.grads[r.bn + '.bias'] = dgam, dbet
            self.grads[name + '.bias'] = V(torch.zeros_like(self.params[name + '.bias']), None)
        else:
            S = dz.v.sum(0)
            loc = U * S.abs() + tpb.gamma64(dz.v.shape[0]) * dz.v.abs().sum(0)
            self.grads[name + '.bias'] = V(S, (_sq(dz.e).sum(0) + _sq(loc)).sqrt())
        M, N = dz.v.shape
        K = r.x.v.shape[1]
        dW = _mm(_T(dz), r.x, self.ar.tn(M, N, K, 1))
        common = getattr(dz, 'common', None)
        if common is not None:
            c1, c2, xh = common
            ax = r.x.v.abs() if r.x.e is None else r.x.v.abs() + r.x.e
            extra = _sq(c1.unsqueeze(1) * ax.sum(0).unsqueeze(0)) + _sq(c2.unsqueeze(1) * (xh.abs().t() @ ax))
            dW = V(dW.v, (_sq(dW.e) + extra).sqrt())
        self.grads[name + '.weight'] = dW
        if not need_dx:
            return None
        W = self.params[name + '.weight']
        return _mm(dz, V(W, None), self.ar.nt(M, K, N, 1))

    def _stn_fwd(self, prefix, x, B, n):
        tape = []
        h = self._lin(tape, x, prefix + 'conv1', prefix + 'bn1', True)
        h = self._lin(tape, h, prefix + 'conv2', prefix + 'bn2', True)
        g = self._lin_pool(tape, h, prefix + 'conv3', prefix + 'bn3', True, B, n)
        f = self._lin(tape, g, prefix + 'fc1', prefix + 'bn4', True)
        f = self._lin(tape, f, prefix + 'fc2', prefix + 'bn5', True)
        return self._lin(tape, f, prefix + 'fc3', None, False), tape

    def _stn_bwd(self, tape, dout, need_dx):
        d = dout
        for r in tape[:0:-1]:
            d = self._lin_bwd(r, d)
        return self._lin_bwd(tape[0], d, need_dx)

    def _feat_fwd(self, prefix, pts, B, n):
        tape = []
        a = self._lin(tape, _view(pts, B * n, 3), prefix + 'conv0a', prefix + 'bn0a', True)
        hb = self._lin(tape, a, prefix + 'conv0b', prefix + 'bn0b', True)
        traw, stn = self._stn_fwd(prefix + 'stn2.', hb, B, n)
        Tv = traw.v + torch.eye(64, dtype=torch.float64, device=self.dev).reshape(1, -1)
        T = V(Tv.view(B, 64, 64), (_sq(traw.e) + _sq(U * Tv.abs())).sqrt().view(B, 64, 64))
        ht = _view(_mm(_view(hb, B, n, 64), _T(T), self.ar.nt(n, 64, 64, B)), B * n, 64)
        h = self._lin(tape, ht, prefix + 'conv1', prefix + 'bn1', True)
        h = self._lin(tape, h, prefix + 'conv2', prefix + 'bn2', True)
        g = self._lin_pool(tape, h, prefix + 'conv3', prefix + 'bn3', False, B, n)
        return g, (tape, stn, T, hb, B, n)

    def _feat_bwd(self, ctx, dg, need_dpts):
        tape, stn, T, hb, B, n = ctx
        d = self._lin_bwd(tape[4], dg)
        d = self._lin_bwd(tape[3], d)
        dht = _view(self._lin_bwd(tape[2], d), B, n, 64)
        dhb = _view(_mm(dht, T, self.ar.nt(n, 64, 64, B)), B * n, 64)
        dT = _view(_mm(_T(dht), _view(hb, B, n, 64), self.ar.tn(n, 64, 64, B)), B, 64 * 64)
        dhb = _add(dhb, self._stn_bwd(stn, dT, True))
        d = self._lin_bwd(tape[1], dhb)
        return self._lin_bwd(tape[0], d, need_dpts)

    # ------------------------------------------------------------------ quaternion
    @staticmethod
    def _R_and_J(q):
        s = 2.0 / (q * q).sum(1, keepdim=True)
        A, _ = tpb._A_and_abs(q)
        R = s * A + torch.eye(3, dtype=q.dtype, device=q.device).reshape(1, 9)
        J = s.unsqueeze(1) * tpb._dA(q) - (s * s).unsqueeze(1) * q.unsqueeze(2) * A.unsqueeze(1)     # [B, 4, 9]
        return R, J

    def _quat(self, q4):
        one = torch.tensor([1.0, 0.0, 0.0, 0.0], dtype=torch.float64, device=self.dev)
        q = q4.v + one
        eq = q4.e.clone()
        eq[:, 0] = (_sq(eq[:, 0]) + _sq(U * q[:, 0].abs())).sqrt()
        R, J = self._R_and_J(q)
        _, bR = tpb.quat_to_rot_exact(q4.v)
        eR = ((_sq(J) * _sq(eq).unsqueeze(2)).sum(1) + _sq(bR)).sqrt()
        return V(R.view(-1, 3, 3), eR.view(-1, 3, 3)), q, eq

    def _quat_bwd(self, q, eq, q4v, dR):
        g = dR.v.reshape(-1, 9)
        eg = dR.e.reshape(-1, 9)
        qq = q.detach().clone().requires_grad_(True)
        with torch.enable_grad():
            _, J = self._R_and_J(qq)
            dq = (J * g.unsqueeze(1)).sum(2)
            H = torch.stack([torch.autograd.grad(dq[:, k].sum(), qq, retain_graph=k < 3)[0] for k in range(4)], 1)
        dq, J = dq.detach(), J.detach()
        _, bdq = tpb.quat_to_rot_bwd_exact(q4v, g)
        var = (_sq(J) * _sq(eg).unsqueeze(1)).sum(2) + (_sq(H) * _sq(eq).unsqueeze(1)).sum(2) + _sq(bdq)
        return V(dq, var.sqrt())

    # ------------------------------------------------------------------ loss
    def _loss(self, logits, batch):
        c = self.c
        B = logits.v.shape[0]
        radius = batch['patch_radius_ms'].reshape(-1).double().to(self.dev)
        if c['output_dim'] == 1:
            t = batch['imp_surf_ms'].reshape(-1).double().to(self.dev)
            w = f32(c['loss_weights']['imp_surf'])
            L, bL, _, bdp = tpb.loss_distance_exact(logits.v, t, radius, w, c['fixed_radius'])
            p, ep = logits.v[:, 0], logits.e[:, 0]
            tt = t if c['fixed_radius'] else t / radius
            a, b = torch.tanh(p), torch.tanh(tt)
            d, F = a - b, 1 - a * a
            L = (w * (d * d).sum() / B).reshape(1)
            dp = 2 * w * d * F / B
            eL = ((_sq(dp * ep)).sum() + _sq(bL[0])).sqrt().reshape(1)
            edp = (_sq(2 * w / B * (F * F - 2 * a * d * F) * ep) + _sq(bdp[:, 0])).sqrt()
            return V(L, eL), V(dp.reshape(-1, 1), edp.reshape(-1, 1))
        tm = batch['imp_surf_magnitude_ms'].reshape(-1).double().to(self.dev)
        sgn_t = batch['imp_surf_dist_sign_ms'].reshape(-1).double().to(self.dev)
        wm, ws = f32(c['loss_weights']['imp_surf_magnitude']), f32(c['loss_weights']['imp_surf_sign'])
        _, bL, _, bdp = tpb.loss_exact(logits.v, tm, radius, sgn_t, wm, ws, c['fixed_radius'])
        p0, p1 = logits.v[:, 0], logits.v[:, 1]
        e0, e1 = logits.e[:, 0], logits.e[:, 1]
        sg = self.dec['sign_p0'].to(torch.float64)
        tt = tm if c['fixed_radius'] else tm / radius
        a, b = torch.tanh(sg * p0), torch.tanh(tt.abs())
        d, F = a - b, 1 - a * a
        l1 = torch.clamp_min(p1, 0) - p1 * sgn_t + torch.log1p(torch.exp(-p1.abs()))
        L = torch.stack([wm * (d * d).sum() / B, ws * l1.sum() / B])
        dp0 = 2 * wm * d * F * sg / B
        sig = torch.sigmoid(p1)
        dp1 = ws * (sig - sgn_t) / B
        eL = torch.stack([(_sq(dp0 * e0).sum() + _sq(bL[0])).sqrt(), (_sq(dp1 * e1).sum() + _sq(bL[1])).sqrt()])
        ed0 = (_sq(2 * wm / B * (F * F - 2 * a * d * F) * sg * e0) + _sq(bdp[:, 0])).sqrt()
        ed1 = (_sq(ws / B * sig * (1 - sig) * e1) + _sq(bdp[:, 1])).sqrt()
        return V(L, eL), V(torch.stack([dp0, dp1], 1), torch.stack([ed0, ed1], 1))

    # ------------------------------------------------------------------ the step
    def run(self, batch):
        c, dev = self.c, self.dev
        patch = batch['patch_pts_ps'].to(dev).double()
        B = patch.shape[0]
        sub_v = batch['pts_sub_sample_ms'].to(dev).double() - batch['imp_surf_query_point_ms'].to(dev).double().unsqueeze(1)
        sub = V(sub_v, U * sub_v.abs())
        P, S = c['P'], c['S']
        rot = None
        if c['use_point_stn']:
            if c['shared']:
                allp = V(torch.cat((patch, sub.v), 1), torch.cat((torch.zeros_like(patch), sub.e), 1))
                q4, qtape = self._stn_fwd('point_stn.', _view(allp, B * (P + S), 3), B, P + S)
            else:
                q4, qtape = self._stn_fwd('feat_global.stn1.', _view(sub, B * S, 3), B, S)
            R, q, eq = self._quat(q4)
            rot = (R, q, eq, q4, qtape)
            sub_t = _mm(sub, _T(R), self.ar.nt(S, 3, 3, B))
            patch_t = _mm(V(patch, None), _T(R), self.ar.nt(P, 3, 3, B))
        else:
            sub_t, patch_t = sub, V(patch, None)
        g_glob, fg = self._feat_fwd('feat_global.', sub_t, B, S)
        head = []
        f_glob = self._lin(head, g_glob, 'fc1_global', 'bn1_global', True)
        g_loc, fl = self._feat_fwd('feat_local.', patch_t, B, P)
        f_loc = self._lin(head, g_loc, 'fc1_local', 'bn1_local', True)
        x = V(torch.cat((f_loc.v, f_glob.v), 1), torch.cat((f_loc.e, f_glob.e), 1))
        x = self._lin(head, x, 'fc2', 'bn2', True)
        x = self._lin(head, x, 'fc3', 'bn3', True)
        logits = self._lin(head, x, 'fc4', None, False)
        losses, dlogits = self._loss(logits, batch)
        # backward
        d = self._lin_bwd(head[4], dlogits)
        d = self._lin_bwd(head[3], d)
        d = self._lin_bwd(head[2], d)
        half = c['net'] // 2
        d_loc, d_glob = V(d.v[:, :half], d.e[:, :half]), V(d.v[:, half:], d.e[:, half:])
        need_R = rot is not None
        dpatch_t = self._feat_bwd(fl, self._lin_bwd(head[1], d_loc), need_R)
        dsub_t = self._feat_bwd(fg, self._lin_bwd(head[0], d_glob), need_R)
        del fl, fg
        if need_R:
            R, q, eq, q4, qtape = rot
            dR = _mm(_T(_view(dsub_t, B, S, 3)), sub, self.ar.tn(S, 3, 3, B))
            dR = _add(dR, _mm(_T(_view(dpatch_t, B, P, 3)), V(patch, None), self.ar.tn(P, 3, 3, B)))
            dq = self._quat_bwd(q, eq, q4.v, dR)
            self._stn_bwd(qtape, dq, False)
        # SGD
        lr, mu = c['lr'], c['momentum']
        new_p, new_m = {}, {}
        for k, p in self.params.items():
            g = self.grads[k]
            ge = g.e if g.e is not None else torch.zeros_like(g.v)
            old = self.mom[k]
            buf = g.v.clone() if self.first else mu * old + g.v
            eb = (_sq(ge) + _sq(U * ((0.0 if self.first else mu * old.abs()) + buf.abs()))).sqrt()
            p2 = p - lr * buf
            new_m[k] = V(buf, eb)
            new_p[k] = V(p2, (_sq(lr * eb) + _sq(U * ((lr * buf).abs() + p2.abs()))).sqrt())
        return dict(logits=logits, losses=losses, grads=self.grads, params=new_p, mom=new_m, buffers=self.out_buf)


# ---------------------------------------------------------------------------------------------- driving a TrainStep
def config(ts, exact_scalars=False):
    """The BoundStep configuration of TrainStep `ts`; exact_scalars keeps lr, momenta and eps as the float64 step uses
    them (the consistency check), else they are the fp32 values the kernels receive."""
    cv = (lambda x: float(x)) if exact_scalars else f32
    return dict(use_point_stn=ts.use_point_stn, shared=ts.shared, P=ts.P, S=ts.S, net=ts.net, output_dim=ts.output_dim,
                lr=cv(ts.lr), momentum=cv(ts.momentum), loss_weights=dict(ts.loss_weights), fixed_radius=ts.fixed_radius,
                bn_eps=cv(EPS), bn_momentum=cv(BN_MOM))


def state_of(ts):
    """(params, momentum buffers, BatchNorm buffers, steps_done) of `ts`, cloned, momentum per parameter name."""
    mom, off = {}, 0
    for k, t in ts.params.items():
        n = t.numel()
        mom[k] = ts.flat_mom[off:off + n].view(t.shape).detach().clone()
        off += n
    return dict(params={k: t.detach().clone() for k, t in ts.params.items()}, mom=mom,
                buffers={k: t.detach().clone() for k, t in ts.buffers.items()}, steps_done=ts.steps_done)


def decisions(rec, logits):
    """name -> the step's decision, read from TrainStep's tapes (`ts._rec`, before backward clears it): the ReLU mask
    (y > 0) of a non-pooled layer, (arg, out > 0 or None) of a fused BN + max-pool; 'sign_p0': sign of the step's p0."""
    tapes = list(rec['head'])
    if rec.get('qstn') is not None:
        tapes += rec['qstn']
    for k in ('feat_global', 'feat_local'):
        tapes += rec[k][0] + rec[k][1]
    dec = {}
    for t in tapes:
        if t.pool is not None:
            out, arg = t.pool[0], t.pool[1]
            dec[t.name] = (arg.long().clone(), (out > 0).clone() if t.relu else None)
        elif t.relu:
            dec[t.name] = (t.y_mask > 0).clone()
    dec['sign_p0'] = torch.sign(logits[:, 0]).clone()
    return dec


def drive(ts, batch):
    """One iteration of `ts` exactly as `_forward_backward` + `optimizer_step`, keeping what the check needs:
    -> dict(before, dec, logits, losses, grads, after)."""
    from points2surf_b200.train import compute_loss
    before = state_of(ts)
    ts.zero_grad()
    logits = ts.forward(batch)
    losses, dlogits = compute_loss(logits, batch, ts.outputs, ts.loss_weights, ts.fixed_radius, prims=ts.p, need_grad=True)
    dec = decisions(ts._rec, logits)
    ts.backward(dlogits)
    grads = {k: g.detach().clone() for k, g in ts.grads.items()}
    ts.optimizer_step()
    return dict(before=before, dec=dec, logits=logits.detach().clone(), losses=torch.stack([l.reshape(()) for l in losses]),
                grads=grads, after=state_of(ts))


def reference(ts, run, batch, fp32_only, device=None, exact_scalars=False):
    """The conditioned float64 step (dict of V) for one `drive` record."""
    device = device if device is not None else run['logits'].device
    cfg = config(ts, exact_scalars)
    dec = {k: (tuple(x.to(device) if x is not None else None for x in v) if isinstance(v, tuple) else v.to(device))
           for k, v in run['dec'].items()}
    return BoundStep(cfg, Arith(fp32_only), run['before'], dec, device).run(batch)


def checks(ts, run, ref):
    """[(tensor name, got fp32 tensor, V)] in layer order: logits, losses, gradients, parameters, momentum buffers,
    running statistics."""
    out = [('logits', run['logits'], ref['logits']), ('losses', run['losses'], ref['losses'])]
    out += [('grad ' + k, run['grads'][k], ref['grads'][k]) for k in ts.grads]
    out += [('param ' + k, run['after']['params'][k], ref['params'][k]) for k in ts.params]
    out += [('mom ' + k, run['after']['mom'][k], ref['mom'][k]) for k in ts.params]
    out += [(k, run['after']['buffers'][k], ref['buffers'][k]) for k in ts.buffers if not k.endswith('num_batches_tracked')]
    return out


def ratios(items):
    """[(name, worst ratio, index)] with the ratio |x - v| / (LAMBDA e) (0 where exact, inf where e = 0 and x != v)."""
    res = []
    for name, got, ref in items:
        e = ref.e if ref.e is not None else torch.zeros_like(ref.v)
        r = nb.excess(got.reshape(ref.v.shape), V(ref.v, e))
        r = torch.nan_to_num(r, nan=float('inf'))
        res.append((name,) + nb.worst(r) if r.numel() else (name, 0.0, ()))
    return res


def width_medians(items):
    """name -> median of LAMBDA e / |v| over the elements with v != 0 (how wide the check is)."""
    out = {}
    for name, _, ref in items:
        if ref.e is None:
            continue
        nz = ref.v != 0
        if int(nz.sum()) == 0:
            continue
        out[name] = float((LAMBDA * ref.e[nz] / ref.v[nz].abs()).median())
    return out


def num_batches_tracked_ok(run):
    return all(int(run['after']['buffers'][k]) == int(run['before']['buffers'][k]) + 1
               for k in run['before']['buffers'] if k.endswith('num_batches_tracked'))
