"""Float64 restatement of points2surf_b200.train.EvalGrad (the eval-mode backward behind PointsToSurfModel's autograd),
conditioned on the fp32 recompute's own ReLU masks and max-pool arg-maxes, with a per-element error scale for the fp32
run next to every value: an eval-mode subclass of train_step_bound.BoundStep, checked like the training step,
|x - v| <= LAMBDA e (LAMBDA = 4).

What changes against the train-mode BoundStep (its docstring gives the GEMM, quaternion, add and col_sum rules, which
are reused unchanged):
* BatchNorm uses the running statistics, constants of the network: mu = running_mean (exact), s = 1 / sqrt(running_var
  + 1e-5) exact in the reference.  The fp32 run's invstd = rsqrt(running_var + eps) in fp32 is within 6u s (the sum's
  rounding and a 2-ulp rsqrt).  xh = (z - mu) s carries the propagated e_xh = s e_z; every use of xh adds its rounding
  locally: LOC = 10u relative to |gamma xh| (gamma invstd, the invstd error, z - mu, the product, and a separate
  multiply + add in the torch stand-in), plus u |y| for the final rounding of y.
* Eval BatchNorm backward (bn_eval_bwd_kernel), g = dy mask:
      dz = gamma s g,                e_dz^2 = (gamma s e_g)^2 + (LOC |dz|)^2
      dgamma = sum g xh,             e^2 = sum (xh^2 e_g^2 + g^2 e_xh^2) + (LOC sum |g xh| + u |dgamma|)^2
      dbeta = sum g,                 e^2 = sum e_g^2 + (u |dbeta|)^2
      dbias = sum dz,                e^2 = sum (gamma s e_g)^2 + (LOC sum |dz| + u |dbias|)^2
  (f64 sums of fp32 terms: their own rounding is below gamma64(M) sum |.|, added too).  The invstd error is the same
  for every row of a column, so the weight gradient dW = dz^T x adds LOC |dz|^T |x| linearly to the GEMM rule.
* Pooled conv3 layers (bn_maxpool_eval_bwd_w_kernel / _x_kernel): only the arg row of each (query, channel) carries
  dz[b,c] = gamma s dout[b,c] (0 where the pooled value is not > 0 under ReLU).  The weight gradient is the gather
  sum_b dz[b,c] x[b n + arg, :] in fp32 with ranges of queries added by fp32 atomics,
      e^2 = sum_b (e_dz^2 x^2 + dz^2 e_x^2) + ((LOC + gamma_{B + splits + 2}) sum_b |dz| |x|)^2,
  the input gradient the scatter dx[b n + i, :] = sum_{c: arg = i} dz[b,c] W[c,:] over the t channels of that point,
      e^2 = sum_c e_dz^2 W^2 + ((LOC + gamma_{t + 2}) sum_c |dz| |W|)^2,
  and dgamma, dbeta, dbias as above over the B arg rows.
* Input gradients: through conv0a, the rotation (d points = d rotated points R), the QSTN's input and the centring
  (d query = -sum over the points of d sub-sample, a batched fp32 GEMM; the sign flip is exact).
The upstream gradient dlogits is exact."""
import torch

import train_step_bound as tsb
from oracle.net_bound import V
from train_prims_bound import gamma64

U = tsb.U
LOC = 10 * U
EPS = 1e-5


def _sq(x):
    return x * x


def _gam(n):
    return n * U / (1 - n * U)


class EvalBoundStep(tsb.BoundStep):
    """Conditioned float64 EvalGrad; `dec` from train_step_bound.decisions(eg._rec, logits) after eg.forward."""

    def __init__(self, cfg, arith, params, buffers, dec, device, sm_count=132):
        super().__init__(cfg, arith, dict(params=params, mom=params, buffers=buffers, steps_done=0), dec, device)
        self.splits = 8 * sm_count        # the most query ranges the fused weight-gradient kernel adds atomically

    # ------------------------------------------------------------------ eval-mode BatchNorm
    def _bn_fwd(self, z, bn, rec):
        mu = self.buf[bn + '.running_mean']
        s = 1.0 / torch.sqrt(self.buf[bn + '.running_var'] + EPS)
        xh = (z.v - mu) * s
        rec.xh, rec.st, rec.M = V(xh, s * z.e), dict(mean=mu, invstd=s), z.v.shape[0]
        return self.params[bn + '.weight'], self.params[bn + '.bias'], rec.st

    def _apply(self, xh, z, gamma, beta, st):
        gx = gamma * xh.v
        y = gx + beta
        return V(y, (_sq(gamma * xh.e) + _sq(LOC * gx.abs() + U * y.abs())).sqrt())

    def _col_grads(self, r, g, eg, xh):
        """dgamma, dbeta, dbias V and dz (value, propagated error) from the masked dy (g, eg) on rows with xh (V)."""
        gamma, s = self.params[r.bn + '.weight'], r.st['invstd']
        gi = gamma * s
        n = g.shape[0]
        dz, edz = gi * g, gi.abs() * eg
        S2, A2 = (g * xh.v).sum(0), (g * xh.v).abs().sum(0)
        S1, A1 = g.sum(0), g.abs().sum(0)
        S3, A3 = dz.sum(0), dz.abs().sum(0)
        dgamma = V(S2, ((_sq(xh.v) * _sq(eg) + _sq(g) * _sq(xh.e)).sum(0)
                        + _sq((LOC + gamma64(n)) * A2 + U * S2.abs())).sqrt())
        dbeta = V(S1, (_sq(eg).sum(0) + _sq(gamma64(n) * A1 + U * S1.abs())).sqrt())
        dbias = V(S3, (_sq(edz).sum(0) + _sq((LOC + gamma64(n)) * A3 + U * S3.abs())).sqrt())
        self.grads[r.bn + '.weight'], self.grads[r.bn + '.bias'], self.grads[r.name + '.bias'] = dgamma, dbeta, dbias
        return dz, edz

    def _lin_bwd(self, r, dy, need_dx=True):
        name = r.name
        W = self.params[name + '.weight']
        if r.pool is not None:
            arg, pos, B, n = r.pool
            C, K = W.shape
            dv, de = dy.v, dy.e
            if pos is not None:
                pm = pos.to(dv.dtype)
                dv, de = dv * pm, de * pm
            idx = arg.unsqueeze(1)
            xg = V(r.xh.v.view(B, n, C).gather(1, idx).squeeze(1), r.xh.e.view(B, n, C).gather(1, idx).squeeze(1))
            dz, edz = self._col_grads(r, dv, de, xg)                       # [B, C]
            rows = torch.arange(B, device=dv.device).view(B, 1) * n + arg  # [B, C]
            xv = r.x.v[rows]                                               # [B, C, K]
            xe = r.x.e[rows] if r.x.e is not None else torch.zeros_like(xv)
            loc = LOC + _gam(B + self.splits + 2)
            dW = torch.einsum('bc,bck->ck', dz, xv)
            mag = torch.einsum('bc,bck->ck', dz.abs(), xv.abs() + xe)
            var = torch.einsum('bc,bck->ck', _sq(edz), _sq(xv)) + torch.einsum('bc,bck->ck', _sq(dz), _sq(xe))
            self.grads[name + '.weight'] = V(dW, (var + _sq(loc * mag)).sqrt())
            del xv, xe
            if not need_dx:
                return None
            dense = torch.zeros(B * n, C, dtype=dz.dtype, device=dz.device)
            dense.scatter_(0, rows, dz)
            edense = torch.zeros_like(dense).scatter_(0, rows, edz)
            cnt = torch.zeros(B * n, dtype=dz.dtype, device=dz.device).scatter_add_(
                0, rows.reshape(-1), torch.ones(B * C, dtype=dz.dtype, device=dz.device))
            dx = dense @ W
            e = (_sq(edense) @ _sq(W) + _sq((LOC + _gam(cnt + 2)).unsqueeze(1) * (dense.abs() @ W.abs()))).sqrt()
            return V(dx, e)
        if r.bn is not None:
            m = r.mask if r.mask is not None else 1.0
            dzv, edz = self._col_grads(r, dy.v * m, dy.e * m, r.xh)
            dz = V(dzv, (_sq(edz) + _sq(LOC * dzv.abs())).sqrt())
        else:
            dz = dy
            S = dz.v.sum(0)
            loc = U * S.abs() + gamma64(dz.v.shape[0]) * dz.v.abs().sum(0)
            self.grads[name + '.bias'] = V(S, (_sq(dz.e).sum(0) + _sq(loc)).sqrt())
        M, N = dz.v.shape
        K = r.x.v.shape[1]
        dW = tsb._mm(tsb._T(dz), r.x, self.ar.tn(M, N, K, 1))
        if r.bn is not None:                                               # the invstd error is common to the rows
            ax = r.x.v.abs() if r.x.e is None else r.x.v.abs() + r.x.e
            dW = V(dW.v, (_sq(dW.e) + _sq(LOC * (dz.v.abs().t() @ ax))).sqrt())
        self.grads[name + '.weight'] = dW
        if not need_dx:
            return None
        return tsb._mm(dz, V(W, None), self.ar.nt(M, K, N, 1))

    # ------------------------------------------------------------------ forward + backward with input gradients
    def run_eval(self, batch, dlogits):
        """-> dict(logits, grads{name: V}, dpatch, dsub, dquery) for the exact upstream gradient dlogits."""
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
                q4, qtape = self._stn_fwd('point_stn.', tsb._view(allp, B * (P + S), 3), B, P + S)
            else:
                q4, qtape = self._stn_fwd('feat_global.stn1.', tsb._view(sub, B * S, 3), B, S)
            R, q, eq = self._quat(q4)
            rot = (R, q, eq, q4, qtape)
            sub_t = tsb._mm(sub, tsb._T(R), self.ar.nt(S, 3, 3, B))
            patch_t = tsb._mm(V(patch, None), tsb._T(R), self.ar.nt(P, 3, 3, B))
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
        dl = dlogits.to(dev).double()
        d = self._lin_bwd(head[4], V(dl, torch.zeros_like(dl)))
        d = self._lin_bwd(head[3], d)
        d = self._lin_bwd(head[2], d)
        half = c['net'] // 2
        d_loc, d_glob = V(d.v[:, :half], d.e[:, :half]), V(d.v[:, half:], d.e[:, half:])
        dpatch_t = tsb._view(self._feat_bwd(fl, self._lin_bwd(head[1], d_loc), True), B, P, 3)
        dsub_t = tsb._view(self._feat_bwd(fg, self._lin_bwd(head[0], d_glob), True), B, S, 3)
        if rot is not None:
            R, q, eq, q4, qtape = rot
            dR = tsb._mm(tsb._T(dsub_t), sub, self.ar.tn(S, 3, 3, B))
            dR = tsb._add(dR, tsb._mm(tsb._T(dpatch_t), V(patch, None), self.ar.tn(P, 3, 3, B)))
            dq = self._quat_bwd(q, eq, q4.v, dR)
            dsrc = self._stn_bwd(qtape, dq, True)
            dpatch = tsb._mm(dpatch_t, R, self.ar.nt(P, 3, 3, B))
            dsub = tsb._mm(dsub_t, R, self.ar.nt(S, 3, 3, B))
            if c['shared']:
                dsrc = tsb._view(dsrc, B, P + S, 3)
                dpatch = tsb._add(dpatch, V(dsrc.v[:, :P], dsrc.e[:, :P]))
                dsub = tsb._add(dsub, V(dsrc.v[:, P:], dsrc.e[:, P:]))
            else:
                dsub = tsb._add(dsub, tsb._view(dsrc, B, S, 3))
        else:
            dpatch, dsub = dpatch_t, dsub_t
        ones = V(torch.ones(B, 1, S, dtype=torch.float64, device=dev), None)
        sq = tsb._mm(ones, dsub, self.ar.tn(S, 1, 3, B))
        dquery = V(-sq.v.reshape(B, 3), sq.e.reshape(B, 3))
        return dict(logits=logits, grads=self.grads, dpatch=dpatch, dsub=dsub, dquery=dquery)


def reference(eg, dec, batch, dlogits, fp32_only, sm_count=132):
    """The conditioned float64 EvalGrad for the fp32 EvalGrad `eg` (its parameters and running statistics)."""
    dev = dlogits.device
    params = {k: t.detach().to(dev) for k, t in eg.params.items()}
    buffers = {k: t.detach().to(dev) for k, t in eg.buffers.items() if not k.endswith('num_batches_tracked')}
    dec = {k: (tuple(x.to(dev) if x is not None else None for x in v) if isinstance(v, tuple) else v.to(dev))
           for k, v in dec.items()}
    return EvalBoundStep(tsb.config(eg), tsb.Arith(fp32_only), params, buffers, dec, dev, sm_count).run_eval(batch, dlogits)


def checks(eg, got_inputs, ref):
    """[(name, got, V)]: the three input gradients, then every parameter gradient."""
    out = list(zip(('d patch', 'd sub-sample', 'd query'), got_inputs, (ref['dpatch'], ref['dsub'], ref['dquery'])))
    grads = eg.named_gradients()
    out += [('grad ' + k, eg.grads[k], ref['grads'][k]) for k in grads]
    return out
