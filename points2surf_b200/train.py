"""Training step of PointsToSurfModel on the device (SURVEY.md section 8a row a14, BASELINE config 4):
train-mode forward, `compute_loss`, backward and the SGD(momentum) update of source/points_to_surf_train.py:441-461,
406, 537-563, sequenced layer by layer over the C-ABI primitives `p2s_op_*` (csrc/train_ops.cu).  The backward pass is
written out by hand (there is no autograd on this path); tests compare every parameter gradient with torch autograd
over the reference module.

Supported configuration (the hot-path subset, see points2surf_b200/eval.py:_check_supported): sym_op 'max',
use_feat_stn 1, single_transformer 0; use_point_stn x shared_transformer in {(1,1) vanilla, (0,0) max, (1,0) uniform};
outputs either (imp_surf_magnitude, imp_surf_sign), the two-output head, or (imp_surf,), the one-output head of the
regression ablation (experiments/train_p2s_regression.sh), whose loss is sdf_nn.calc_loss_distance.  imp_surf together
with magnitude / sign (the reference's three-output default) is rejected.

Data parallel: one process per GPU; every rank runs the step on its shard of the batch, the flat gradient buffer is
averaged with one all_reduce (NCCL over NVLink) and every rank applies the same update.  BatchNorm statistics stay
per rank, like the per-replica statistics of the reference's nn.DataParallel (points_to_surf_train.py:416).
"""
import torch
import torch.distributed as dist

from . import arch
from .weights import strip_module_prefix

BN_EPS = 1e-5
BN_MOMENTUM = 0.1


def loss_columns(outputs):
    """Network outputs the loss reads: 1 for (imp_surf,), 2 for (imp_surf_magnitude, imp_surf_sign); else ValueError."""
    outputs = list(outputs)
    if 'imp_surf' in outputs:
        if 'imp_surf_magnitude' in outputs or 'imp_surf_sign' in outputs:
            raise ValueError('Unsupported outputs %s: imp_surf (regression) together with imp_surf_magnitude / imp_surf_sign'
                             % outputs)
        return 1
    if not ('imp_surf_magnitude' in outputs and 'imp_surf_sign' in outputs):
        raise ValueError('outputs must contain imp_surf_magnitude and imp_surf_sign, or imp_surf')
    return 2


def compute_loss(pred, batch_data, outputs, output_loss_weights, fixed_radius, prims=None, need_grad=False):
    """Mirror of points_to_surf_train.compute_loss (:537-563): for outputs (imp_surf_magnitude, imp_surf_sign)
    -> [loss_magnitude, loss_sign], for (imp_surf,) -> [loss_imp_surf], as 0-d float64 CUDA tensors (and
    d(sum)/dpred [B, columns] when need_grad).  The batch is not modified (the reference divides
    batch_data['imp_surf_ms'] / ['imp_surf_magnitude_ms'] by the radius in place; calc_metrics restates that)."""
    cols = loss_columns(outputs)
    if pred.dim() != 2 or pred.shape[1] != cols:
        raise ValueError('pred %s does not match outputs %s (%d column(s))' % (tuple(pred.shape), list(outputs), cols))
    if prims is None:
        from .train_ops import CudaPrims
        prims = CudaPrims()
    if cols == 1:
        # sdf_nn.calc_loss_distance: mse(tanh(pred), tanh(d / r)) with the signed tanh (points_to_surf_train.py:541-548)
        losses, dpred = prims.loss_distance(pred, batch_data['imp_surf_ms'].reshape(-1).contiguous(),
                                            batch_data['patch_radius_ms'].reshape(-1).contiguous(),
                                            output_loss_weights['imp_surf'], fixed_radius=fixed_radius, need_grad=need_grad)
        out = [losses[0]]
        return (out, dpred) if need_grad else out
    losses, dpred = prims.loss(pred, batch_data['imp_surf_magnitude_ms'].reshape(-1).contiguous(),
                               batch_data['patch_radius_ms'].reshape(-1).contiguous(),
                               batch_data['imp_surf_dist_sign_ms'].reshape(-1).contiguous(),
                               output_loss_weights['imp_surf_magnitude'], output_loss_weights['imp_surf_sign'],
                               fixed_radius=fixed_radius, need_grad=need_grad)
    out = [losses[0], losses[1]]
    return (out, dpred) if need_grad else out


class _Tape:
    """Forward records of one linear(+BN)(+ReLU)(+max over points) unit."""
    __slots__ = ('name', 'bn', 'x', 'z', 'y_mask', 'mean', 'invstd', 'pool', 'relu')


class TrainStep:
    """Holds parameters, BatchNorm buffers, gradients and momentum buffers on one device and runs SGD steps.

        ts = TrainStep(state_dict, use_point_stn=1, shared_transformer=1, lr=0.01, momentum=0.9)
        loss = ts.step(batch)          # batch: the dict the reference's DataLoader yields (CUDA tensors)
        ts.state_dict()                # reference-named tensors (loadable by PointsToSurfModel / Engine)
    """

    _momentum = True     # SGD momentum buffers (EvalGrad, which never steps, has none)

    def __init__(self, state_dict, use_point_stn, shared_transformer, points_per_patch=300, sub_sample_size=1000,
                 net_size=1024, lr=0.01, momentum=0.9, device=None, prims=None,
                 outputs=('imp_surf_magnitude', 'imp_surf_sign'), output_loss_weights=None, fixed_radius=False,
                 dtype=torch.float32):
        if prims is None:
            from .train_ops import CudaPrims
            prims = CudaPrims()
        self.p = prims
        self.dtype = dtype   # float32 on the device; float64 only with the torch test primitives (exactness checks)
        self.use_point_stn, self.shared = bool(use_point_stn), bool(shared_transformer)
        self.P, self.S, self.net = int(points_per_patch), int(sub_sample_size), int(net_size)
        self.lr, self.momentum = float(lr), float(momentum)
        self.outputs = tuple(outputs)
        self.output_dim = loss_columns(self.outputs)
        self.loss_weights = output_loss_weights or ({'imp_surf': 1.0} if self.output_dim == 1 else
                                                    {'imp_surf_magnitude': 1.0, 'imp_surf_sign': 1.0})
        self.fixed_radius = bool(fixed_radius)
        sd = strip_module_prefix(state_dict)
        if 'fc4.weight' in sd and sd['fc4.weight'].shape[0] != self.output_dim:
            raise ValueError('the state dict has a %d-output head (fc4 %s), outputs %s need %d' % (
                sd['fc4.weight'].shape[0], tuple(sd['fc4.weight'].shape), list(self.outputs), self.output_dim))
        some = next(iter(sd.values()))
        self.device = torch.device(device) if device is not None else some.device
        specs = arch.layer_specs(self.use_point_stn, self.shared, self.net, self.output_dim)
        # the batch keys the step reads (copied into the static inputs of a captured CUDA graph)
        self._batch_keys = self._INPUT_KEYS + (('imp_surf_ms',) if self.output_dim == 1 else
                                               ('imp_surf_magnitude_ms', 'imp_surf_dist_sign_ms'))
        # flat parameter / gradient / momentum buffers with per-tensor views (one all_reduce, one SGD launch)
        shapes = []
        for name, kind, cout, cin in specs:
            if kind == 'bn':
                shapes += [(name + '.weight', (cout,)), (name + '.bias', (cout,))]
            else:
                shapes += [(name + '.weight', (cout, cin)), (name + '.bias', (cout,))]
        total = sum(int(torch.Size(s).numel()) for _, s in shapes)
        self.flat_params = torch.empty(total, dtype=dtype, device=self.device)
        self.flat_grads = torch.zeros_like(self.flat_params)
        self.flat_mom = torch.zeros_like(self.flat_params) if self._momentum else None
        self.params, self.grads, self._orig_shape = {}, {}, {}
        off = 0
        for name, shp in shapes:
            n = int(torch.Size(shp).numel())
            self.params[name] = self.flat_params[off:off + n].view(shp)
            self.grads[name] = self.flat_grads[off:off + n].view(shp)
            src = sd[name]
            self._orig_shape[name] = tuple(src.shape)
            self.params[name].copy_(src.reshape(shp).to(self.device, dtype))
            off += n
        self.buffers = {}
        for name, kind, cout, _ in specs:
            if kind == 'bn':
                for b in ('running_mean', 'running_var'):
                    self.buffers[name + '.' + b] = sd[name + '.' + b].to(self.device, dtype).clone().contiguous()
                nb = sd.get(name + '.num_batches_tracked')
                # host-side counter (never read by a kernel); kept on the CPU so that it is not captured into CUDA graphs
                self.buffers[name + '.num_batches_tracked'] = (nb.detach().cpu().clone() if nb is not None
                                                               else torch.zeros((), dtype=torch.long))
        self.steps_done = 0
        self._eye64 = torch.eye(64, dtype=dtype, device=self.device).reshape(-1).contiguous()

    # ------------------------------------------------------------------------------------------ units
    def _lin(self, tape, x, name, bn, relu):
        """x [M,K] -> act(BN(x W^T + b)); records what the backward needs."""
        p = self.p
        z = p.gemm_nt(x, self.params[name + '.weight'], self.params[name + '.bias'])
        t = _Tape()
        t.name, t.bn, t.x, t.z, t.pool, t.relu = name, bn, x, z, None, relu
        if bn is not None:
            y, t.mean, t.invstd = self._bn_fwd(z, bn, relu)
            t.y_mask = y if relu else None
        else:
            if relu:
                raise ValueError('ReLU without BatchNorm does not occur in PointsToSurfModel')
            y, t.mean, t.invstd, t.y_mask = z, None, None, None
        tape.append(t)
        return y

    def _lin_pool(self, tape, x, name, bn, relu, B, n):
        """conv + BatchNorm (+ReLU) + max over the n points of each query; the normalised [B*n, C] tensor is never
        materialised (model.py:45-48, 104-107, 203-212)."""
        p = self.p
        z = p.gemm_nt(x, self.params[name + '.weight'], self.params[name + '.bias'])
        out, arg, mean, invstd = self._bn_pool_fwd(z, bn, relu, B, n)
        t = _Tape()
        t.name, t.bn, t.x, t.z, t.y_mask, t.mean, t.invstd, t.pool, t.relu = name, bn, x, z, None, mean, invstd, (out, arg, B, n), relu
        tape.append(t)
        return out

    # train-mode BatchNorm: batch statistics, running statistics updated
    def _bn_fwd(self, z, bn, relu):
        y, mean, invstd = self.p.bn_forward(z, self.params[bn + '.weight'], self.params[bn + '.bias'], relu,
                                            self.buffers[bn + '.running_mean'], self.buffers[bn + '.running_var'],
                                            BN_EPS, BN_MOMENTUM)
        self.buffers[bn + '.num_batches_tracked'] += 1
        return y, mean, invstd

    def _bn_pool_fwd(self, z, bn, relu, B, n):
        out, arg, mean, invstd = self.p.bn_maxpool_forward(z, B, n, self.params[bn + '.weight'], self.params[bn + '.bias'], relu,
                                                           self.buffers[bn + '.running_mean'],
                                                           self.buffers[bn + '.running_var'], BN_EPS, BN_MOMENTUM)
        self.buffers[bn + '.num_batches_tracked'] += 1
        return out, arg, mean, invstd

    def _bn_bwd(self, t, dy):
        """dy -> dz through act + BatchNorm; accumulates the BatchNorm's parameter gradients."""
        p = self.p
        if t.pool is not None:
            out, arg, B, n = t.pool
            dz, dgamma, dbeta = p.bn_maxpool_backward(dy, arg, out, t.z, t.mean, t.invstd, self.params[t.bn + '.weight'], t.relu, B, n)
        else:
            dz, dgamma, dbeta = p.bn_backward(dy, t.z, t.y_mask, t.mean, t.invstd, self.params[t.bn + '.weight'])
        p.axpy_(self.grads[t.bn + '.weight'], dgamma)
        p.axpy_(self.grads[t.bn + '.bias'], dbeta)
        # the bias of a layer in front of a train-mode BatchNorm has an identically zero gradient (dz sums to zero
        # over the rows by construction; torch's value is rounding noise): it stays 0
        return dz

    def _lin_bwd(self, t, dy, need_dx=True):
        p = self.p
        if t.bn is not None:
            dz = self._bn_bwd(t, dy)
        else:
            dz = dy
            p.axpy_(self.grads[t.name + '.bias'], p.col_sum(dz))
        p.gemm_tn(dz, t.x, out=self.grads[t.name + '.weight'])
        if not need_dx:
            return None
        return p.gemm_nt(dz, p.transpose(self.params[t.name + '.weight']))

    # STN / QSTN body: x [B*n, cin] -> raw fc3 output [B, 4 | dim*dim]
    def _stn_fwd(self, prefix, x, B, n):
        tape = []
        h = self._lin(tape, x, prefix + 'conv1', prefix + 'bn1', True)
        h = self._lin(tape, h, prefix + 'conv2', prefix + 'bn2', True)
        g = self._lin_pool(tape, h, prefix + 'conv3', prefix + 'bn3', True, B, n)
        f = self._lin(tape, g, prefix + 'fc1', prefix + 'bn4', True)
        f = self._lin(tape, f, prefix + 'fc2', prefix + 'bn5', True)
        out = self._lin(tape, f, prefix + 'fc3', None, False)
        return out, tape

    def _stn_bwd(self, ctx, dout, need_dx):
        tape = ctx
        d = self._lin_bwd(tape[5], dout)
        d = self._lin_bwd(tape[4], d)
        d = self._lin_bwd(tape[3], d)
        d = self._lin_bwd(tape[2], d)
        d = self._lin_bwd(tape[1], d)
        return self._lin_bwd(tape[0], d, need_dx)

    # PointNetfeat body on already transformed points: pts [B,n,3] -> max feature [B,1024]
    def _feat_fwd(self, prefix, pts, B, n):
        p = self.p
        tape = []
        a = self._lin(tape, pts.reshape(B * n, 3), prefix + 'conv0a', prefix + 'bn0a', True)
        hb = self._lin(tape, a, prefix + 'conv0b', prefix + 'bn0b', True)
        traw, stn_ctx = self._stn_fwd(prefix + 'stn2.', hb, B, n)
        T = p.add_row_(traw, self._eye64).view(B, 64, 64)
        ht = p.gemm_nt(hb.view(B, n, 64), T).view(B * n, 64)          # torch.bmm(trans2, x), model.py:200
        h = self._lin(tape, ht, prefix + 'conv1', prefix + 'bn1', True)
        h = self._lin(tape, h, prefix + 'conv2', prefix + 'bn2', True)
        g = self._lin_pool(tape, h, prefix + 'conv3', prefix + 'bn3', False, B, n)
        return g, (tape, stn_ctx, T, hb, B, n)

    def _feat_bwd(self, ctx, dg, need_dpts):
        p = self.p
        tape, stn_ctx, T, hb, B, n = ctx
        d = self._lin_bwd(tape[4], dg)
        d = self._lin_bwd(tape[3], d)
        dht = self._lin_bwd(tape[2], d).view(B, n, 64)
        dhb = p.gemm_nt(dht, p.transpose(T)).view(B * n, 64)            # dx = T^T dy  (rows: dy_row T)
        dT = p.gemm_tn(dht, hb.view(B, n, 64)).view(B, 64 * 64)          # dT[b] = dy[b]^T x[b]
        p.axpy_(dhb, self._stn_bwd(stn_ctx, dT, True))
        d = self._lin_bwd(tape[1], dhb)
        return self._lin_bwd(tape[0], d, need_dpts)

    def _rotate(self, pts, R):
        """[B,n,3] x [B,3,3] -> per point R p  (torch.bmm(trans, x), model.py:328-329)."""
        return self.p.gemm_nt(pts, R)

    def _rotate_bwd_R(self, dpts_t, pts, B, n):
        return self.p.gemm_tn(dpts_t.view(B, n, 3), pts)                 # dR[b] = dy[b]^T x[b]

    # ------------------------------------------------------------------------------------------ forward / backward
    def forward(self, batch):
        """Train-mode forward -> logits [B, output_dim]; keeps the records for backward()."""
        p = self.p
        patch = batch['patch_pts_ps'].contiguous()
        B = patch.shape[0]
        if patch.shape[1] != self.P or batch['pts_sub_sample_ms'].shape[1] != self.S:
            raise ValueError('batch shapes do not match points_per_patch / sub_sample_size')
        sub = p.center(batch['pts_sub_sample_ms'].contiguous(), batch['imp_surf_query_point_ms'].contiguous())   # model.py:303
        rec = {'B': B}
        R = None
        if self.use_point_stn and self.shared:
            allp = torch.cat((patch, sub), dim=1).contiguous()            # model.py:326
            qraw, rec['qstn'] = self._stn_fwd('point_stn.', allp.reshape(B * (self.P + self.S), 3), B, self.P + self.S)
            R = p.quat_to_rot(qraw)
            rec['qraw'] = qraw
            sub_t, patch_t = self._rotate(sub, R), self._rotate(patch, R)
        elif self.use_point_stn:
            qraw, rec['qstn'] = self._stn_fwd('feat_global.stn1.', sub.reshape(B * self.S, 3), B, self.S)
            R = p.quat_to_rot(qraw)
            rec['qraw'] = qraw
            sub_t, patch_t = self._rotate(sub, R), self._rotate(patch, R)  # model.py:186,337-339
        else:
            sub_t, patch_t = sub, patch
        rec['patch'], rec['sub'], rec['R'] = patch, sub, R
        g_glob, rec['feat_global'] = self._feat_fwd('feat_global.', sub_t, B, self.S)
        head = []
        f_glob = self._lin(head, g_glob, 'fc1_global', 'bn1_global', True)
        g_loc, rec['feat_local'] = self._feat_fwd('feat_local.', patch_t, B, self.P)
        f_loc = self._lin(head, g_loc, 'fc1_local', 'bn1_local', True)
        x = torch.cat((f_loc, f_glob), dim=1).contiguous()                # model.py:346
        x = self._lin(head, x, 'fc2', 'bn2', True)
        x = self._lin(head, x, 'fc3', 'bn3', True)
        logits = self._lin(head, x, 'fc4', None, False)
        rec['head'] = head
        self._rec = rec
        return logits

    def backward(self, dlogits, need_inputs=False):
        """Accumulates into self.grads (call zero_grad() first, like optimizer.zero_grad()).  need_inputs: also
        -> (d patch_pts_ps [B,P,3], d centred sub-sample [B,S,3])."""
        p = self.p
        rec = self._rec
        B, head = rec['B'], rec['head']
        P, S = self.P, self.S
        d = self._lin_bwd(head[4], dlogits.contiguous())
        d = self._lin_bwd(head[3], d)
        d = self._lin_bwd(head[2], d)
        half = self.net // 2
        d_loc, d_glob = d[:, :half].contiguous(), d[:, half:].contiguous()
        need_R = rec['R'] is not None
        need_dpts = need_R or need_inputs
        dg_loc = self._lin_bwd(head[1], d_loc)
        dpatch_t = self._feat_bwd(rec['feat_local'], dg_loc, need_dpts)
        dg_glob = self._lin_bwd(head[0], d_glob)
        dsub_t = self._feat_bwd(rec['feat_global'], dg_glob, need_dpts)
        if need_R:
            dR = self._rotate_bwd_R(dsub_t, rec['sub'], B, S)
            p.axpy_(dR, self._rotate_bwd_R(dpatch_t, rec['patch'], B, P))
            dq = p.quat_to_rot_bwd(rec['qraw'], dR.view(B, 9))
            dsrc = self._stn_bwd(rec['qstn'], dq, need_inputs)       # d of the QSTN's input points
        self._rec = None
        if not need_inputs:
            return None
        if not need_R:
            return dpatch_t.view(B, P, 3), dsub_t.view(B, S, 3)
        Rt = p.transpose(rec['R'])
        dpatch = p.gemm_nt(dpatch_t.view(B, P, 3), Rt)                  # x_t = R x: dx = R^T dx_t (rows: dx_t R)
        dsub = p.gemm_nt(dsub_t.view(B, S, 3), Rt)
        if self.shared:                                                  # the QSTN saw cat(patch, sub)
            dsrc = dsrc.view(B, P + S, 3)
            p.axpy_(dpatch, dsrc[:, :P])
            p.axpy_(dsub, dsrc[:, P:])
        else:                                                            # feat_global.stn1 saw the sub-sample
            p.axpy_(dsub, dsrc)
        return dpatch, dsub

    # ------------------------------------------------------------------------------------------ eval-mode forward
    def evaluate(self, batch):
        """`p2s_model.eval()` forward + compute_loss without gradients (the test batches interleaved with training,
        points_to_surf_train.py:483-500): BatchNorm uses the running statistics, nothing is recorded or updated.
        -> (logits [B, output_dim], compute_loss's list: [loss_magnitude, loss_sign] or [loss_imp_surf])."""
        p = self.p
        P, S = self.P, self.S

        def lin(x, name, bn, relu):
            z = p.gemm_nt(x, self.params[name + '.weight'], self.params[name + '.bias'])
            if bn is None:
                return z
            rv = self.buffers[bn + '.running_var']
            invstd = torch.rsqrt(rv + BN_EPS)
            return p.bn_apply(z, self.buffers[bn + '.running_mean'], invstd, self.params[bn + '.weight'], self.params[bn + '.bias'], relu)

        def stn(prefix, x, B, n):
            h = lin(x, prefix + 'conv1', prefix + 'bn1', True)
            h = lin(h, prefix + 'conv2', prefix + 'bn2', True)
            h = lin(h, prefix + 'conv3', prefix + 'bn3', True)
            g, _ = p.maxpool_fwd(h, B, n)
            f = lin(g, prefix + 'fc1', prefix + 'bn4', True)
            f = lin(f, prefix + 'fc2', prefix + 'bn5', True)
            return lin(f, prefix + 'fc3', None, False)

        def feat(prefix, pts, B, n):
            a = lin(pts.reshape(B * n, 3), prefix + 'conv0a', prefix + 'bn0a', True)
            hb = lin(a, prefix + 'conv0b', prefix + 'bn0b', True)
            T = p.add_row_(stn(prefix + 'stn2.', hb, B, n), self._eye64).view(B, 64, 64)
            h = p.gemm_nt(hb.view(B, n, 64), T).view(B * n, 64)
            h = lin(h, prefix + 'conv1', prefix + 'bn1', True)
            h = lin(h, prefix + 'conv2', prefix + 'bn2', True)
            h = lin(h, prefix + 'conv3', prefix + 'bn3', False)
            return p.maxpool_fwd(h, B, n)[0]

        patch = batch['patch_pts_ps'].contiguous()
        B = patch.shape[0]
        sub = p.center(batch['pts_sub_sample_ms'].contiguous(), batch['imp_surf_query_point_ms'].contiguous())
        if self.use_point_stn:
            src = torch.cat((patch, sub), dim=1).contiguous() if self.shared else sub
            n = P + S if self.shared else S
            R = p.quat_to_rot(stn('point_stn.' if self.shared else 'feat_global.stn1.', src.reshape(B * n, 3), B, n))
            sub, patch = p.gemm_nt(sub, R), p.gemm_nt(patch, R)
        f_glob = lin(feat('feat_global.', sub, B, S), 'fc1_global', 'bn1_global', True)
        f_loc = lin(feat('feat_local.', patch, B, P), 'fc1_local', 'bn1_local', True)
        x = lin(torch.cat((f_loc, f_glob), dim=1).contiguous(), 'fc2', 'bn2', True)
        x = lin(x, 'fc3', 'bn3', True)
        logits = lin(x, 'fc4', None, False)
        losses = compute_loss(logits, batch, self.outputs, self.loss_weights, self.fixed_radius, prims=p, need_grad=False)
        return logits, losses

    def zero_grad(self):
        self.flat_grads.zero_()

    def optimizer_step(self):
        self.p.sgd_(self.flat_params, self.flat_grads, self.flat_mom, self.lr, self.momentum, self.steps_done == 0)
        self.steps_done += 1

    def _forward_backward(self, batch):
        self.zero_grad()
        logits = self.forward(batch)
        losses, dlogits = compute_loss(logits, batch, self.outputs, self.loss_weights, self.fixed_radius, prims=self.p,
                                       need_grad=True)
        self.backward(dlogits)
        return logits, losses

    def _reduce_gradients(self):
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            dist.all_reduce(self.flat_grads)
            self.flat_grads /= dist.get_world_size()

    def step(self, batch):
        """One iteration of the reference's inner loop (points_to_surf_train.py:441-461): zero_grad, forward,
        compute_loss, backward, SGD.  Returns [loss_magnitude, loss_sign], or [loss_imp_surf] for the regression head
        (0-d float64 tensors on the device)."""
        if self._graph is not None and self._graph_matches(batch):     # a partial last batch takes the eager step
            return self._step_graph(batch)
        logits, losses = self._forward_backward(batch)
        self._reduce_gradients()
        self.optimizer_step()
        self.last_logits = logits
        return losses

    # ------------------------------------------------------------------------------------------ CUDA-graph replay
    _graph = None
    _INPUT_KEYS = ('patch_pts_ps', 'pts_sub_sample_ms', 'imp_surf_query_point_ms', 'patch_radius_ms')

    def capture_graph(self, example_batch):
        """Capture forward+backward and the SGD update of one batch shape into two CUDA graphs (the gradient all_reduce
        runs eagerly between them).  A step is ~400 small launches issued from Python; at the 128-queries-per-rank size
        of BASELINE config 4 the host is the bottleneck, replaying a graph removes it.  The parameters, momentum buffers
        and running statistics are restored after the warm-up iterations that size the scratch buffers, so capturing
        does not train."""
        if self.device.type != 'cuda':
            raise ValueError('CUDA graphs need a CUDA device')
        static = {k: example_batch[k].detach().clone().contiguous() for k in self._batch_keys}
        saved = (self.flat_params.clone(), self.flat_mom.clone(), {k: v.clone() for k, v in self.buffers.items()}, self.steps_done)
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            for _ in range(2):
                self._forward_backward(static)
                self.optimizer_step()
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        self.flat_params.copy_(saved[0])
        self.flat_mom.copy_(saved[1])
        for k, v in saved[2].items():
            self.buffers[k].copy_(v)
        self.steps_done = saved[3]
        bn_before = {k: int(v) for k, v in self.buffers.items() if k.endswith('num_batches_tracked')}
        g1, g2 = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        with torch.cuda.graph(g1):
            logits, losses = self._forward_backward(static)
        with torch.cuda.graph(g2):
            # momentum buffers are zero before the first step, so `buf = mu * buf + g` equals torch's `buf = g`
            self.p.sgd_(self.flat_params, self.flat_grads, self.flat_mom, self.lr, self.momentum, False)
        for k, n in bn_before.items():      # the capture pass incremented the host-side counters once: undo
            self.buffers[k].fill_(n)
        self._graph = (g1, g2, static, logits, losses)
        self._graph_lr = (float(self.lr), float(self.momentum))
        return self

    def _capture_sgd(self):
        """The SGD kernel takes lr / momentum as launch arguments, i.e. a captured graph bakes them in: re-capture the
        (one-kernel) update graph whenever the schedule changed them."""
        g2 = torch.cuda.CUDAGraph()
        torch.cuda.synchronize(self.device)
        with torch.cuda.graph(g2):
            self.p.sgd_(self.flat_params, self.flat_grads, self.flat_mom, self.lr, self.momentum, False)
        g1, _, static, logits, losses = self._graph
        self._graph = (g1, g2, static, logits, losses)
        self._graph_lr = (float(self.lr), float(self.momentum))

    def _graph_matches(self, batch):
        static = self._graph[2]
        return all(tuple(batch[k].shape) == tuple(static[k].shape) for k in self._batch_keys)

    def _step_graph(self, batch):
        if (float(self.lr), float(self.momentum)) != self._graph_lr:
            self._capture_sgd()
        g1, g2, static, logits, losses = self._graph
        for k in self._batch_keys:
            static[k].copy_(batch[k], non_blocking=True)
        g1.replay()
        self._reduce_gradients()
        g2.replay()
        self.steps_done += 1
        for k, v in self.buffers.items():
            if k.endswith('num_batches_tracked'):
                v += 1
        self.last_logits = logits
        return losses

    def state_dict(self):
        """Reference-named state dict (conv weights back to [out, in, 1])."""
        out = {}
        for name, t in self.params.items():
            out[name] = t.detach().clone().reshape(self._orig_shape[name])
        for name, t in self.buffers.items():
            out[name] = t.detach().clone()
        return out

    def named_gradients(self):
        return {name: g.reshape(self._orig_shape[name]) for name, g in self.grads.items()}


class EvalGrad(TrainStep):
    """Gradients of the eval-mode network (`model.eval()`: every BatchNorm uses running_mean / running_var, eps 1e-5)
    with respect to its parameters and inputs, for autograd through points2surf_b200.model.PointsToSurfModel.

        eg = EvalGrad(state_dict, use_point_stn, shared_transformer, P, S, output_dim=2)
        eg.forward(batch)                                 # fp32 recompute, records ReLU masks and arg-maxes
        dpatch, dsub, dquery = eg.backward_inputs(dlogits)   # eg.named_gradients(): every parameter

    TrainStep's network walk and backward run with eval-mode BatchNorm units: the statistics are constants, so the
    backward is a row-local scaling (p2s_op_bn_eval_backward) and every max-pooled conv3 layer sends its gradient to one
    point per (query, channel) (p2s_op_bn_maxpool_eval_bwd: weight gradient as a gather over B rows, input gradient as a
    scatter).  Unlike the train-mode step, the bias in front of a BatchNorm gets its gradient (sum of dz).  Nothing is
    updated: running statistics and num_batches_tracked stay as they are."""

    _momentum = False

    def __init__(self, state_dict, use_point_stn, shared_transformer, points_per_patch=300, sub_sample_size=1000,
                 net_size=1024, output_dim=2, device=None, prims=None, dtype=torch.float32):
        outputs = ('imp_surf',) if output_dim == 1 else ('imp_surf_magnitude', 'imp_surf_sign')
        super().__init__(state_dict, use_point_stn, shared_transformer, points_per_patch, sub_sample_size, net_size,
                         device=device, prims=prims, outputs=outputs, dtype=dtype)
        self._invstd = {k[:-len('.running_var')]: torch.rsqrt(v + BN_EPS) for k, v in self.buffers.items()
                        if k.endswith('.running_var')}

    def _bn_fwd(self, z, bn, relu):
        mean, invstd = self.buffers[bn + '.running_mean'], self._invstd[bn]
        y = self.p.bn_apply(z, mean, invstd, self.params[bn + '.weight'], self.params[bn + '.bias'], relu)
        return y, mean, invstd

    def _bn_pool_fwd(self, z, bn, relu, B, n):
        mean, invstd = self.buffers[bn + '.running_mean'], self._invstd[bn]
        out, arg = self.p.bn_maxpool_apply(z, B, n, mean, invstd, self.params[bn + '.weight'], self.params[bn + '.bias'], relu)
        return out, arg, mean, invstd

    def _bn_bwd(self, t, dy):
        p = self.p
        dz, dgamma, dbeta, dbias = p.bn_eval_backward(dy, t.z, t.y_mask, t.mean, t.invstd, self.params[t.bn + '.weight'])
        p.axpy_(self.grads[t.bn + '.weight'], dgamma)
        p.axpy_(self.grads[t.bn + '.bias'], dbeta)
        p.axpy_(self.grads[t.name + '.bias'], dbias)
        return dz

    def _lin_bwd(self, t, dy, need_dx=True):
        if t.pool is None:
            return super()._lin_bwd(t, dy, need_dx)
        p = self.p
        out, arg, B, n = t.pool
        dx, dgamma, dbeta, dbias = p.bn_maxpool_eval_backward(dy, arg, out, t.z, t.x, self.params[t.name + '.weight'], t.mean,
                                                              t.invstd, self.params[t.bn + '.weight'], t.relu, B, n,
                                                              self.grads[t.name + '.weight'], need_dx)
        p.axpy_(self.grads[t.bn + '.weight'], dgamma)
        p.axpy_(self.grads[t.bn + '.bias'], dbeta)
        p.axpy_(self.grads[t.name + '.bias'], dbias)
        return dx

    def backward_inputs(self, dlogits, dsub_extra=None):
        """Parameter gradients into self.grads and -> (d patch_pts_ps, d pts_sub_sample_ms, d imp_surf_query_point_ms)
        through the centring sub = pts_sub_sample_ms - query; dsub_extra [B,S,3]: a gradient that reaches the centred
        sub-sample by another way (the reference centres the caller's tensor in place, later uses of it add theirs)."""
        p = self.p
        dpatch, dsub = self.backward(dlogits, need_inputs=True)
        if dsub_extra is not None:
            p.axpy_(dsub, dsub_extra)
        B = dsub.shape[0]
        ones = torch.ones((B, self.S, 1), dtype=dsub.dtype, device=dsub.device)
        dquery = torch.zeros((B, 3), dtype=dsub.dtype, device=dsub.device)
        p.axpy_(dquery, p.gemm_tn(ones, dsub), -1.0)                     # d query = -sum over the points of d sub
        return dpatch, dsub, dquery
