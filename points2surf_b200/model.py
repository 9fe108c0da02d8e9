"""Drop-in for source/points_to_surf_model.py: `PointsToSurfModel` with the reference's constructor
signature (points_to_surf_model.py:238-240), parameter names and shapes (so the reference's checkpoints load,
with or without the DataParallel 'module.' prefix), whose forward runs on the CUDA kernels.

Supported subset (SURVEY.md section 8b): sym_op='max', single_transformer=False, use_feat_stn=True,
output_dim 2 (imp_surf_magnitude, imp_surf_sign) or 1 (imp_surf, the regression ablation; forward returns [B, 1]
logits, evaluated with ops.distance_from_logits).  Anything else raises ValueError like the reference does for unknown options
(points_to_surf_model.py:175).  forward() ignores .train() and always uses running BatchNorm statistics (the
reference evaluates with .eval(), points_to_surf_eval.py:170).

Gradients.  In eval mode (`m.eval()`), with grad enabled and some parameter or input requiring grad, the logits carry a
grad_fn and `backward()` fills `.grad` of every parameter (conv / linear weight and bias, BatchNorm weight and bias) and
input (patch_pts_ps, pts_sub_sample_ms, imp_surf_query_point_ms) that requires grad, with the gradient of the reference's
eval-mode network (points_to_surf_model.py:296-352, BatchNorm with running_mean / running_var, eps 1e-5), computed by
CUDA backward kernels (points2surf_b200.train.EvalGrad).  The logits stay the engine's, bit for bit; the backward
recomputes the activations in fp32, records that network's ReLU masks and max-pool arg-maxes, and differentiates it.  So
the gradients are those of the fp32 network, which can differ from a precision='tc' forward's decisions near a ReLU or
max-pool tie.  The caller's sub-sample is centred in place like the reference's `shape_features -= query`: a leaf
sub-sample that requires grad raises, a non-leaf one passes its gradient on, and the query receives minus the sum of it.
Train mode and torch.no_grad() return logits without grad_fn.  Double backward is not supported; train-mode
(batch-statistics) gradients are points2surf_b200.train.TrainStep's.
"""
import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import arch
from . import ops


class _Block(nn.Module):
    """Plain container so that nested names ('feat_local.stn2.conv1') resolve like the reference's."""


class PointsToSurfModel(nn.Module):
    def __init__(self, net_size_max=1024, num_points=500, output_dim=3, use_point_stn=True, use_feat_stn=True,
                 sym_op='max', use_query_point=False, sub_sample_size=500, do_augmentation=True,
                 single_transformer=False, shared_transformation=False, precision='tc', guard_band=0.05):
        super().__init__()
        if sym_op != 'max':
            raise ValueError('Unsupported symmetric operation: %s' % sym_op)
        if single_transformer:
            raise ValueError('Unsupported option: single_transformer=1 (shared encoder ablation)')
        if not use_feat_stn:
            raise ValueError('Unsupported option: use_feat_stn=0')
        if output_dim not in (1, 2):
            raise ValueError('Unsupported output_dim %d: only (imp_surf_magnitude, imp_surf_sign) or imp_surf is supported'
                             % output_dim)
        if net_size_max != 1024:
            raise ValueError('Unsupported net_size %d' % net_size_max)
        self.net_size_max = net_size_max
        self.num_points = num_points
        self.use_query_point = use_query_point
        self.use_point_stn = bool(use_point_stn)
        self.sub_sample_size = sub_sample_size
        self.do_augmentation = do_augmentation
        self.single_transformer = False
        self.shared_transformation = bool(shared_transformation)
        self.precision, self.guard_band = precision, guard_band
        self.output_dim = output_dim
        for name, kind, cout, cin in arch.layer_specs(self.use_point_stn, self.shared_transformation, net_size_max, output_dim):
            parent = self
            parts = name.split('.')
            for p in parts[:-1]:
                if not hasattr(parent, p):
                    setattr(parent, p, _Block())
                parent = getattr(parent, p)
            if kind == 'conv':
                mod = nn.Conv1d(cin, cout, 1)
            elif kind == 'fc':
                mod = nn.Linear(cin, cout)
            else:
                mod = nn.BatchNorm1d(cout)
            setattr(parent, parts[-1], mod)
        self._engine = None
        self._engine_key = None

    # any parameter update invalidates the packed device weights
    def _invalidate(self):
        if self._engine is not None:
            self._engine.close()
        self._engine, self._engine_key = None, None

    def load_state_dict(self, state_dict, strict=True, **kw):
        from .weights import strip_module_prefix
        self._invalidate()
        return super().load_state_dict(strip_module_prefix(state_dict), strict=strict, **kw)

    def _get_engine(self, device):
        key = (device.index, tuple(int(p._version) for p in self.parameters()))
        if self._engine is None or self._engine_key != key:
            self._invalidate()
            self._engine = ops.Engine(self.state_dict(), self.use_point_stn, self.shared_transformation,
                                      points_per_patch=self.num_points, sub_sample_size=self.sub_sample_size,
                                      net_size=self.net_size_max, device=device.index or 0,
                                      precision=self.precision, guard_band=self.guard_band, output_dim=self.output_dim)
            self._engine_key = key
        return self._engine

    def forward(self, x):
        patch = x['patch_pts_ps']
        shape = x['pts_sub_sample_ms']
        query = x['imp_surf_query_point_ms']
        if not patch.is_cuda:
            raise ops.P2SError('PointsToSurfModel.forward needs CUDA tensors: points2surf_b200 has no CPU path')
        if not self.training and torch.is_grad_enabled():
            params = tuple(self.parameters())
            if any(t.requires_grad for t in (patch, shape, query) + params):
                if shape.is_leaf and shape.requires_grad:
                    # what the reference's in-place centring raises (points_to_surf_model.py:303), before any work
                    raise RuntimeError('a leaf Variable that requires grad is being used in an in-place operation.')
                out, _ = _EvalForward.apply(self, patch, shape, query, *params)
                return out
        eng = self._get_engine(patch.device)
        out = eng.forward(patch, shape, query)
        # the reference centres the caller's sub-sample in place (points_to_surf_model.py:303); keep that side effect
        shape -= query.unsqueeze(1).expand(shape.shape)
        return out


class _EvalForward(torch.autograd.Function):
    """Eval-mode forward on the engine + the in-place centring of the sub-sample, differentiable in all inputs and the
    parameters (passed explicitly, in `model.parameters()` order, so autograd hands their gradients to the Parameters).
    Keeps references to its inputs only; the backward recomputes the fp32 activations (train.EvalGrad)."""

    @staticmethod
    def forward(ctx, model, patch, shape, query, *params):
        out = model._get_engine(patch.device).forward(patch, shape, query)
        shape -= query.unsqueeze(1).expand(shape.shape)      # the reference's in-place centring (model.py:303)
        ctx.mark_dirty(shape)
        if not (shape.requires_grad or query.requires_grad):
            ctx.mark_non_differentiable(shape)              # like `shape -= query` on two tensors without grad
        ctx.model = model
        ctx.save_for_backward(patch, shape, query, *params)
        return out, shape

    @staticmethod
    @once_differentiable
    def backward(ctx, dout, dshape_out):
        from .train import EvalGrad
        m = ctx.model
        patch, shape, query = ctx.saved_tensors[:3]
        params = ctx.saved_tensors[3:]
        sd = dict(zip((n for n, _ in m.named_parameters()), (t.detach() for t in params)))
        sd.update((n, b.detach()) for n, b in m.named_buffers())
        eg = EvalGrad(sd, m.use_point_stn, m.shared_transformation, m.num_points, m.sub_sample_size, m.net_size_max,
                      output_dim=m.output_dim, device=patch.device)
        # `shape` holds the centred sub-sample (the same fp32 subtraction as the recompute's centring, which a zero
        # query leaves exact)
        eg.forward({'patch_pts_ps': patch.detach(), 'pts_sub_sample_ms': shape.detach(),
                    'imp_surf_query_point_ms': torch.zeros_like(query.detach())})
        dpatch, dshape, dquery = eg.backward_inputs(dout, dshape_out)
        grads = eg.named_gradients()
        need = ctx.needs_input_grad
        dparams = [grads[n].reshape(t.shape) if need[4 + i] else None
                   for i, (n, t) in enumerate(zip((n for n, _ in m.named_parameters()), params))]
        return (None, dpatch if need[1] else None, dshape if need[2] else None, dquery if need[3] else None, *dparams)
