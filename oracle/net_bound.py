"""Float64 model of the eval-mode inference network with a per-element error bound for each of the engine's arithmetics.

The network is evaluated in float64 on the parameters the engine receives: the float32 outputs of `weights.fold`
(BatchNorm folded into the preceding layer).  Alongside every value v the model carries a scale e of the engine's
error, element by element; the engine's float32 result x is held to |x - v| <= LAMBDA e (`excess`).  Three arithmetic
models are covered:

  'fp32'        csrc/net_fp32.cu: float32 FMA everywhere.
  'tc'          csrc/net_tc.cu `pointnet_pass_kernel<false>`: fp16 operands, fp32 accumulation on the tensor cores;
                FC tails on the split-precision kernel of csrc/fc_tc.cu.
  'tc_precise'  `pointnet_pass_kernel<true>` plus the split FC tails: the guard-band recompute path.

Why a root-sum-square and not the worst case.  The worst-case rule e_y = |W| e_x + ... multiplies the bound by a layer's
row 1-norm, 10 to 40 on these layers, and on the golden inputs it put the fp32 engine's logits at 1e12 times their value:
true, and useless.  The rounding errors of the many terms of one output are not aligned, so the rules below add the
per-term bounds in quadrature and the check allows LAMBDA = 4 times the result.  For independent, centred terms that is
Hoeffding's inequality, P(|sum| > 4 sqrt(sum b_k^2)) <= 2 e^-8 per element; every per-term bound b_k is itself a worst
case.  The CPU emulations of the three arithmetics stay below 1/20 of the check and single faults break it
(tests/test_net_bound_host.py).

Rules (u32 = 2^-24; |.| and squares are element-wise; sums over the K terms of one output):

* Linear step y = W x + b over K terms (net_tc.cu:243-252 mid layers, :294-303 big layer; fc_tc.cu:153-183;
  net_fp32.cu:63-82):
      e_y^2 = W^2 e_x^2 + e_W^2 x^2 + rho^2 W^2 x^2 + n u^2 (W^2 x^2 + b^2 + y^2) + floor^2
  with |x| + e_x and |W| + e_W in the operand terms (the engine rounds its own operands, not the float64 ones).  The
  accumulation term is the random-walk size of n roundings of partial sums, which grow like sqrt(sum (w x)^2) for mixed
  signs and like |y| for aligned ones; n counts K products (3K for split operands: three MMAs per k-step) plus one
  for the bias.
* ReLU and the max over points are 1-Lipschitz: ReLU keeps e, the max takes the max over points of e
  (net_tc.cu:309-327, net_fp32.cu:85-100: max is exact).  A bias added after the max (net_fp32.cu:296-302 and
  fc_tc.cu:239 / :95) adds one fp32 rounding, u32 (|v + b| + e).
* Operand rounding rho of a product:
    fp16   2 2^-11 + 2^-22 relative (both operands rounded to nearest fp16: `cvt.rn...f16x2`, net_tc.cu:88,
           pack_kmajor_kernel net_tc.cu:343, the per-query image fc_tc.cu:197-203);
    split  3 2^-22 relative: hi = fp16(x), lo = fp16(x - hi) keeps |x - hi - lo| <= 2^-22 |x| per operand, and the
           omitted lo*lo product is below 2^-22 |a||b| (net_tc.cu:92-96, :108, :298; fc_tc.cu:38-44, :153-155);
    fp32   none: the weights are exact inputs.
  fp16 and split add a floor for subnormals: an operand below TINY (2^-14 for fp16; 2^-3 for a split, whose lo part is
  then subnormal) is off by up to 2^-25 absolute, so floor^2 = (2^-24)^2 (sum_{|x_k| < TINY} w_k^2 + sum_{|w_k| < TINY}
  x_k^2), the factor 2 covering the products of the two operand errors.  The split of a weight below 2^-3 keeps about
  20 bits, not 22.  No operand may exceed 65504, because `cvt...satfinite` saturates: this is asserted, not bounded.
* Accumulation: fp32 FMA uses u = 2^-24.  The tensor cores' fp32 accumulation is not IEEE round-to-nearest: the
  products of one MMA are aligned to the largest exponent and the sum is truncated (Fasi, Higham, Mikaitis, Pranesh,
  "Numerical behavior of NVIDIA tensor cores", PeerJ CS 2021), so each addition can lose up to one ulp instead of half
  of one.  The tensor-core steps therefore use u = 2^-23.
* Steps only the tensor-core path has:
    - W0 R formed in fp32 per query (net_tc.cu:185-187) and the point minus the query point (net_tc.cu:211) ahead of the
      3-term FMA chain (net_tc.cu:226): e = (u32 + gamma_3 + gamma_4) |W0| |R| |x| + gamma_4 |b| -- the same bound as
      the fp32 path's transform_points (net_fp32.cu:353-359) followed by a K = 3 GEMM.
    - the STN64's last layer folded into conv1 (fold_fc3_kernel, net_tc.cu:400-413): G = W1 Wfc3 and g0 = W1 + W1 bfc3
      are fp32 64-term FMA sums, e_G = u32 sqrt(64 (W1^2 Wfc3^2 + G^2)), e_g0 = u32 sqrt(65 (W1^2 + W1^2 bfc3^2 + g0^2)).
    - the per-query image conv1 (T + I) = f2 G^T + g0 on the split FC kernel (net_tc.cu:759), stored as fp16
      (`pack_img` 1) or hi | lo (`pack_img` 2): it is the W operand of pass C's second mid layer, rounded like the
      pass kernel's other operands.
    - the conv3 bias added by pack_a_kernel (fc_tc.cu:239) before the split of the first FC layer.
    - fc4 and the QSTN's fc3 on the fp32 `gemm_nt` kernel (net_tc.cu:735, :798).
* The fp32 path's STN64 applies T = fc3(f2) + I (net_fp32.cu:335-338, one rounding) as a per-query 64-term GEMM and then
  conv1 (net_fp32.cu:411-412).
* The quaternion step is not propagated.  `network` takes an optional rotation R (the engine's own, from
  `forward_with_aux`) and evaluates everything downstream of R with it, exactly as the engine does.  R itself is
  bounded from the bound of q4: every entry of quat_to_rot(q) is 1 - 2 (q_i^2 + q_j^2) / |q|^2 or
  2 (q_i q_j +- q_k q_l) / |q|^2, whose gradient has 1-norm <= 14 / |q|.  Over the box |q' - q|_inf <= e_q4 this is
  at most L = 24 / (|q| - LAMBDA |e_q4|_2), so R is checked against the bound
      e_R = L (LAMBDA max_k e_q4,k + u32 |q_0|) + 2^-18,
  the u32 |q_0| for the fp32 `+ 1` and 2^-18 (64 u32) for the fp32 evaluation of the formula itself
  (net_fp32.cu:310-330: entries of magnitude <= 1 built from terms of magnitude <= 2 in about ten roundings).
"""
import numpy as np
import torch

from points2surf_b200 import synth
from points2surf_b200 import weights as _weights

U32 = 2.0 ** -24
UTC = 2.0 ** -23
U16 = 2.0 ** -11
SUB = 2.0 ** -24
FP16_MAX = 65504.0
LAMBDA = 4.0
RHO = {'fp32': 0.0, 'fp16': 2 * U16 + U16 * U16, 'split': 3 * 2.0 ** -22}
# below these magnitudes an operand's rounding error is the absolute 2^-25 of fp16 subnormals, not relative: fp16(x) is
# subnormal under 2^-14; the lo part of a split can be subnormal whenever |x| < 2^-3
TINY = {'fp16': 2.0 ** -14, 'split': 2.0 ** -3}
# (operand rounding, MMAs per k-step, unit roundoff) of the point-wise layers and of the FC tails
MODELS = {
    'fp32': dict(conv=('fp32', 1, U32), fc=('fp32', 1, U32)),
    'tc': dict(conv=('fp16', 1, UTC), fc=('split', 3, UTC)),
    'tc_precise': dict(conv=('split', 3, UTC), fc=('split', 3, UTC)),
}
FP32_FC = ('fp32', 1, U32)


def gamma(n, u=U32):
    """gamma_n = n u / (1 - n u) (Higham eq. 3.5): the worst case of n roundings, used for the 3-term first layer."""
    return n * u / (1.0 - n * u)


class V:
    """A float64 value and the scale of its per-element error bound."""

    def __init__(self, v, e):
        self.v, self.e = v, e

    def relu(self):
        return V(self.v.clamp_min(0.0), self.e)

    def max_points(self):
        return V(self.v.amax(-2), self.e.amax(-2))

    def add_bias(self, b):
        v = self.v + b
        return V(v, self.e + U32 * (v.abs() + self.e))


def fold_params(sd, variant):
    """name -> (W [N, K], b [N]) float64 tensors holding the float32 folded parameters the engine receives."""
    sd = _weights.strip_module_prefix(sd)
    v = synth.VARIANTS[variant]
    names = []

    def stn(p):
        names.extend([(p + c, p + bn) for c, bn in (('conv1', 'bn1'), ('conv2', 'bn2'), ('conv3', 'bn3'), ('fc1', 'bn4'), ('fc2', 'bn5'))])
        names.append((p + 'fc3', None))

    def feat(p, qstn):
        if qstn:
            stn(p + 'stn1.')
        stn(p + 'stn2.')
        names.extend([(p + c, p + bn) for c, bn in (('conv0a', 'bn0a'), ('conv0b', 'bn0b'), ('conv1', 'bn1'), ('conv2', 'bn2'), ('conv3', 'bn3'))])

    if v['use_point_stn'] and v['shared_transformer']:
        stn('point_stn.')
    feat('feat_local.', False)
    feat('feat_global.', bool(v['use_point_stn'] and not v['shared_transformer']))
    names += [('fc1_local', 'bn1_local'), ('fc1_global', 'bn1_global'), ('fc2', 'bn2'), ('fc3', 'bn3'), ('fc4', None)]
    out = {}
    for layer, bn in names:
        w, b = _weights.fold(sd, layer, bn)
        out[layer] = (torch.from_numpy(w.astype(np.float64)).reshape(b.size, -1), torch.from_numpy(b.astype(np.float64)))
    return out


def _linear(x, W, b, arith, eW=None, eb=None):
    """y = x W^T + b over the last axis of x.  W is [N, K], or per query [B, N, K] with x [B, n, K]."""
    op, terms, u = arith
    rho = RHO[op]
    aW = W.abs() if eW is None else W.abs() + eW
    ax = x.v.abs() + x.e
    if op != 'fp32':
        assert float(ax.max()) <= FP16_MAX and float(aW.max()) <= FP16_MAX, 'an fp16 operand would saturate'
    v = x.v @ W.transpose(-1, -2)
    mag2 = (ax * ax) @ (aW * aW).transpose(-1, -2)
    var = (x.e * x.e) @ (W * W).transpose(-1, -2) + rho * rho * mag2
    if eW is not None:
        var = var + (ax * ax) @ (eW * eW).transpose(-1, -2)
    n = terms * W.shape[-1]
    if b is not None:           # b, eb: [N]
        v = v + b
        mag2 = mag2 + b * b
        n += 1
        if eb is not None:
            var = var + eb * eb
    var = var + n * (u * (1 + 2.0 ** -9)) ** 2 * (mag2 + v * v)
    if op != 'fp32':
        th = TINY[op]
        var = var + SUB * SUB * ((ax < th).double() @ (aW * aW).transpose(-1, -2) + (ax * ax) @ (aW < th).double().transpose(-1, -2))
    return V(v, var.sqrt())


def _first(pts, center, R, W0, b0):
    """The 3 -> 64 layer on the (centred, rotated) points: fp32 on every path."""
    xc = pts - center.unsqueeze(1) if center is not None else pts
    if R is not None:
        xr, ar = xc @ R.transpose(1, 2), xc.abs() @ R.abs().transpose(1, 2)
    else:
        xr, ar = xc, xc.abs()
    v = xr @ W0.t() + b0
    mag = ar @ W0.abs().t()
    e = (U32 + gamma(3) + gamma(4)) * (1 + 2.0 ** -9) * mag + gamma(4) * b0.abs()
    return V(v, e)


def _big_max(x, W, b, arith):
    """128 -> 1024 without bias, max over the points, then the bias in fp32."""
    return _linear(x, W, None, arith).max_points().add_bias(b)


def _fc_tail(P, p, g, fc, fc3_arith):
    f1 = _linear(g, *P[p + 'fc1'], fc).relu()
    f2 = _linear(f1, *P[p + 'fc2'], fc).relu()
    return f2, (_linear(f2, *P[p + 'fc3'], fc3_arith) if fc3_arith else None)


def _qstn(P, p, pts, center, m):
    x = _first(pts, center, None, *P[p + 'conv1']).relu()
    x = _linear(x, *P[p + 'conv2'], m['conv']).relu()
    g = _big_max(x, *P[p + 'conv3'], m['conv']).relu()
    return _fc_tail(P, p, g, m['fc'], FP32_FC)[1]


def _feat(P, p, pts, center, R, model):
    """PointNetfeat after the optional QSTN: conv0a, conv0b, STN64, conv1 (T), conv2, conv3, max (+ bias, no ReLU)."""
    m = MODELS[model]
    x = _first(pts, center, R, *P[p + 'conv0a']).relu()
    x = _linear(x, *P[p + 'conv0b'], m['conv']).relu()
    s = p + 'stn2.'
    h = _linear(x, *P[s + 'conv1'], m['conv']).relu()
    h = _linear(h, *P[s + 'conv2'], m['conv']).relu()
    g = _big_max(h, *P[s + 'conv3'], m['conv']).relu()
    f2, _ = _fc_tail(P, s, g, m['fc'], None)
    W1, b1 = P[p + 'conv1']
    Wf, bf = P[s + 'fc3']
    B = x.v.shape[0]
    eye = torch.eye(64, dtype=W1.dtype, device=W1.device)
    if model == 'fp32':
        T = _linear(f2, Wf, bf, FP32_FC)
        Tv = T.v + eye.reshape(-1)
        T = V(Tv, T.e + U32 * (Tv.abs() + T.e))
        y = _linear(x, T.v.view(B, 64, 64), None, FP32_FC, eW=T.e.view(B, 64, 64))
        y = _linear(y, W1, b1, FP32_FC).relu()
    else:
        Wf3 = Wf.view(64, 64, 256)
        G = torch.einsum('oj,jik->oik', W1, Wf3).reshape(4096, 256)
        eG = U32 * (64 * (torch.einsum('oj,jik->oik', W1 * W1, Wf3 * Wf3).reshape(4096, 256) + G * G)).sqrt()
        g0 = (W1 + W1 @ bf.view(64, 64)).reshape(-1)
        eg0 = U32 * (65 * ((W1 * W1 + (W1 * W1) @ (bf * bf).view(64, 64)).reshape(-1) + g0 * g0)).sqrt()
        M = _linear(f2, G, g0, m['fc'], eW=eG, eb=eg0)
        y = _linear(x, M.v.view(B, 64, 64), b1, m['conv'], eW=M.e.view(B, 64, 64)).relu()
    y = _linear(y, *P[p + 'conv2'], m['conv']).relu()
    return _big_max(y, *P[p + 'conv3'], m['conv'])


def quat_to_rot(q):
    """source/base/utils.py:13-46 in float64 (the quaternion is not normalised)."""
    s = 2.0 / (q * q).sum(-1)
    h = q.unsqueeze(-1) * q.unsqueeze(-2)
    R = torch.stack([1 - (h[:, 2, 2] + h[:, 3, 3]) * s, (h[:, 1, 2] - h[:, 3, 0]) * s, (h[:, 1, 3] + h[:, 2, 0]) * s,
                     (h[:, 1, 2] + h[:, 3, 0]) * s, 1 - (h[:, 1, 1] + h[:, 3, 3]) * s, (h[:, 2, 3] - h[:, 1, 0]) * s,
                     (h[:, 1, 3] - h[:, 2, 0]) * s, (h[:, 2, 3] + h[:, 1, 0]) * s, 1 - (h[:, 1, 1] + h[:, 2, 2]) * s], -1)
    return R.view(-1, 3, 3)


def _rotation(q4):
    q = q4.v.clone()
    q[:, 0] += 1.0
    nq = q.norm(dim=-1)
    en = q4.e.norm(dim=-1)
    en = LAMBDA * en
    L = torch.where(nq > en, 24.0 / (nq - en), torch.full_like(nq, float('inf')))
    # |R| <= 1 entry-wise for any q, so 2 bounds any error
    eR = (L * (LAMBDA * q4.e.amax(-1) + U32 * q[:, 0].abs()) + 2.0 ** -18).clamp_max(2.0)
    return quat_to_rot(q), eR[:, None, None].expand(-1, 3, 3)


def network(P, variant, patch, sub, query, model, R=None):
    """Float64 forward of the eval-mode network with its bound under `model`.

    P: `fold_params(...)` (moved to the device of the inputs); patch [B, P, 3], sub [B, S, 3], query [B, 3] float32
    tensors.  R [B, 3, 3] (optional): the rotation the engine computed, used for everything downstream of the
    quaternion.  -> dict of V: 'q4', 'feat_global_max', 'feat_local_max', 'logits'; 'R' = (float64 R, bound) or None."""
    m = MODELS[model]
    v = synth.VARIANTS[variant]
    patch, sub, query = patch.double(), sub.double(), query.double()
    out = {'q4': None, 'R': None}
    Rq = None
    if v['use_point_stn']:
        if v['shared_transformer']:
            pts = torch.cat([patch, sub - query.unsqueeze(1)], 1)
            q4 = _qstn(P, 'point_stn.', pts, None, m)
        else:
            q4 = _qstn(P, 'feat_global.stn1.', sub, query, m)
        out['q4'] = q4
        out['R'] = _rotation(q4)
        Rq = out['R'][0] if R is None else R.double()
    fg = _feat(P, 'feat_global.', sub, query, Rq, model)
    fl = _feat(P, 'feat_local.', patch, None, Rq, model)
    out['feat_global_max'], out['feat_local_max'] = fg, fl
    hl = _linear(fl, *P['fc1_local'], m['fc']).relu()
    hg = _linear(fg, *P['fc1_global'], m['fc']).relu()
    h = _linear(V(torch.cat([hl.v, hg.v], -1), torch.cat([hl.e, hg.e], -1)), *P['fc2'], m['fc']).relu()
    h = _linear(h, *P['fc3'], m['fc']).relu()
    out['logits'] = _linear(h, *P['fc4'], FP32_FC)
    return out


def to_device(P, device):
    return {k: (W.to(device), b.to(device)) for k, (W, b) in P.items()}


def excess(got, ref):
    """Error-to-bound ratio per element of `got` (float32 tensor) against V `ref` (ratio 0 where the error is 0)."""
    err = (got.double().to(ref.v.device) - ref.v).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / (LAMBDA * ref.e))
    return torch.where(torch.isfinite(got.to(ref.v.device)), r, torch.full_like(r, float('inf')))


def worst(ratio):
    """(max ratio, index tuple of the worst element) of an excess tensor."""
    i = int(torch.argmax(ratio))
    return float(ratio.reshape(-1)[i]), tuple(int(j) for j in np.unravel_index(i, tuple(ratio.shape)))
