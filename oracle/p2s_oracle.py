"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the Points2Surf SDF-inference hot path.

This file is the *oracle* of SURVEY.md section 8(c).  It is a plain NumPy / SciPy / torch-CPU
restatement of the reference algorithm (each function cites the reference file:line under
/root/reference it follows).  It is imported only by tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs -- never by the product path
(points2surf_b200/), which must fail loudly when the CUDA library is missing.

Pinning status (see tests/golden/make_golden.py, which imports the real reference in the
build container and writes tests/golden/*.npz):
  * network forward (a7), post-process (a8)      -- pinned against the unmodified
    source/points_to_surf_model.py + source/sdf_nn.py (fp32 CPU).
  * candidate grid (a1), kNN patch (a4, a5), sub-sample (a6) -- pinned against the shimmed
    source/sdf.py, source/data_loader.py, source/base/{point_cloud,utils}.py.
  * scatter (a10), sign propagation (a11)        -- pinned against the shimmed source/sdf.py,
    bit-exact.
  * marching cubes + mesh clean-up (a12)         -- PARITY UNPINNED: the reference calls
    skimage.measure.marching_cubes_lewiner (scikit-image>=0.16, requirements.txt:3; removed
    upstream in 0.19) and trimesh (requirements.txt:13); neither is installed nor installable
    here.  `marching_cubes` below restates the published algorithm and is judged through the
    reference's Chamfer definition (source/base/evaluation.py:222-256, restated in `chamfer`).

Third-party arithmetic the reference itself delegates to (and that is present in this image)
is called, not re-derived: scipy.spatial.cKDTree (kNN), scipy.ndimage.convolve (box sums),
numpy.random.RandomState (sub-sampling).
"""
import numpy as np

# --------------------------------------------------------------------------------------
# a1: candidate query grid  -- source/sdf.py:46-79
# --------------------------------------------------------------------------------------


def model_space_to_volume_space(pts_ms, vol_res):
    """source/sdf.py:73-75.  NB float32 arithmetic when pts_ms is float32."""
    pts_pos_octant = (pts_ms + 1.0) / 2.0
    return np.floor(pts_pos_octant * vol_res).astype(int)


def volume_space_to_model_space(pts_vs, vol_res):
    """source/sdf.py:78-79 (float64 for integer input)."""
    return ((pts_vs + 0.5) / vol_res) * 2.0 - 1.0


def query_grid_indices(pts, grid_resolution, epsilon):
    """Voxel indices [Q,3] (C order == np.nonzero order) within an eps^3 box of any occupied
    voxel, last index plane on every axis dropped.  source/sdf.py:57-67."""
    from scipy.ndimage import convolve
    pts_vs = model_space_to_volume_space(pts, grid_resolution)
    vol = np.zeros((grid_resolution,) * 3, dtype=np.float32)
    vol[pts_vs[:, 0], pts_vs[:, 1], pts_vs[:, 2]] = 1.0
    kernel = np.ones((epsilon,) * 3, dtype=np.float32)
    near = convolve(vol, kernel, mode='nearest')
    return np.stack(np.nonzero(near[:-1, :-1, :-1]), axis=1)


def query_grid(pts, grid_resolution, epsilon):
    """source/sdf.py:46-70 -> float32 [Q,3] voxel centres in model space."""
    idx = query_grid_indices(pts, grid_resolution, epsilon)
    return volume_space_to_model_space(idx, grid_resolution).astype(np.float32)


def query_grid_indices_shifts(pts, grid_resolution, epsilon):
    """Same set as `query_grid_indices`, restated without scipy: an occupied voxel i marks the
    outputs i+d, d in [-floor(e/2), ceil(e/2)-1] per axis (SURVEY.md section 10, probe-verified)."""
    res = grid_resolution
    pts_vs = model_space_to_volume_space(pts, res)
    occ = np.zeros((res,) * 3, dtype=bool)
    occ[pts_vs[:, 0], pts_vs[:, 1], pts_vs[:, 2]] = True
    lo, hi = -(epsilon // 2), (epsilon + 1) // 2 - 1
    for ax in range(3):
        out = np.zeros_like(occ)
        for d in range(lo, hi + 1):
            src = [slice(None)] * 3
            dst = [slice(None)] * 3
            if d >= 0:
                src[ax] = slice(0, res - d)
                dst[ax] = slice(d, res)
            else:
                src[ax] = slice(-d, res)
                dst[ax] = slice(0, res + d)
            out[tuple(dst)] |= occ[tuple(src)]
        occ = out
    return np.stack(np.nonzero(occ[:-1, :-1, :-1]), axis=1)


# --------------------------------------------------------------------------------------
# a4 / a5: kNN patch, radius, patch-space normalisation
# --------------------------------------------------------------------------------------


def make_kdtree(pts):
    """source/data_loader.py:39-42 (leafsize 1000)."""
    import scipy.spatial as spatial
    return spatial.cKDTree(pts, 1000)


def knn_patch(pts, kdtree, query_point, k):
    """source/base/point_cloud.py:174-175 (kNN mode) + source/data_loader.py:340-350 +
    source/base/utils.py:62-69,80-88.
    Returns ids[k] int32 ascending by f64 distance, patch_pts_ps[k,3] f32, radius f32."""
    _, ids = kdtree.query(x=query_point, k=k)
    ids = np.array(ids, dtype=np.int32)
    pts_patch_ms = pts[ids, :]
    # get_patch_radii: cartesian_dist(repeat(query), pts_patch) = norm(q - p, axis=1); max
    dist = np.linalg.norm(np.repeat(np.expand_dims(query_point, 0), k, axis=0) - pts_patch_ms, axis=1)
    radius = np.max(dist, axis=0)
    patch_ps = (pts_patch_ms - np.repeat(np.expand_dims(query_point, 0), k, axis=-2)) / radius
    return ids, patch_ps.astype(np.float32), np.float32(radius)


def ball_patch(pts, kdtree, query_point, patch_radius, points_per_patch, rng):
    """Ball-query patch: source/base/point_cloud.py:176-192 (all points within patch_radius; a random subset when there
    are too many -- consumes `rng` like the reference's dataset rng; -1 padding when there are too few) followed by the
    padding rule and the fixed-radius normalisation of source/data_loader.py:340-350.
    Returns (ids [P] int32 with pads set to 0, patch_pts_ps [P,3] f32, in-ball count)."""
    ids = np.array(kdtree.query_ball_point(x=query_point, r=patch_radius), dtype=np.int32)
    count = ids.shape[0]
    if count > points_per_patch:
        ids = ids[rng.choice(np.arange(count), points_per_patch, replace=False)]
    if count < points_per_patch:
        padding = np.full((points_per_patch - count), -1, dtype=np.int32)
        ids = padding if count == 0 else np.concatenate((ids, padding), axis=0)
    pad = ids == -1
    ids[pad] = 0
    pts_patch_ms = pts[ids, :]
    pts_patch_ms[pad, :] = query_point
    rep = np.repeat(np.expand_dims(query_point, axis=0), pts_patch_ms.shape[-2], axis=-2)
    patch_ps = (pts_patch_ms - rep) / patch_radius
    return ids, patch_ps.astype(np.float32), count


def knn_bruteforce(pts, query_point, k):
    """Restatement of what cKDTree.query computes: Euclidean distances evaluated in float64 on
    the float32 coordinates; k smallest, ascending.  Returns (ids, d2_f64) with ties broken by id."""
    d = pts.astype(np.float64) - query_point.astype(np.float64)[None, :]
    d2 = (d * d).sum(axis=1)
    order = np.lexsort((np.arange(len(d2)), d2))[:k]
    return order.astype(np.int32), d2[order]


# --------------------------------------------------------------------------------------
# a6: global sub-sample  -- source/base/utils.py:196-227
# --------------------------------------------------------------------------------------


def sub_sample_weights(pts_ms, query_point_ms):
    """The unnormalised weights of source/base/utils.py:200-207 (float32 arithmetic like the reference)."""
    query_pts = np.broadcast_to(query_point_ms, pts_ms.shape)
    dist = np.linalg.norm(query_pts - pts_ms, axis=1)
    dist_normalized = dist / np.max(dist)
    prob = 1.0 - 1.5 * dist_normalized
    return np.clip(prob, 0.05, 1.0)


def sub_sample_probabilities(pts_ms, query_point_ms):
    """source/base/utils.py:200-208 (float32 arithmetic like the reference)."""
    prob_clipped = sub_sample_weights(pts_ms, query_point_ms)
    return prob_clipped / np.sum(prob_clipped)


def sub_sample_ids(sub_sample_size, pts_ms, query_point_ms, rng, uniform=False, fixed=False):
    """source/base/utils.py:196-219 for N >= sub_sample_size; returns the indices (the reference
    returns pts_ms[ids])."""
    if pts_ms.shape[0] < sub_sample_size:
        raise ValueError('oracle: N < sub_sample_size (reference shuffles the cloud in place, utils.py:222-226)')
    if fixed:
        rng.seed(42)
    if uniform:
        return rng.randint(low=0, high=pts_ms.shape[0], size=sub_sample_size)
    prob = sub_sample_probabilities(pts_ms, query_point_ms)
    return rng.choice(pts_ms.shape[0], size=sub_sample_size, replace=False, p=prob)


def assemble_query(pts, kdtree, query_point, k, sub_sample_size, rng_global, uniform):
    """One query's model inputs in reconstruction mode -- source/data_loader.py:322-421."""
    ids, patch_ps, radius = knn_patch(pts, kdtree, query_point, k)
    sids = sub_sample_ids(sub_sample_size, pts, query_point, rng_global, uniform=uniform)
    return dict(patch_pts_ids=ids, patch_pts_ps=patch_ps, patch_radius_ms=radius,
                sub_sample_ids=np.asarray(sids, dtype=np.int64), pts_sub_sample_ms=pts[sids, :],
                imp_surf_query_point_ms=query_point)


# --------------------------------------------------------------------------------------
# a7: network forward  -- source/points_to_surf_model.py:296-352 (eval mode)
# --------------------------------------------------------------------------------------


def _t(sd, name):
    import torch
    v = sd[name]
    return v if isinstance(v, torch.Tensor) else torch.from_numpy(np.asarray(v))


_CONV_TF32 = False   # set (temporarily) by model_forward(conv_tf32=True)


def _round_tf32(t):
    """Round-to-nearest-even to TF32 (10 explicit mantissa bits): what the tensor cores behind cuDNN's default
    `torch.backends.cudnn.allow_tf32 = True` Conv1d path do to both conv operands on Ampere and later."""
    import torch
    i = t.contiguous().view(torch.int32)
    i = (i + 0x0FFF + ((i >> 13) & 1)) & ~0x1FFF
    return i.view(torch.float32)


def _conv_bn(sd, x, conv, bn, relu=True):
    import torch.nn.functional as F
    w = _t(sd, conv + '.weight')
    if _CONV_TF32:
        x, w = _round_tf32(x), _round_tf32(w)
    y = F.conv1d(x, w, _t(sd, conv + '.bias'))
    y = F.batch_norm(y, _t(sd, bn + '.running_mean'), _t(sd, bn + '.running_var'),
                     _t(sd, bn + '.weight'), _t(sd, bn + '.bias'), training=False, eps=1e-5)
    return F.relu(y) if relu else y


def _fc_bn(sd, x, fc, bn=None, relu=True):
    import torch.nn.functional as F
    y = F.linear(x, _t(sd, fc + '.weight'), _t(sd, fc + '.bias'))
    if bn is not None:
        y = F.batch_norm(y, _t(sd, bn + '.running_mean'), _t(sd, bn + '.running_var'),
                         _t(sd, bn + '.weight'), _t(sd, bn + '.bias'), training=False, eps=1e-5)
    return F.relu(y) if relu else y


def quat_to_rotmat(q):
    """source/base/utils.py:13-46: s = 2/sum(q^2); the quaternion is NOT normalised first."""
    import torch
    s = 2 / torch.sum(q.pow(2), 1)
    h = torch.bmm(q.unsqueeze(2), q.unsqueeze(1))
    out = q.new_empty(q.size(0), 3, 3)
    out[:, 0, 0] = 1 - (h[:, 2, 2] + h[:, 3, 3]).mul(s)
    out[:, 0, 1] = (h[:, 1, 2] - h[:, 3, 0]).mul(s)
    out[:, 0, 2] = (h[:, 1, 3] + h[:, 2, 0]).mul(s)
    out[:, 1, 0] = (h[:, 1, 2] + h[:, 3, 0]).mul(s)
    out[:, 1, 1] = 1 - (h[:, 1, 1] + h[:, 3, 3]).mul(s)
    out[:, 1, 2] = (h[:, 2, 3] - h[:, 1, 0]).mul(s)
    out[:, 2, 0] = (h[:, 1, 3] - h[:, 2, 0]).mul(s)
    out[:, 2, 1] = (h[:, 2, 3] + h[:, 1, 0]).mul(s)
    out[:, 2, 2] = 1 - (h[:, 1, 1] + h[:, 2, 2]).mul(s)
    return out


def _qstn(sd, p, x):
    """QSTN.forward, source/points_to_surf_model.py:100-131 (num_scales == 1)."""
    import torch
    x = _conv_bn(sd, x, p + 'conv1', p + 'bn1')
    x = _conv_bn(sd, x, p + 'conv2', p + 'bn2')
    x = _conv_bn(sd, x, p + 'conv3', p + 'bn3')
    x = torch.max(x, dim=2)[0]
    x = _fc_bn(sd, x, p + 'fc1', p + 'bn4')
    x = _fc_bn(sd, x, p + 'fc2', p + 'bn5')
    x = _fc_bn(sd, x, p + 'fc3', None, relu=False)
    quat = x + x.new_tensor([1, 0, 0, 0])
    return quat_to_rotmat(quat), quat


def _stn64(sd, p, x):
    """STN.forward with dim=64, source/points_to_surf_model.py:41-69."""
    import torch
    b = x.size(0)
    x = _conv_bn(sd, x, p + 'conv1', p + 'bn1')
    x = _conv_bn(sd, x, p + 'conv2', p + 'bn2')
    x = _conv_bn(sd, x, p + 'conv3', p + 'bn3')
    x = torch.max(x, dim=2)[0]
    x = _fc_bn(sd, x, p + 'fc1', p + 'bn4')
    x = _fc_bn(sd, x, p + 'fc2', p + 'bn5')
    x = _fc_bn(sd, x, p + 'fc3', None, relu=False)
    x = x + torch.eye(64, dtype=x.dtype).view(1, 64 * 64).repeat(b, 1)
    return x.view(-1, 64, 64)


def _pointnetfeat(sd, p, x, point_stn):
    """PointNetfeat.forward, source/points_to_surf_model.py:177-234 (num_scales 1, sym_op max)."""
    import torch
    trans = None
    if point_stn:
        trans, _ = _qstn(sd, p + 'stn1.', x)
        x = torch.bmm(trans, x)
    x = _conv_bn(sd, x, p + 'conv0a', p + 'bn0a')
    x = _conv_bn(sd, x, p + 'conv0b', p + 'bn0b')
    trans2 = _stn64(sd, p + 'stn2.', x)
    x = torch.bmm(trans2, x)
    x = _conv_bn(sd, x, p + 'conv1', p + 'bn1')
    x = _conv_bn(sd, x, p + 'conv2', p + 'bn2')
    x = _conv_bn(sd, x, p + 'conv3', p + 'bn3', relu=False)
    return torch.max(x, dim=2)[0], trans


def _model_forward_impl(sd, patch_pts_ps, pts_sub_sample_ms, imp_surf_query_point_ms,
                  use_point_stn=True, shared_transformer=True, return_aux=False):
    """PointsToSurfModel.forward in eval mode (single_transformer=0, use_feat_stn=1, sym_op='max').
    `sd` is a reference-named state dict WITHOUT the 'module.' prefix.  Inputs are [B,P,3],
    [B,S,3], [B,3] float32 arrays/tensors; pts_sub_sample_ms is NOT modified (the reference centres
    it in place, points_to_surf_model.py:303).  Returns [B,2] float32 logits (numpy)."""
    import torch
    as_t = lambda a: a.clone() if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))
    patch = as_t(patch_pts_ps).float().transpose(1, 2)
    shape = as_t(pts_sub_sample_ms).float().transpose(1, 2)
    q = as_t(imp_surf_query_point_ms).float().unsqueeze(2)
    shape = shape - q.expand(shape.shape)                                   # :303
    aux = {}
    if use_point_stn and shared_transformer:                                 # :325-331
        feats = torch.cat((patch, shape), dim=2)
        trans, quat = _qstn(sd, 'point_stn.', feats)
        shape = torch.bmm(trans, shape)
        patch = torch.bmm(trans, patch)
        aux['trans'] = trans.numpy()
        aux['quat'] = quat.numpy()
    shape_feat, trans_global = _pointnetfeat(sd, 'feat_global.', shape,      # :333-335
                                             bool(use_point_stn and not shared_transformer))
    aux['feat_global_max'] = shape_feat.numpy()
    shape_feat = _fc_bn(sd, shape_feat, 'fc1_global', 'bn1_global')
    if use_point_stn and not shared_transformer:                             # :337-339
        patch = torch.bmm(trans_global, patch)
    patch_feat, _ = _pointnetfeat(sd, 'feat_local.', patch, False)           # :341-343
    aux['feat_local_max'] = patch_feat.numpy()
    patch_feat = _fc_bn(sd, patch_feat, 'fc1_local', 'bn1_local')
    x = torch.cat((patch_feat, shape_feat), dim=1)                           # :346
    x = _fc_bn(sd, x, 'fc2', 'bn2')
    x = _fc_bn(sd, x, 'fc3', 'bn3')
    aux['fc3_out'] = x.numpy()
    x = _fc_bn(sd, x, 'fc4', None, relu=False)
    out = x.numpy()
    return (out, aux) if return_aux else out


def model_forward(sd, patch_pts_ps, pts_sub_sample_ms, imp_surf_query_point_ms,
                  use_point_stn=True, shared_transformer=True, return_aux=False, conv_tf32=False):
    """PointsToSurfModel.forward in eval mode, without autograd (see _model_forward_impl).
    conv_tf32=True emulates the reference's stock GPU arithmetic on Ampere+ (cuDNN Conv1d with TF32 operands,
    fp32 accumulate; nn.Linear / bmm stay fp32 because torch.backends.cuda.matmul.allow_tf32 defaults to False):
    the yardstick for the tensor-core engine's own deviation from the fp32 result."""
    import torch
    global _CONV_TF32
    prev, _CONV_TF32 = _CONV_TF32, bool(conv_tf32)
    try:
        with torch.no_grad():
            return _model_forward_impl(sd, patch_pts_ps, pts_sub_sample_ms, imp_surf_query_point_ms, use_point_stn,
                                       shared_transformer, return_aux)
    finally:
        _CONV_TF32 = prev


# --------------------------------------------------------------------------------------
# a8: post-process  -- source/sdf_nn.py:11-21, source/points_to_surf_eval.py:184-196,263-271
# --------------------------------------------------------------------------------------


def post_process(logits, patch_radius):
    """|d| = tanh(p0)^2 * r ; sign = +1 if p1 >= 0 else -1 ; sdf = |d| * sign  (float32).
    NaN -> 1.0 as in save_reconstruction_data (points_to_surf_eval.py:205-207)."""
    import torch
    lg = torch.from_numpy(np.asarray(logits, dtype=np.float32))
    r = torch.from_numpy(np.asarray(patch_radius, dtype=np.float32))
    mag = torch.tanh(lg[:, 0]).pow(2) * r
    sign = torch.where(lg[:, 1] >= 0.0, torch.ones_like(mag), -torch.ones_like(mag))
    sdf = (mag * sign).numpy()
    sdf[np.isnan(sdf)] = 1.0
    return sdf


# --------------------------------------------------------------------------------------
# a10 / a11: scatter + sign propagation  -- source/sdf.py:82-178
# --------------------------------------------------------------------------------------


def add_samples_to_volume(vol, pos_ms, val):
    """source/sdf.py:82-111 for the reconstruction case (query points are voxel centres, one
    sample per voxel, lexicographically sorted): degenerates to a scatter."""
    pos_vs = model_space_to_volume_space(pos_ms, vol.shape[0])
    vol[pos_vs[:, 0], pos_vs[:, 1], pos_vs[:, 2]] = val
    return vol


def _box_sum_nearest(s, sigma):
    """convolve(s, ones(sigma^3), mode='nearest') for integer-valued s, separable, exact."""
    lo, hi = -(sigma // 2), (sigma + 1) // 2 - 1   # output o sums inputs o-hi .. o-lo  (flipped kernel)
    out = s.astype(np.int32)
    for ax in range(3):
        n = out.shape[ax]
        acc = np.zeros_like(out)
        for d in range(lo, hi + 1):
            idx = np.clip(np.arange(n) - d, 0, n - 1)
            acc += np.take(out, idx, axis=ax)
        out = acc
    return out


def propagate_sign(vol, sigma=5, certainty_threshold=13):
    """source/sdf.py:114-178, restated on integer sign volumes (box sums of {-1,0,1} are exact
    integers in the reference's float32/float64 arithmetic as well).  Returns (vol, iterations)."""
    s = np.sign(vol).astype(np.int8)
    unknown_initially = s == 0
    vol[+0, :, :] = -1.0
    vol[-1, :, :] = -1.0
    vol[:, +0, :] = -1.0
    vol[:, -1, :] = -1.0
    vol[:, :, +0] = -1.0
    vol[:, :, -1] = -1.0
    it = 0
    while True:
        unknown_before = int((s == 0).sum())
        if unknown_before == 0:
            break
        n = _box_sum_nearest(s, sigma)
        n[np.abs(n) < certainty_threshold] = 0
        n = np.sign(n).astype(np.int8)
        if int((n == 0).sum()) >= unknown_before:
            break
        s[unknown_initially] = n[unknown_initially]
        it += 1
    zero = vol == 0
    vol[zero] = s[zero]
    return vol, it


def sdf_to_volume(query_dist_ms, query_pts_ms, grid_res, sigma, certainty_threshold):
    """source/sdf.py:187-202: zeros(res^3) float64, scatter, propagate, clamp to [-1,1].
    Returns None when all distances are exactly 0 (sdf.py:187-189)."""
    if query_dist_ms.max() == 0.0 and query_dist_ms.min() == 0.0:
        return None
    volume = np.zeros((grid_res,) * 3)
    volume = add_samples_to_volume(volume, query_pts_ms, query_dist_ms)
    volume, _ = propagate_sign(volume, sigma, certainty_threshold)
    volume[volume < -1.0] = -1.0
    volume[volume > 1.0] = 1.0
    return volume


# --------------------------------------------------------------------------------------
# acceptance metric: Chamfer  -- source/base/evaluation.py:222-256
# --------------------------------------------------------------------------------------


def sample_mesh_surface(verts, faces, num_samples, rng):
    """Area-weighted uniform surface sampling (what trimesh.sample.sample_surface does; the
    reference uses sample_surface_even, evaluation.py:235, which additionally rejects samples
    closer than a radius -- a variance reduction, not a change of the estimated quantity)."""
    v0, v1, v2 = verts[faces[:, 0]], verts[faces[:, 1]], verts[faces[:, 2]]
    area = 0.5 * np.linalg.norm(np.cross(v1 - v0, v2 - v0), axis=1)
    cdf = np.cumsum(area)
    f = np.searchsorted(cdf, rng.random_sample(num_samples) * cdf[-1])
    f = np.minimum(f, len(faces) - 1)
    r1, r2 = rng.random_sample(num_samples), rng.random_sample(num_samples)
    flip = r1 + r2 > 1.0
    r1[flip], r2[flip] = 1.0 - r1[flip], 1.0 - r2[flip]
    return v0[f] + r1[:, None] * (v1[f] - v0[f]) + r2[:, None] * (v2[f] - v0[f])


def chamfer(new_samples, ref_samples):
    """sum of nearest-neighbour distances in both directions, evaluation.py:244-254."""
    import scipy.spatial as spatial
    kd_new = spatial.cKDTree(new_samples, 100)
    kd_ref = spatial.cKDTree(ref_samples, 100)
    ref_new, _ = kd_new.query(ref_samples, 1)
    new_ref, _ = kd_ref.query(new_samples, 1)
    return float(np.sum(ref_new) + np.sum(new_ref))


def hausdorff(new_samples, ref_samples):
    """(directed new->ref, directed ref->new, symmetric) -- source/base/evaluation.py:301-304 (scipy's
    directed_hausdorff is max-min of exact Euclidean distances; restated through cKDTree for speed)."""
    import scipy.spatial as spatial
    d_new_ref, _ = spatial.cKDTree(ref_samples).query(new_samples, 1)
    d_ref_new, _ = spatial.cKDTree(new_samples).query(ref_samples, 1)
    a, b = float(d_new_ref.max()), float(d_ref_new.max())
    return a, b, max(a, b)
