"""TEST INFRASTRUCTURE ONLY -- sign propagation (source/sdf.py:114-202) restated in torch, so that it runs on the device
the volume is on and can check the CUDA kernel at 256^3 and 512^3, where the NumPy restatement (oracle/p2s_oracle.py)
takes minutes.

Every iteration is a full recomputation, exactly as the reference does it: the {-1, 0, 1} sign volume, its box sum with
'nearest' edges as clamped index gathers in int32 (exact), the |n| < thr rule and the two stop rules.  No work list, no
incremental counts, no packed bytes: nothing is shared with csrc/volume.cu but the definition."""
import torch


def box_sum_nearest(s, sigma):
    """convolve(s, ones(sigma^3), mode='nearest') for an integer-valued s: int32, separable, exact.  Output o sums the
    inputs o-hi .. o-lo (the flipped kernel), indices clamped to the volume."""
    lo, hi = -(sigma // 2), (sigma + 1) // 2 - 1
    out = s.to(torch.int32)
    for ax in range(3):
        n = out.shape[ax]
        ar = torch.arange(n, device=out.device)
        acc = torch.zeros_like(out)
        for d in range(lo, hi + 1):
            acc += out.index_select(ax, (ar - d).clamp_(0, n - 1))
        out = acc
    return out


def propagate_sign_torch(vol, sigma=5, thr=13):
    """source/sdf.py:114-178 on a float volume on any device -> (new volume, iterations).  `vol` is not modified."""
    vol = vol.clone()
    s = torch.sign(vol).to(torch.int8)
    unknown_initially = s == 0
    vol[0], vol[-1] = -1.0, -1.0
    vol[:, 0], vol[:, -1] = -1.0, -1.0
    vol[:, :, 0], vol[:, :, -1] = -1.0, -1.0
    # `np.abs(n) < certainty_threshold` compares int32 with a float64 scalar; a 0-dim float64 tensor makes torch compare
    # in float64 too, so thr <= 0, NaN and inf behave as in NumPy
    t = torch.tensor(float(thr), dtype=torch.float64, device=vol.device)
    it = 0
    while True:
        unknown_before = int((s == 0).sum())
        if unknown_before == 0:
            break
        n = box_sum_nearest(s, sigma)
        n = torch.where(n.abs() < t, torch.zeros_like(n), n).sign().to(torch.int8)
        if int((n == 0).sum()) >= unknown_before:
            break
        s = torch.where(unknown_initially, n, s)
        it += 1
    zero = vol == 0
    vol[zero] = s[zero].to(vol.dtype)
    return vol, it


def sdf_to_volume(lin, dist, res, sigma, thr):
    """source/sdf.py:187-202 with the query points given as linear voxel indices (ix*res+iy)*res+iz: scatter into a
    zero float32 volume, propagate, clamp to [-1, 1] -> (volume, iterations), or (None, -1) when every distance is 0
    (the reference returns without a volume).  float32 holds the reference's float64 volume exactly: its values are
    float32 distances and +-1."""
    lin = torch.as_tensor(lin).long()
    dist = torch.as_tensor(dist, dtype=torch.float32, device=lin.device)
    if bool((dist == 0).all()):
        return None, -1
    V = res ** 3
    assert bool(((lin >= 0) & (lin < V)).all()), 'voxel index outside [0, res^3)'
    vol = torch.zeros(V, dtype=torch.float32, device=lin.device)
    vol[lin] = dist
    vol, it = propagate_sign_torch(vol.view(res, res, res), sigma, thr)
    return vol.clamp_(-1.0, 1.0), it
