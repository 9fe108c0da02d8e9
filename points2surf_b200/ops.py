"""Tensor-level wrappers over the C ABI.  PyTorch is used for device memory and streams only;
every computation happens in libp2s_b200.so.  All functions require CUDA tensors and raise otherwise."""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import ModelConfig, ReconConfig, P2SError, check
from . import weights as _weights


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dev(t, dtype, name):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise P2SError('%s must be a CUDA tensor (points2surf_b200 has no CPU path)' % name)
    if t.dtype != dtype:
        raise P2SError('%s must have dtype %s, got %s' % (name, dtype, t.dtype))
    return t.contiguous()


def _ptr(t):
    return C.c_void_p(t.data_ptr())


class Engine:
    """Device-resident model (replaces make_regressor, source/points_to_surf_eval.py:150-171)."""

    def __init__(self, state_dict, use_point_stn, shared_transformer, points_per_patch=300,
                 sub_sample_size=1000, net_size=1024, device=0, precision='fp32', guard_band=0.0, output_dim=2,
                 single_transformer=False):
        """output_dim 2: logits (|d| logit, sign logit); output_dim 1: the regression head's signed-distance logit.
        reconstruct() applies the matching post-process.  single_transformer: the shared-encoder ablation (one
        feat_local_global over patch + sub-sample; needs use_point_stn and no shared_transformer)."""
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise P2SError('CUDA is not available: points2surf_b200 has no CPU fallback')
        self.device = torch.device('cuda', device if isinstance(device, int) else torch.device(device).index or 0)
        self.cfg = ModelConfig(int(bool(use_point_stn)), int(bool(shared_transformer)), int(points_per_patch),
                               int(sub_sample_size), int(net_size))
        self.output_dim = int(output_dim)
        self.single_transformer = int(bool(single_transformer))
        blob = _weights.pack_blob(state_dict, use_point_stn, shared_transformer, self.output_dim, self.single_transformer)
        expect = self.lib.p2s_model_blob_floats_enc(C.byref(self.cfg), self.output_dim, self.single_transformer)
        if blob.size != expect:
            raise P2SError('state_dict does not match the model config (%d floats, expected %d)' % (blob.size, expect))
        h = C.c_void_p()
        check(self.lib.p2s_model_create_enc(C.byref(self.cfg), self.output_dim, self.single_transformer,
                                            blob.ctypes.data_as(C.c_void_p), blob.size, self.device.index, C.byref(h)))
        self.handle = h
        self.P, self.S = int(points_per_patch), int(sub_sample_size)
        self.set_precision(precision, guard_band)

    def set_precision(self, precision, guard_band=0.0):
        p = {'fp32': _lib.PRECISION_FP32, 'tc': _lib.PRECISION_TC}[precision]
        check(self.lib.p2s_model_set_precision(self.handle, p, float(guard_band)))
        self.precision = precision

    def close(self):
        if getattr(self, 'handle', None):
            self.lib.p2s_model_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def forward_with_aux(self, patch_pts_ps, pts_sub_sample_ms, imp_surf_query_point_ms):
        """-> (logits, dict(trans [B,3,3], feat_local_max [B,1024], feat_global_max [B,1024])) -- parity diagnostics.
        A single_transformer engine has one encoder: dict(trans [B,3,3], feat_max [B,1024])."""
        B = patch_pts_ps.shape[0]
        aux = torch.zeros((B, 2064), dtype=torch.float32, device=patch_pts_ps.device)
        check(self.lib.p2s_model_set_debug_aux(self.handle, _ptr(aux)))
        try:
            out = self.forward(patch_pts_ps, pts_sub_sample_ms, imp_surf_query_point_ms)
            torch.cuda.synchronize()
        finally:
            check(self.lib.p2s_model_set_debug_aux(self.handle, None))
        if self.single_transformer:
            return out, {'trans': aux[:, :9].reshape(B, 3, 3), 'feat_max': aux[:, 9:1033]}
        return out, {'trans': aux[:, :9].reshape(B, 3, 3), 'feat_local_max': aux[:, 9:1033], 'feat_global_max': aux[:, 1033:2057]}

    def profile_enable(self, on=True):
        check(self.lib.p2s_profile_enable(self.handle, int(bool(on))))

    def profile_get(self):
        ms, n, fl = C.c_double(), C.c_int64(), C.c_double()
        check(self.lib.p2s_profile_get(self.handle, C.byref(ms), C.byref(n), C.byref(fl)))
        return {'ms': ms.value, 'launches': n.value, 'flops': fl.value, 'kernel': 'pointnet_pass_kernel'}

    def last_guard_count(self):
        n = C.c_int64()
        check(self.lib.p2s_model_last_guard_count(self.handle, C.byref(n)))
        return n.value

    # ---- a7 ----
    def forward(self, patch_pts_ps, pts_sub_sample_ms, imp_surf_query_point_ms):
        pa = _dev(patch_pts_ps, torch.float32, 'patch_pts_ps')
        su = _dev(pts_sub_sample_ms, torch.float32, 'pts_sub_sample_ms')
        qu = _dev(imp_surf_query_point_ms, torch.float32, 'imp_surf_query_point_ms')
        B = pa.shape[0]
        if pa.shape != (B, self.P, 3) or su.shape != (B, self.S, 3) or qu.shape != (B, 3):
            raise P2SError('bad input shapes %s %s %s' % (tuple(pa.shape), tuple(su.shape), tuple(qu.shape)))
        out = torch.empty((B, self.output_dim), dtype=torch.float32, device=pa.device)
        if B == 0:
            return out
        with torch.cuda.device(pa.device):
            check(self.lib.p2s_forward_dev(self.handle, _ptr(pa), _ptr(su), _ptr(qu), B, _ptr(out), _stream()))
        return out

    def forward_host(self, patch_pts_ps, pts_sub_sample_ms, imp_surf_query_point_ms):
        pa = np.ascontiguousarray(patch_pts_ps, dtype=np.float32)
        su = np.ascontiguousarray(pts_sub_sample_ms, dtype=np.float32)
        qu = np.ascontiguousarray(imp_surf_query_point_ms, dtype=np.float32)
        B = pa.shape[0]
        out = np.empty((B, self.output_dim), dtype=np.float32)
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        check(self.lib.p2s_forward_host(self.handle, vp(pa), vp(su), vp(qu), B, vp(out)))
        return out

    def post_process(self, logits, patch_radius):
        """The post-process of this model's head: sdf_from_logits (output_dim 2) or distance_from_logits (output_dim 1)."""
        return (distance_from_logits if self.output_dim == 1 else sdf_from_logits)(logits, patch_radius)

    # ---- fused a1..a9 ----
    def reconstruct(self, pts, res, eps, uniform_subsample, seed, first_query=0, num_queries=-1, batch=0, cap=None,
                    patch_radius=0.0):
        """patch_radius > 0: ball-query patches of that radius and un-scaled magnitudes (train_opt.patch_radius)."""
        pts = _dev(pts, torch.float32, 'pts')
        N = pts.shape[0]
        if cap is None:
            cap = query_grid(pts, res, eps).numel() if num_queries < 0 else num_queries
        rc = ReconConfig(int(res), int(eps), _lib.SUBSAMPLE_UNIFORM if uniform_subsample else _lib.SUBSAMPLE_WEIGHTED,
                         int(batch), int(seed) & (2**64 - 1), float(patch_radius), 0)
        lin = torch.empty((max(cap, 1),), dtype=torch.int32, device=pts.device)
        sdf = torch.empty((max(cap, 1),), dtype=torch.float32, device=pts.device)
        Q = C.c_int64()
        with torch.cuda.device(pts.device):
            check(self.lib.p2s_reconstruct_dev(self.handle, C.byref(rc), _ptr(pts), N, int(first_query), int(num_queries),
                                               _ptr(lin), _ptr(sdf), int(cap), C.byref(Q), _stream()))
        return lin[:Q.value], sdf[:Q.value]

    def reconstruct_host(self, pts_np, res, eps, uniform_subsample, seed, cap, batch=0, out_lin=None, out_sdf=None,
                         patch_radius=0.0):
        pts_np = np.ascontiguousarray(pts_np, dtype=np.float32)
        rc = ReconConfig(int(res), int(eps), _lib.SUBSAMPLE_UNIFORM if uniform_subsample else _lib.SUBSAMPLE_WEIGHTED,
                         int(batch), int(seed) & (2**64 - 1), float(patch_radius), 0)
        lin = out_lin if out_lin is not None else np.empty((cap,), dtype=np.int32)
        sdf = out_sdf if out_sdf is not None else np.empty((cap,), dtype=np.float32)
        Q = C.c_int64()
        vp = lambda a: a.ctypes.data_as(C.c_void_p)
        check(self.lib.p2s_reconstruct_host(self.handle, C.byref(rc), vp(pts_np), pts_np.shape[0], vp(lin), vp(sdf),
                                            int(cap), C.byref(Q)))
        return lin[:Q.value], sdf[:Q.value]


def launch_count(reset=False):
    lib = _lib.load()
    n = lib.p2s_launch_count()
    if reset:
        lib.p2s_launch_count_reset()
    return int(n)


def sdf_from_logits(logits, patch_radius):
    """patch_radius None = fixed-radius patches: the magnitude is not rescaled (points_to_surf_eval.py:364-368)."""
    lg = _dev(logits, torch.float32, 'logits')
    r = _dev(patch_radius, torch.float32, 'patch_radius') if patch_radius is not None else None
    out = torch.empty((lg.shape[0],), dtype=torch.float32, device=lg.device)
    with torch.cuda.device(lg.device):
        check(_lib.load().p2s_sdf_from_logits_dev(_ptr(lg), _ptr(r) if r is not None else None, lg.shape[0], _ptr(out), _stream()))
    return out


def distance_from_logits(logits, patch_radius):
    """Regression head (outputs imp_surf): logits [B,1] -> tanh(l)^2 * sign(l) * radius, NaN -> 1
    (source/sdf_nn.py:6-8, points_to_surf_eval.py:176-183,205-207).  patch_radius None = fixed-radius patches: not rescaled."""
    lg = _dev(logits, torch.float32, 'logits')
    if lg.dim() != 2 or lg.shape[1] != 1:
        raise P2SError('logits must have shape [B, 1], got %s' % (tuple(lg.shape),))
    r = _dev(patch_radius, torch.float32, 'patch_radius') if patch_radius is not None else None
    if r is not None and r.shape != (lg.shape[0],):
        raise P2SError('patch_radius must have shape [B]')
    out = torch.empty((lg.shape[0],), dtype=torch.float32, device=lg.device)
    with torch.cuda.device(lg.device):
        check(_lib.load().p2s_distance_from_logits_dev(_ptr(lg), _ptr(r) if r is not None else None, lg.shape[0], _ptr(out),
                                                        _stream()))
    return out


def query_grid(pts, res, eps):
    """-> int32 linear voxel indices (ix*res+iy)*res+iz in np.nonzero order (source/sdf.py:46-70)."""
    pts = _dev(pts, torch.float32, 'pts')
    lib = _lib.load()
    n = C.c_int64()
    with torch.cuda.device(pts.device):
        check(lib.p2s_query_grid_dev(_ptr(pts), pts.shape[0], int(res), int(eps), None, 0, C.byref(n), _stream()))
        out = torch.empty((max(n.value, 1),), dtype=torch.int32, device=pts.device)
        check(lib.p2s_query_grid_dev(_ptr(pts), pts.shape[0], int(res), int(eps), _ptr(out), n.value, C.byref(n), _stream()))
    return out[:n.value]


def query_points(lin_idx, res):
    lin = _dev(lin_idx, torch.int32, 'lin_idx')
    out = torch.empty((lin.shape[0], 3), dtype=torch.float32, device=lin.device)
    with torch.cuda.device(lin.device):
        check(_lib.load().p2s_query_points_dev(_ptr(lin), lin.shape[0], int(res), _ptr(out), _stream()))
    return out


def knn_patch(pts, query_pts, k):
    pts = _dev(pts, torch.float32, 'pts')
    q = _dev(query_pts, torch.float32, 'query_pts')
    Q = q.shape[0]
    ids = torch.empty((Q, k), dtype=torch.int32, device=pts.device)
    patch = torch.empty((Q, k, 3), dtype=torch.float32, device=pts.device)
    radius = torch.empty((Q,), dtype=torch.float32, device=pts.device)
    with torch.cuda.device(pts.device):
        check(_lib.load().p2s_knn_patch_dev(_ptr(pts), pts.shape[0], _ptr(q), Q, int(k), _ptr(ids), _ptr(patch),
                                            _ptr(radius), _stream()))
    return ids, patch, radius


def ball_patch(pts, query_pts, k, patch_radius, seed, query_index_base=0):
    """Ball-query patches (source/base/point_cloud.py:176-192 + data_loader.py:340-350)
    -> (ids [Q,k] (pads 0), patch_pts_ps [Q,k,3] (pads at the origin), radius [Q] = patch_radius, in-ball counts [Q])."""
    pts = _dev(pts, torch.float32, 'pts')
    q = _dev(query_pts, torch.float32, 'query_pts')
    Q = q.shape[0]
    ids = torch.empty((Q, k), dtype=torch.int32, device=pts.device)
    patch = torch.empty((Q, k, 3), dtype=torch.float32, device=pts.device)
    radius = torch.empty((Q,), dtype=torch.float32, device=pts.device)
    counts = torch.empty((Q,), dtype=torch.int32, device=pts.device)
    with torch.cuda.device(pts.device):
        check(_lib.load().p2s_ball_patch_dev(_ptr(pts), pts.shape[0], _ptr(q), Q, int(query_index_base), int(k), float(patch_radius),
                                             int(seed) & (2**64 - 1), _ptr(ids), _ptr(patch), _ptr(radius), _ptr(counts), _stream()))
    return ids, patch, radius, counts


def subsample(pts, query_pts, S, uniform, seed, query_index_base=0):
    pts = _dev(pts, torch.float32, 'pts')
    q = _dev(query_pts, torch.float32, 'query_pts')
    Q = q.shape[0]
    ids = torch.empty((Q, S), dtype=torch.int32, device=pts.device)
    mode = _lib.SUBSAMPLE_UNIFORM if uniform else _lib.SUBSAMPLE_WEIGHTED
    with torch.cuda.device(pts.device):
        check(_lib.load().p2s_subsample_dev(_ptr(pts), pts.shape[0], _ptr(q), Q, int(query_index_base), int(S), mode,
                                            int(seed) & (2**64 - 1), _ptr(ids), _stream()))
    return ids


def gather_points(pts, ids):
    pts = _dev(pts, torch.float32, 'pts')
    ids = _dev(ids, torch.int32, 'ids')
    out = torch.empty(tuple(ids.shape) + (3,), dtype=torch.float32, device=pts.device)
    with torch.cuda.device(pts.device):
        check(_lib.load().p2s_gather_points_dev(_ptr(pts), _ptr(ids), ids.numel(), _ptr(out), _stream()))
    return out


def sdf_to_volume(lin_idx, sdf, res, sigma, certainty_threshold):
    """-> (vol [res,res,res] fp32 clamped to [-1,1], iterations); iterations == -1 when all samples are 0
    (the reference returns without output, source/sdf.py:187-189)."""
    lin = _dev(lin_idx, torch.int32, 'lin_idx')
    sd = _dev(sdf, torch.float32, 'sdf')
    vol = torch.empty((res, res, res), dtype=torch.float32, device=lin.device)
    it = C.c_int()
    with torch.cuda.device(lin.device):
        check(_lib.load().p2s_sdf_to_volume_dev(_ptr(lin), _ptr(sd), lin.shape[0], int(res), int(sigma),
                                                float(certainty_threshold), _ptr(vol), C.byref(it), _stream()))
    return vol, it.value


def marching_cubes(vol, level=0.0):
    """-> (verts [V,3] fp32 model space, faces [F,3] int32)."""
    vol = _dev(vol, torch.float32, 'vol')
    res = vol.shape[0]
    lib = _lib.load()
    nv, nf = C.c_int64(), C.c_int64()
    with torch.cuda.device(vol.device):
        check(lib.p2s_marching_cubes_dev(_ptr(vol), res, float(level), None, 0, None, 0, C.byref(nv), C.byref(nf), _stream()))
        verts = torch.empty((max(nv.value, 1), 3), dtype=torch.float32, device=vol.device)
        faces = torch.empty((max(nf.value, 1), 3), dtype=torch.int32, device=vol.device)
        check(lib.p2s_marching_cubes_dev(_ptr(vol), res, float(level), _ptr(verts), nv.value, _ptr(faces), nf.value,
                                         C.byref(nv), C.byref(nf), _stream()))
    return verts[:nv.value], faces[:nf.value]


def mesh_sample(verts, faces, num_samples, seed=0, return_face_ids=False):
    """Area-weighted surface samples [n,3] fp32 (the sampler of source/base/evaluation.py:229-238)."""
    verts = _dev(verts, torch.float32, 'verts')
    faces = _dev(faces, torch.int32, 'faces')
    n = int(num_samples)
    out = torch.empty((n, 3), dtype=torch.float32, device=verts.device)
    fid = torch.empty((n,), dtype=torch.int32, device=verts.device) if return_face_ids else None
    with torch.cuda.device(verts.device):
        check(_lib.load().p2s_mesh_sample_dev(_ptr(verts), verts.shape[0], _ptr(faces), faces.shape[0], n,
                                              int(seed) & (2**64 - 1), _ptr(out), _ptr(fid) if fid is not None else None,
                                              _stream()))
    return (out, fid) if return_face_ids else out


def mesh_signed_distance(verts, faces, query, return_face_ids=False, return_winding=False):
    """Signed distance [Q] fp32 from every query point to the mesh, positive inside (the generalised winding number > 0.5)
    and on the surface (|d| <= 1e-8) -- trimesh.proximity.signed_distance's convention (source/sdf.py:318-348).
    Optionally also the closest face [Q] int32 (lowest index on ties) and the winding number [Q] fp32."""
    verts = _dev(verts, torch.float32, 'verts')
    faces = _dev(faces, torch.int32, 'faces')
    q = _dev(query, torch.float32, 'query')
    if verts.dim() != 2 or verts.shape[1] != 3 or faces.dim() != 2 or faces.shape[1] != 3 or q.dim() != 2 or q.shape[1] != 3:
        raise P2SError('verts, faces and query must have shape [n, 3]')
    Q = q.shape[0]
    dist = torch.empty((Q,), dtype=torch.float32, device=q.device)
    fid = torch.empty((Q,), dtype=torch.int32, device=q.device) if return_face_ids else None
    wind = torch.empty((Q,), dtype=torch.float32, device=q.device) if return_winding else None
    with torch.cuda.device(q.device):
        check(_lib.load().p2s_mesh_signed_distance_dev(_ptr(verts), verts.shape[0], _ptr(faces), faces.shape[0], _ptr(q), Q,
                                                       _ptr(dist), _ptr(fid) if fid is not None else None,
                                                       _ptr(wind) if wind is not None else None, _stream()))
    out = (dist,) + ((fid,) if return_face_ids else ()) + ((wind,) if return_winding else ())
    return out if len(out) > 1 else dist


def mesh_closest_point(verts, faces, query):
    """Closest point on the mesh of every query point (trimesh.proximity.closest_point, as called by
    source/base/point_cloud.py:195-218) -> (closest [Q,3] fp32, unsigned distance [Q] fp32, face [Q] int32, lowest index
    on ties).  Distance and face equal mesh_signed_distance's |d| and face bit for bit; rules in include/p2s_b200.h."""
    verts = _dev(verts, torch.float32, 'verts')
    faces = _dev(faces, torch.int32, 'faces')
    q = _dev(query, torch.float32, 'query')
    if verts.dim() != 2 or verts.shape[1] != 3 or faces.dim() != 2 or faces.shape[1] != 3 or q.dim() != 2 or q.shape[1] != 3:
        raise P2SError('verts, faces and query must have shape [n, 3]')
    Q = q.shape[0]
    closest = torch.empty((Q, 3), dtype=torch.float32, device=q.device)
    dist = torch.empty((Q,), dtype=torch.float32, device=q.device)
    fid = torch.empty((Q,), dtype=torch.int32, device=q.device)
    with torch.cuda.device(q.device):
        check(_lib.load().p2s_mesh_closest_point_dev(_ptr(verts), verts.shape[0], _ptr(faces), faces.shape[0], _ptr(q), Q,
                                                     _ptr(closest), _ptr(dist), _ptr(fid), _stream()))
    return closest, dist, fid


def mesh_clean(verts, faces):
    """The mesh repair of make_dataset.py:_clean_mesh (rules and output order in include/p2s_b200.h): weld, drop
    non-finite, degenerate and duplicate faces, fill 3- and 4-edge holes, orient every component consistently and
    outward when the winding is inconsistent, drop unreferenced vertices.
    -> (verts [V',3] fp32, faces [F',3] int32, report dict of p2s_clean_report; the four flags as bool)."""
    verts = _dev(verts, torch.float32, 'verts')
    faces = _dev(faces, torch.int32, 'faces')
    if verts.dim() != 2 or verts.shape[1] != 3 or faces.dim() != 2 or faces.shape[1] != 3:
        raise P2SError('verts and faces must have shape [n, 3]')
    V, F = verts.shape[0], faces.shape[0]
    vout = torch.empty((max(V, 1), 3), dtype=torch.float32, device=verts.device)
    fout = torch.empty((max(2 * F, 1), 3), dtype=torch.int32, device=verts.device)
    rep = _lib.CleanReport()
    with torch.cuda.device(verts.device):
        check(_lib.load().p2s_mesh_clean_dev(_ptr(verts), V, _ptr(faces), F, _ptr(vout), V, _ptr(fout), 2 * F,
                                             C.byref(rep), _stream()))
    report = {name: getattr(rep, name) for name, _ in _lib.CleanReport._fields_}
    for k in ('watertight_before', 'winding_consistent_before', 'watertight', 'winding_consistent'):
        report[k] = bool(report[k])
    return vout[:rep.vertices_out], fout[:rep.faces_out], report


def poisson_solve(pts, normals, depth=8, point_weight=4.0, scale=1.1, iters=8):
    """Screened Poisson solve on the dense (2^depth + 1)^3 node grid (system, solver and deviations from PoissonRecon in
    include/p2s_b200.h).  pts, normals [N,3] fp32; zero normals drop their point.
    -> (values [R,R,R] fp32 = iso - chi, positive inside, zero on the surface; report dict of p2s_poisson_report with
    origin as a tuple and stage_ms as a list).  Node (i, j, k) lies at origin + edge * (i, j, k) / 2^depth."""
    pts = _dev(pts, torch.float32, 'pts')
    nrm = _dev(normals, torch.float32, 'normals')
    if pts.dim() != 2 or pts.shape[1] != 3 or nrm.shape != pts.shape:
        raise P2SError('pts and normals must have the same shape [N, 3]')
    cfg = _lib.PoissonConfig(int(depth), float(point_weight), float(scale), int(iters))
    rep = _lib.PoissonReport()
    lib = _lib.load()
    with torch.cuda.device(pts.device):
        check(lib.p2s_poisson_solve_dev(None, None, 0, C.byref(cfg), None, 0, C.byref(rep), _stream()))
        R = rep.grid_res
        values = torch.empty((R, R, R), dtype=torch.float32, device=pts.device)
        check(lib.p2s_poisson_solve_dev(_ptr(pts), _ptr(nrm), pts.shape[0], C.byref(cfg), _ptr(values), values.numel(),
                                        C.byref(rep), _stream()))
    report = {name: getattr(rep, name) for name, _ in _lib.PoissonReport._fields_ if name != 'reserved'}
    report['origin'] = tuple(rep.origin)
    report['stage_ms'] = list(rep.stage_ms)
    return values, report


def _normals_stats(st):
    return dict(degenerate=st.degenerate, components=st.components, flipped=st.flipped, rounds=st.rounds, sweeps=st.sweeps,
                stage_ms=list(st.stage_ms))


def point_normals(pts, k=10, mode='propagate', viewpoint=None, return_neighbours=False, return_stats=False):
    """Oriented unit normals [N,3] fp32 of the cloud pts [N,3] (rules in include/p2s_b200.h, "point normals"): plane fit
    over the k nearest points, then mode 'propagate' (signs along the minimum spanning forest of the kNN graph, each
    component's highest point facing up) or 'viewpoint' (every normal faces `viewpoint`).  A point whose fit is degenerate
    gets (0, 0, 0).  Optionally also the neighbour ids [N,k] int32 and the stats dict of p2s_normals_stats."""
    pts = _dev(pts, torch.float32, 'pts')
    if pts.dim() != 2 or pts.shape[1] != 3:
        raise P2SError('pts must have shape [N, 3]')
    if mode not in ('propagate', 'viewpoint'):
        raise ValueError("mode must be 'propagate' or 'viewpoint', got %r" % (mode,))
    if mode == 'viewpoint' and viewpoint is None:
        raise ValueError("mode 'viewpoint' needs a viewpoint")
    N, k = pts.shape[0], int(k)
    vp = (C.c_double * 3)(*[float(x) for x in viewpoint]) if viewpoint is not None else None
    normals = torch.empty((N, 3), dtype=torch.float32, device=pts.device)
    ids = torch.empty((N, max(k, 0)), dtype=torch.int32, device=pts.device) if return_neighbours else None
    st = _lib.NormalsStats()
    with torch.cuda.device(pts.device):
        check(_lib.load().p2s_point_normals_dev(
            _ptr(pts), N, k, _lib.NORMALS_VIEWPOINT if mode == 'viewpoint' else _lib.NORMALS_PROPAGATE, vp, _ptr(normals),
            _ptr(ids) if ids is not None else None, C.byref(st), _stream()))
    out = (normals,) + ((ids,) if return_neighbours else ()) + ((_normals_stats(st),) if return_stats else ())
    return out if len(out) > 1 else normals


def orient_normals(pts, normals, nbr_ids, return_parents=False, return_stats=False):
    """The 'propagate' orientation of point_normals alone, on caller-supplied normals [N,3] fp32 (unit, or zero for a point
    to leave out) and neighbour ids [N,k] int32.  -> oriented normals, optionally the forest parent of every point [N]
    int32 (a root's own id, -1 without a normal) and the stats dict."""
    pts = _dev(pts, torch.float32, 'pts')
    nrm = _dev(normals, torch.float32, 'normals')
    ids = _dev(nbr_ids, torch.int32, 'nbr_ids')
    if pts.dim() != 2 or pts.shape[1] != 3 or nrm.shape != pts.shape or ids.dim() != 2 or ids.shape[0] != pts.shape[0]:
        raise P2SError('pts and normals must have shape [N, 3] and nbr_ids [N, k]')
    N = pts.shape[0]
    out = torch.empty((N, 3), dtype=torch.float32, device=pts.device)
    parents = torch.empty((N,), dtype=torch.int32, device=pts.device) if return_parents else None
    st = _lib.NormalsStats()
    with torch.cuda.device(pts.device):
        check(_lib.load().p2s_orient_normals_dev(_ptr(pts), _ptr(nrm), _ptr(ids), N, ids.shape[1], _ptr(out),
                                                 _ptr(parents) if parents is not None else None, C.byref(st), _stream()))
    res = (out,) + ((parents,) if return_parents else ()) + ((_normals_stats(st),) if return_stats else ())
    return res if len(res) > 1 else out


SCANNER_DEFAULTS = dict(res_x=176, res_y=144, lens_angle_w=43.6, lens_angle_h=34.6, max_distance=10.0, noise_mu=0.0)


def range_scan(verts, faces, rotations, locations, noise_sigma=0.0, seed=0, first_scan=0, **scanner):
    """Simulated time-of-flight scans of a mesh (BlenSor's TOF scanner of make_dataset.py:sample_blensor, scanner frame
    in include/p2s_b200.h).  rotations [S,3,3] and locations [S,3] place the model point p at R p + loc in front of the
    scanner; scanner settings (`SCANNER_DEFAULTS`) can be overridden by keyword.  The range noise of scan s is keyed by
    (seed, first_scan + s, pixel), so scanning the poses in pieces gives the same points.
    -> (noisy [H,3] fp32, clean [H,3] fp32, face_ids [H] int32, hits_per_scan [S] int32), hits in (scan, row, col)
    order, in model space."""
    unknown = set(scanner) - set(SCANNER_DEFAULTS)
    if unknown:
        raise P2SError('unknown scanner settings: %s' % sorted(unknown))
    s = dict(SCANNER_DEFAULTS, **scanner)
    verts = _dev(verts, torch.float32, 'verts')
    faces = _dev(faces, torch.int32, 'faces')
    if verts.dim() != 2 or verts.shape[1] != 3 or faces.dim() != 2 or faces.shape[1] != 3:
        raise P2SError('verts and faces must have shape [n, 3]')
    dev = verts.device
    rot = torch.as_tensor(rotations, dtype=torch.float64).to(dev).reshape(-1, 3, 3)
    loc = torch.as_tensor(locations, dtype=torch.float64).to(dev).reshape(-1, 3)
    if rot.shape[0] != loc.shape[0]:
        raise P2SError('rotations and locations must describe the same number of scans')
    S = rot.shape[0]
    poses = torch.cat([rot.reshape(S, 9), loc], 1).contiguous()
    cfg = _lib.ScanConfig(int(s['res_x']), int(s['res_y']), float(s['lens_angle_w']), float(s['lens_angle_h']),
                          float(s['max_distance']), float(s['noise_mu']), float(noise_sigma), int(first_scan))
    cap = S * int(s['res_x']) * int(s['res_y'])
    noisy = torch.empty((cap, 3), dtype=torch.float32, device=dev)
    clean = torch.empty((cap, 3), dtype=torch.float32, device=dev)
    fid = torch.empty((cap,), dtype=torch.int32, device=dev)
    hps = torch.empty((S,), dtype=torch.int32, device=dev)
    total = C.c_int64(0)
    with torch.cuda.device(dev):
        check(_lib.load().p2s_range_scan_dev(_ptr(verts), verts.shape[0], _ptr(faces), faces.shape[0], _ptr(poses), S,
                                             C.byref(cfg), int(seed) & (2 ** 64 - 1), _ptr(noisy), _ptr(clean), _ptr(fid),
                                             cap, _ptr(hps), C.byref(total), _stream()))
    H = total.value
    return noisy[:H], clean[:H], fid[:H], hps


def nn_distance(a, b):
    """Nearest neighbour in b of every point of a -> (dist [na] fp32, idx [na] int32)  (cKDTree.query(a, 1))."""
    a = _dev(a, torch.float32, 'a')
    b = _dev(b, torch.float32, 'b')
    dist = torch.empty((a.shape[0],), dtype=torch.float32, device=a.device)
    idx = torch.empty((a.shape[0],), dtype=torch.int32, device=a.device)
    with torch.cuda.device(a.device):
        check(_lib.load().p2s_nn_distance_dev(_ptr(a), a.shape[0], _ptr(b), b.shape[0], _ptr(dist), _ptr(idx), _stream()))
    return dist, idx


def chamfer_hausdorff(a, b):
    """-> dict(chamfer, hausdorff_ab, hausdorff_ba, hausdorff) between two sample sets, the reference's definitions
    (source/base/evaluation.py:252-254, 301-304)."""
    a = _dev(a, torch.float32, 'a')
    b = _dev(b, torch.float32, 'b')
    out = (C.c_double * 4)()
    with torch.cuda.device(a.device):
        check(_lib.load().p2s_chamfer_hausdorff_dev(_ptr(a), a.shape[0], _ptr(b), b.shape[0], out, _stream()))
    return {'chamfer': out[0] + out[1], 'hausdorff_ab': out[2], 'hausdorff_ba': out[3], 'hausdorff': max(out[2], out[3])}
