"""ctypes binding of libp2s_b200.so (include/p2s_b200.h).  No fallback: a missing library is an error."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libp2s_b200.so')


class P2SError(RuntimeError):
    pass


class ModelConfig(C.Structure):
    _fields_ = [('use_point_stn', C.c_int32), ('shared_transformer', C.c_int32),
                ('points_per_patch', C.c_int32), ('sub_sample_size', C.c_int32), ('net_size', C.c_int32)]


class ReconConfig(C.Structure):
    _fields_ = [('res', C.c_int32), ('eps', C.c_int32), ('subsample_mode', C.c_int32), ('batch', C.c_int32),
                ('seed', C.c_uint64), ('patch_radius', C.c_float), ('reserved', C.c_int32)]


class ScanConfig(C.Structure):
    _fields_ = [('res_x', C.c_int32), ('res_y', C.c_int32), ('lens_angle_w_deg', C.c_float), ('lens_angle_h_deg', C.c_float),
                ('max_distance', C.c_float), ('noise_mu', C.c_float), ('noise_sigma', C.c_float), ('first_scan', C.c_int32)]


class CleanReport(C.Structure):
    _fields_ = [(n, C.c_int64) for n in (
        'vertices_in', 'faces_in', 'vertices_out', 'faces_out', 'merged_vertices', 'unreferenced_vertices',
        'nonfinite_faces', 'degenerate_faces', 'duplicate_faces', 'boundary_edges', 'nonmanifold_edges', 'holes_filled',
        'faces_added', 'components', 'nonorientable_components', 'faces_reversed')] + \
        [(n, C.c_int32) for n in ('watertight_before', 'winding_consistent_before', 'watertight', 'winding_consistent')] + \
        [('volume', C.c_double)]


class RepairStats(C.Structure):
    _fields_ = [(n, C.c_int64) for n in (
        'vertices_in', 'faces_in', 'vertices_out', 'faces_out', 'faces_removed', 'vertices_split', 'holes_closed',
        'holes_left_open', 'faces_added')]


class PoissonConfig(C.Structure):
    _fields_ = [('depth', C.c_int32), ('point_weight', C.c_float), ('scale', C.c_float), ('iters', C.c_int32)]


class PoissonReport(C.Structure):
    _fields_ = [('origin', C.c_double * 3), ('edge', C.c_double), ('iso', C.c_double), ('residual', C.c_double),
                ('grid_res', C.c_int64), ('points_used', C.c_int64), ('dropped_points', C.c_int64),
                ('occupied_cells', C.c_int64), ('iterations', C.c_int32), ('reserved', C.c_int32),
                ('stage_ms', C.c_float * 4)]


class NormalsStats(C.Structure):
    _fields_ = [('degenerate', C.c_int64), ('components', C.c_int64), ('flipped', C.c_int64), ('rounds', C.c_int32),
                ('sweeps', C.c_int32), ('stage_ms', C.c_float * 3), ('reserved', C.c_int32)]


PRECISION_FP32, PRECISION_TC = 0, 1
NORMALS_PROPAGATE, NORMALS_VIEWPOINT = 0, 1
SUBSAMPLE_WEIGHTED, SUBSAMPLE_UNIFORM = 0, 1

_vp, _i64, _i32, _f32 = C.c_void_p, C.c_int64, C.c_int, C.c_float
# name -> (restype, argtypes); every symbol declared in include/p2s_b200.h
SIGNATURES = {
    'p2s_abi_version': (C.c_int, []),
    'p2s_last_error': (C.c_char_p, []),
    'p2s_launch_count': (C.c_uint64, []),
    'p2s_launch_count_reset': (None, []),
    'p2s_model_blob_floats': (C.c_size_t, [C.POINTER(ModelConfig)]),
    'p2s_model_create': (C.c_int, [C.POINTER(ModelConfig), _vp, C.c_size_t, C.c_int, C.POINTER(_vp)]),
    'p2s_model_blob_floats_ex': (C.c_size_t, [C.POINTER(ModelConfig), C.c_int]),
    'p2s_model_create_ex': (C.c_int, [C.POINTER(ModelConfig), C.c_int, _vp, C.c_size_t, C.c_int, C.POINTER(_vp)]),
    'p2s_model_blob_floats_enc': (C.c_size_t, [C.POINTER(ModelConfig), C.c_int, C.c_int]),
    'p2s_model_create_enc': (C.c_int, [C.POINTER(ModelConfig), C.c_int, C.c_int, _vp, C.c_size_t, C.c_int, C.POINTER(_vp)]),
    'p2s_model_destroy': (None, [_vp]),
    'p2s_model_set_precision': (C.c_int, [_vp, C.c_int, _f32]),
    'p2s_model_last_guard_count': (C.c_int, [_vp, C.POINTER(_i64)]),
    'p2s_model_set_debug_aux': (C.c_int, [_vp, _vp]),
    'p2s_profile_enable': (C.c_int, [_vp, C.c_int]),
    'p2s_profile_get': (C.c_int, [_vp, C.POINTER(C.c_double), C.POINTER(_i64), C.POINTER(C.c_double)]),
    'p2s_forward_dev': (C.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, _vp]),
    'p2s_forward_host': (C.c_int, [_vp, _vp, _vp, _vp, _i64, _vp]),
    'p2s_sdf_from_logits_dev': (C.c_int, [_vp, _vp, _i64, _vp, _vp]),
    'p2s_distance_from_logits_dev': (C.c_int, [_vp, _vp, _i64, _vp, _vp]),
    'p2s_query_grid_dev': (C.c_int, [_vp, _i64, _i32, _i32, _vp, _i64, C.POINTER(_i64), _vp]),
    'p2s_query_points_dev': (C.c_int, [_vp, _i64, _i32, _vp, _vp]),
    'p2s_knn_patch_dev': (C.c_int, [_vp, _i64, _vp, _i64, _i32, _vp, _vp, _vp, _vp]),
    'p2s_ball_patch_dev': (C.c_int, [_vp, _i64, _vp, _i64, _i64, _i32, C.c_double, C.c_uint64, _vp, _vp, _vp, _vp, _vp]),
    'p2s_subsample_dev': (C.c_int, [_vp, _i64, _vp, _i64, _i64, _i32, _i32, C.c_uint64, _vp, _vp]),
    'p2s_gather_points_dev': (C.c_int, [_vp, _vp, _i64, _vp, _vp]),
    'p2s_reconstruct_dev': (C.c_int, [_vp, C.POINTER(ReconConfig), _vp, _i64, _i64, _i64, _vp, _vp, _i64,
                                      C.POINTER(_i64), _vp]),
    'p2s_reconstruct_host': (C.c_int, [_vp, C.POINTER(ReconConfig), _vp, _i64, _vp, _vp, _i64, C.POINTER(_i64)]),
    'p2s_sdf_to_volume_dev': (C.c_int, [_vp, _vp, _i64, _i32, _i32, _f32, _vp, C.POINTER(C.c_int), _vp]),
    'p2s_marching_cubes_dev': (C.c_int, [_vp, _i32, _f32, _vp, _i64, _vp, _i64, C.POINTER(_i64), C.POINTER(_i64), _vp]),
    'p2s_mesh_sample_dev': (C.c_int, [_vp, _i64, _vp, _i64, _i64, C.c_uint64, _vp, _vp, _vp]),
    'p2s_nn_distance_dev': (C.c_int, [_vp, _i64, _vp, _i64, _vp, _vp, _vp]),
    'p2s_op_gemm_nt': (C.c_int, [_vp, _i64, _i32, _vp, _i64, _vp, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    'p2s_op_gemm_tn': (C.c_int, [_vp, _i64, _i32, _vp, _i64, _i32, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    'p2s_op_transpose': (C.c_int, [_vp, _vp, _i32, _i32, _i32, _vp]),
    'p2s_op_col_stats': (C.c_int, [_vp, _i64, _i32, _vp, _vp, _vp]),
    'p2s_op_col_sum': (C.c_int, [_vp, _i64, _i32, _vp, _vp]),
    'p2s_op_bn_finalize': (C.c_int, [_vp, _vp, _i64, _i32, _f32, _f32, _vp, _vp, _vp, _vp, _vp]),
    'p2s_op_bn_stats': (C.c_int, [_vp, _i64, _i32, _f32, _f32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    'p2s_op_bn_apply': (C.c_int, [_vp, _i64, _i32, _vp, _vp, _vp, _vp, _i32, _vp, _vp]),
    'p2s_op_bn_backward': (C.c_int, [_vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    'p2s_op_bn_maxpool_fwd': (C.c_int, [_vp, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp]),
    'p2s_op_bn_maxpool_bwd': (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i32, _i32, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp]),
    'p2s_op_bn_eval_backward': (C.c_int, [_vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    'p2s_op_bn_maxpool_eval_bwd': (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _vp, _vp, _vp, _i32, _vp, _vp,
                                             _vp, _vp, _vp, _vp]),
    'p2s_op_maxpool_fwd': (C.c_int, [_vp, _i64, _i32, _i32, _vp, _vp, _vp]),
    'p2s_op_maxpool_bwd': (C.c_int, [_vp, _vp, _i64, _i32, _i32, _vp, _vp]),
    'p2s_op_loss': (C.c_int, [_vp, _vp, _vp, _vp, _i64, _f32, _f32, _i32, _vp, _vp, _vp]),
    'p2s_op_loss_distance': (C.c_int, [_vp, _vp, _vp, _i64, _f32, _i32, _vp, _vp, _vp]),
    'p2s_op_quat_to_rot': (C.c_int, [_vp, _vp, _i64, _vp]),
    'p2s_op_quat_to_rot_bwd': (C.c_int, [_vp, _vp, _i64, _vp, _vp]),
    'p2s_op_add_row': (C.c_int, [_vp, _vp, _i64, _i32, _vp]),
    'p2s_op_center': (C.c_int, [_vp, _vp, _i64, _i32, _vp, _vp]),
    'p2s_op_axpy': (C.c_int, [_vp, _vp, _f32, _i64, _vp]),
    'p2s_op_sgd': (C.c_int, [_vp, _vp, _vp, _i64, _f32, _f32, _i32, _vp]),
    'p2s_chamfer_hausdorff_dev': (C.c_int, [_vp, _i64, _vp, _i64, C.POINTER(C.c_double), _vp]),
    'p2s_mesh_signed_distance_dev': (C.c_int, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _vp, _vp]),
    'p2s_mesh_closest_point_dev': (C.c_int, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _vp, _vp]),
    'p2s_mesh_inside_grid_dev': (C.c_int, [_vp, _i64, _vp, _i64, _i32, _vp, _vp]),
    'p2s_range_scan_dev': (C.c_int, [_vp, _i64, _vp, _i64, _vp, _i64, C.POINTER(ScanConfig), C.c_uint64, _vp, _vp, _vp,
                                     _i64, _vp, C.POINTER(_i64), _vp]),
    'p2s_mesh_clean_dev': (C.c_int, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, C.POINTER(CleanReport), _vp]),
    'p2s_mesh_repair_dev': (C.c_int, [_vp, _i64, _vp, _i64, _i32, _i32, _vp, _i64, _vp, _i64, C.POINTER(RepairStats),
                                      _vp]),
    'p2s_poisson_solve_dev': (C.c_int, [_vp, _vp, _i64, C.POINTER(PoissonConfig), _vp, _i64, C.POINTER(PoissonReport),
                                        _vp]),
    'p2s_point_normals_dev': (C.c_int, [_vp, _i64, _i32, _i32, C.POINTER(C.c_double), _vp, _vp, C.POINTER(NormalsStats),
                                        _vp]),
    'p2s_orient_normals_dev': (C.c_int, [_vp, _vp, _vp, _i64, _i32, _vp, _vp, C.POINTER(NormalsStats), _vp]),
}

_lib = None


def load():
    """Load the library (once) and declare every prototype.  Raises P2SError if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise P2SError('%s not found: build it with `python -m points2surf_b200.build` '
                       '(there is no CPU fallback)' % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)   # AttributeError here means the .so is stale
        fn.restype = res
        fn.argtypes = args
    if lib.p2s_abi_version() != 2:
        raise P2SError('libp2s_b200.so ABI version mismatch')
    _lib = lib
    return lib


def check(status):
    if status != 0:
        raise P2SError(load().p2s_last_error().decode('utf-8', 'replace'))
