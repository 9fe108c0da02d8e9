/*
 * p2s_b200.h -- C ABI of libp2s_b200.so, the H100 (sm_90a) implementation of the Points2Surf
 * SDF-inference hot path (SURVEY.md section 8).  Plain pointers and sizes only; no torch types.
 *
 * The reference (ErlerPhilipp/points2surf) is pure Python, so "the FFI a maintainer would bind" is
 * a ctypes stub; INTEGRATION.md shows it.  Each entry point names the reference interface it
 * replaces (paths relative to the reference root).
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on failure; p2s_last_error() gives the message
 *     (thread-local, valid until the next call on the same thread).
 *   - `*_dev` functions take DEVICE pointers on the model's device and enqueue on `stream`
 *     (a cudaStream_t passed as void*; NULL = default stream).  They do not synchronise unless
 *     documented ("sync: count read-back").
 *   - `*_host` functions take HOST pointers, perform H2D/D2H copies on the model's internal stream
 *     and return after the result is in the host buffer.
 *   - all float data is IEEE fp32, all index data int32, row-major, densely packed.
 *   - there is no CPU fallback anywhere behind this ABI.
 *
 * Scratch memory
 *   Device scratch of the library is kept per (entry point, device, calling thread), grows only, and is
 *   reused by the next call in stream order.  Calls to one entry point from one thread on two streams are
 *   therefore not independent: order them (or use one thread per stream).  Under CUDA graph capture:
 *   - a call whose scratch would have to grow while its stream is capturing fails with an error before it
 *     enqueues anything; make an eager call of the same size first;
 *   - scratch handed out during a capture is never freed: when a later eager call needs more, it gets new
 *     memory and the captured graph keeps the old one for the rest of the process.
 */
#ifndef P2S_B200_H
#define P2S_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define P2S_ABI_VERSION 2

/* ------------------------------------------------------------------ library / errors ----------- */
int p2s_abi_version(void);
const char* p2s_last_error(void);
/* number of kernels this library has launched since load / since the last reset (bench.py's
 * gpu_launches claim is read from here). */
uint64_t p2s_launch_count(void);
void p2s_launch_count_reset(void);

/* ------------------------------------------------------------------ model ---------------------- */
typedef struct p2s_model p2s_model;

/* Mirrors the constructor arguments of source/points_to_surf_model.py:238-240 as used by
 * source/points_to_surf_eval.py:150-166.  Supported subset (SURVEY.md section 8b): sym_op='max', use_feat_stn=1.
 * The head's output_dim and single_transformer are not part of this struct: the functions without a suffix mean
 * output_dim=2 (imp_surf_magnitude, imp_surf_sign) and single_transformer=0; the _ex variants also take output_dim=1, the
 * regression head of the imp_surf ablation (experiments/train_p2s_regression.sh); the _enc variants also take
 * single_transformer=1, the shared-encoder ablation (experiments/train_p2s_shared_encoder.sh), which requires
 * use_point_stn=1 and shared_transformer=0. */
typedef struct {
    int32_t use_point_stn;      /* train_opt.use_point_stn                                  */
    int32_t shared_transformer; /* train_opt.shared_transformer                             */
    int32_t points_per_patch;   /* train_opt.points_per_patch (300)                         */
    int32_t sub_sample_size;    /* train_opt.sub_sample_size (1000)                         */
    int32_t net_size;           /* train_opt.net_size (1024; must be 1024 for the TC path)  */
} p2s_model_config;

/* Weight blob: BatchNorm (eval mode, eps 1e-5) already folded into the preceding Conv1d/Linear
 * (w' = w*g/sqrt(var+eps), b' = (b-mean)*g/sqrt(var+eps)+beta), every layer stored as
 * W[Cout][Cin] row-major followed by b[Cout], layers concatenated in this order:
 *   STN3(p)  := p.conv1 p.conv2 p.conv3 p.fc1 p.fc2 p.fc3            (QSTN, fc3 -> 4)
 *   STN64(p) := p.conv1 p.conv2 p.conv3 p.fc1 p.fc2 p.fc3            (STN dim 64, fc3 -> 4096)
 *   FEAT(p, qstn) := [STN3(p.stn1) if qstn] STN64(p.stn2) p.conv0a p.conv0b p.conv1 p.conv2 p.conv3
 *   blob := [STN3(point_stn) if use_point_stn && shared_transformer]
 *           FEAT(feat_local, 0)  FEAT(feat_global, use_point_stn && !shared_transformer)
 *           fc1_local fc1_global fc2 fc3 fc4            (fc4: 128 -> output_dim)
 * and with single_transformer=1 (one PointNetfeat over cat(patch, sub-sample - q), points_to_surf_model.py:253-263):
 *   blob := FEAT(feat_local_global, 1)  fc1_local_global  fc2 fc3 fc4
 *           (fc1_local_global: 1024 -> 1024 with bn1_local_global folded; fc2: 1024 -> 256 as above)
 * points2surf_b200/weights.py builds it from a reference state_dict. */
size_t p2s_model_blob_floats(const p2s_model_config* cfg);
/* the same for a head of output_dim outputs (1 or 2); 0 for any other output_dim */
size_t p2s_model_blob_floats_ex(const p2s_model_config* cfg, int output_dim);
/* the same for single_transformer 0 or 1; 0 for an unsupported combination (single_transformer=1 needs use_point_stn=1
 * and shared_transformer=0).  p2s_model_blob_floats_ex(cfg, d) == p2s_model_blob_floats_enc(cfg, d, 0). */
size_t p2s_model_blob_floats_enc(const p2s_model_config* cfg, int output_dim, int single_transformer);

/* Replaces make_regressor (source/points_to_surf_eval.py:150-171): builds the device-resident,
 * kernel-ready weight set on CUDA device `device`. */
int p2s_model_create(const p2s_model_config* cfg, const float* blob_host, size_t blob_floats,
                     int device, p2s_model** out);
/* output_dim 2: p2s_model_create.  output_dim 1: the regression head (outputs imp_surf).  Any other value is an error. */
int p2s_model_create_ex(const p2s_model_config* cfg, int output_dim, const float* blob_host, size_t blob_floats,
                        int device, p2s_model** out);
/* single_transformer 0: p2s_model_create_ex.  1: the shared encoder; the configuration is checked (use_point_stn=1,
 * shared_transformer=0) before any device work, and anything else is an error with a message.  Both engines run it:
 * the tensor-core path as three passes over both segments (QSTN -> R; STN64 with R; final stack with R and the per-query
 * conv1 * (T + I) image), then fc1_local_global, fc2, fc3, fc4. */
int p2s_model_create_enc(const p2s_model_config* cfg, int output_dim, int single_transformer, const float* blob_host,
                         size_t blob_floats, int device, p2s_model** out);
void p2s_model_destroy(p2s_model* m);

/* Arithmetic of the per-point MLP stacks:
 *   P2S_PRECISION_FP32  CUDA-core fp32 FMA everywhere (accuracy path; also the guard-band recompute path)
 *   P2S_PRECISION_TC    wgmma tensor cores,  fp16 operands (11-bit significand, same as the TF32 the
 *                       reference's cuDNN Conv1d uses on Ampere+), fp32 accumulate; queries whose
 *                       |sign logit| (output_dim 2) or |logit| (output_dim 1) < guard_band are recomputed on
 *                       the fp32 path. */
#define P2S_PRECISION_FP32 0
#define P2S_PRECISION_TC 1
int p2s_model_set_precision(p2s_model* m, int precision, float guard_band);
/* number of queries the last forward recomputed on the fp32 path (guard band); sync. */
int p2s_model_last_guard_count(p2s_model* m, int64_t* count);

/* Instrumentation for bench.py's roofline: when enabled, every launch of the dominant kernel (the tensor-core
 * PointNet pass) is bracketed by CUDA events on its stream.  p2s_profile_get synchronises on those events and
 * returns the summed device time, the number of launches and their algorithmic FLOPs (un-padded points,
 * SURVEY.md section 8d), then keeps accumulating until the next p2s_profile_enable call. */
int p2s_profile_enable(p2s_model* m, int on);
int p2s_profile_get(p2s_model* m, double* ms, int64_t* launches, double* flops);

/* Diagnostic tap used by the parity tests: when `aux` (device, [B][P2S_AUX_STRIDE] floats) is non-NULL every
 * following forward also writes, per query, the point rotation R (9), feat_local's max feature (1024) and
 * feat_global's max feature (1024) -- trans / the PointNetfeat outputs of points_to_surf_model.py:326-343.  For a
 * single_transformer model: R (9), feat_local_global's max feature (1024, conv3 bias included), then 1024 zeros. */
#define P2S_AUX_STRIDE 2064
int p2s_model_set_debug_aux(p2s_model* m, float* aux);

/* PointsToSurfModel.forward (source/points_to_surf_model.py:296-352), eval mode.
 *   patch_pts_ps            [B, points_per_patch, 3]   x['patch_pts_ps']
 *   pts_sub_sample_ms       [B, sub_sample_size, 3]    x['pts_sub_sample_ms'] (model space, NOT yet centred;
 *                                                       unlike the reference this op does not modify it)
 *   imp_surf_query_point_ms [B, 3]                     x['imp_surf_query_point_ms']
 *   logits                  [B, output_dim]            (|d| logit, sign logit), or the single signed-distance
 *                                                       logit of an output_dim 1 model */
int p2s_forward_dev(p2s_model* m, const float* patch_pts_ps, const float* pts_sub_sample_ms,
                    const float* imp_surf_query_point_ms, int64_t B, float* logits, void* stream);
int p2s_forward_host(p2s_model* m, const float* patch_pts_ps, const float* pts_sub_sample_ms,
                     const float* imp_surf_query_point_ms, int64_t B, float* logits);

/* post_process + combine (source/sdf_nn.py:11-21, source/points_to_surf_eval.py:184-196,263-271,205-207):
 * sdf = tanh(l0)^2 * radius * (l1 >= 0 ? +1 : -1), NaN -> 1.  patch_radius_ms == NULL is the fixed-radius case
 * (train_opt.patch_radius > 0): the magnitude is not rescaled (points_to_surf_eval.py:188-189,364-368). */
int p2s_sdf_from_logits_dev(const float* logits, const float* patch_radius_ms, int64_t B,
                            float* sdf, void* stream);
/* post_process of the regression head (source/sdf_nn.py:6-8, source/points_to_surf_eval.py:176-183,205-207):
 * logits [B, 1], sdf = tanh(l)^2 * sign(l) * radius with sign(0) = 0, NaN -> 1.  patch_radius_ms == NULL is the
 * fixed-radius case: not rescaled. */
int p2s_distance_from_logits_dev(const float* logits, const float* patch_radius_ms, int64_t B,
                                 float* sdf, void* stream);

/* ------------------------------------------------------------------ query assembly ------------- */
/* sdf.get_voxel_centers_grid_smaller_pc (source/sdf.py:46-70): candidate voxels within an eps^3 box
 * of any occupied voxel, last index plane dropped, in np.nonzero (C) order.
 *   pts [N,3] in [-1,1)^3 (points outside are ignored; the reference would raise / wrap)
 *   lin_idx [cap] receives (ix*res+iy)*res+iz ; *count_host the number found (may exceed cap: then
 *   only the first cap are written).  sync: count read-back. */
int p2s_query_grid_dev(const float* pts, int64_t N, int res, int eps, int32_t* lin_idx, int64_t cap,
                       int64_t* count_host, void* stream);
/* volume_space_to_model_space (source/sdf.py:78-79) of the voxel centres, cast to fp32: [Q,3]. */
int p2s_query_points_dev(const int32_t* lin_idx, int64_t Q, int res, float* query_pts_ms, void* stream);

/* point_cloud.get_patch_kdtree in kNN mode + get_patch_radii + model_space_to_patch_space
 * (source/base/point_cloud.py:174-175, source/base/utils.py:62-69,80-88, source/data_loader.py:340-350).
 * Exact: neighbours are the k smallest float64 distances on the float32 coordinates, ascending
 * (cKDTree semantics); radius and normalisation are float32 like NumPy's.
 *   patch_ids [Q,k] (may be NULL)  patch_pts_ps [Q,k,3]  patch_radius_ms [Q] */
int p2s_knn_patch_dev(const float* pts, int64_t N, const float* query_pts_ms, int64_t Q, int k,
                      int32_t* patch_ids, float* patch_pts_ps, float* patch_radius_ms, void* stream);

/* point_cloud.get_patch_kdtree in ball-query mode (patch_radius > 0, the radius ablations
 * experiments/train_p2s_{small,medium,large}_radius.sh) + the padding rule and fixed-radius normalisation of
 * PointcloudPatchDataset.__getitem__ (source/base/point_cloud.py:176-192, source/data_loader.py:340-350):
 * every point with float64 distance <= patch_radius (cKDTree.query_ball_point on the float32 coordinates); when there are
 * more than k, a uniformly random k-subset without replacement (the reference's rng.choice; here the k smallest
 * Philox clocks keyed by (seed, query index): same law, different stream, independent of batching); when there are fewer,
 * the patch is padded with the query point (patch-space origin, id 0 like the reference's -1 -> 0).
 *   patch_ids [Q,k] (may be NULL; ascending id when nothing is dropped)  patch_pts_ps [Q,k,3] = (p - q) / patch_radius
 *   patch_radius_ms [Q] = patch_radius   in_ball_counts [Q] (may be NULL) = points found before sub-setting / padding */
int p2s_ball_patch_dev(const float* pts, int64_t N, const float* query_pts_ms, int64_t Q, int64_t query_index_base,
                       int k, double patch_radius, uint64_t seed, int32_t* patch_ids, float* patch_pts_ps,
                       float* patch_radius_ms, int32_t* in_ball_counts, void* stream);

/* utils.get_point_cloud_sub_sample (source/base/utils.py:196-227), N >= sub_sample_size.
 *   mode P2S_SUBSAMPLE_UNIFORM : with replacement, like rng.randint             (utils.py:213-216)
 *   mode P2S_SUBSAMPLE_WEIGHTED: without replacement, p ~ clip(1-1.5 d/dmax, .05, 1) (utils.py:200-208,218-219)
 * Counter-based Philox4x32-10 keyed by (seed, query index): results do not depend on batch
 * partitioning or GPU count.  Same distribution as the reference, not the same MT19937 stream.
 *   sub_ids [Q,S] */
#define P2S_SUBSAMPLE_WEIGHTED 0
#define P2S_SUBSAMPLE_UNIFORM 1
int p2s_subsample_dev(const float* pts, int64_t N, const float* query_pts_ms, int64_t Q,
                      int64_t query_index_base, int S, int mode, uint64_t seed, int32_t* sub_ids,
                      void* stream);
/* pts[sub_ids] -> [Q,S,3] (model space, not centred: what __getitem__ returns, data_loader.py:397). */
int p2s_gather_points_dev(const float* pts, const int32_t* ids, int64_t count, float* out, void* stream);

/* ------------------------------------------------------------------ fused reconstruction ------- */
/* The eval loop of source/points_to_surf_eval.py:337-404 in reconstruction mode for ONE shape:
 * candidate grid -> per query (kNN patch, sub-sample, network, post-process) -> SDF band.
 *   pts [N,3] device;  on return *Q_host queries, lin_idx [cap] and sdf [cap] device arrays filled
 *   (what the reference writes to rec/query_pts_ms and rec/dist_ms).  The post-process follows the model's head:
 *   p2s_sdf_from_logits_dev for output_dim 2, p2s_distance_from_logits_dev for output_dim 1.  first_query/num_queries
 *   select a contiguous slab of the ordered query list (multi-GPU tile sharding); pass 0,-1 for all.
 * sync: count read-back. */
typedef struct {
    int32_t res;              /* --query_grid_resolution */
    int32_t eps;              /* --epsilon               */
    int32_t subsample_mode;   /* train_opt.uniform_subsample ? UNIFORM : WEIGHTED */
    int32_t batch;            /* queries per network batch (0 = library default) */
    uint64_t seed;            /* --seed                  */
    float patch_radius;       /* train_opt.patch_radius: <= 0 kNN patches, > 0 ball-query patches of this radius */
    int32_t reserved;         /* must be 0 */
} p2s_recon_config;
int p2s_reconstruct_dev(p2s_model* m, const p2s_recon_config* rc, const float* pts, int64_t N,
                        int64_t first_query, int64_t num_queries,
                        int32_t* lin_idx, float* sdf, int64_t cap, int64_t* Q_host, void* stream);
int p2s_reconstruct_host(p2s_model* m, const p2s_recon_config* rc, const float* pts_host, int64_t N,
                         int32_t* lin_idx_host, float* sdf_host, int64_t cap, int64_t* Q_host);

/* ------------------------------------------------------------------ volume -> mesh ------------- */
/* add_samples_to_volume + propagate_sign + clamp (source/sdf.py:82-111,114-178,200-202) for the
 * reconstruction case (one sample per voxel).  vol [res^3] fp32 (the reference's float64 volume holds
 * only fp32 distances and -1/0/+1, so fp32 is exact).  *iterations_host = propagation iterations run.
 * sync: convergence flag read-back every few iterations. */
int p2s_sdf_to_volume_dev(const int32_t* lin_idx, const float* sdf, int64_t Q, int res, int sigma,
                          float certainty_threshold, float* vol, int* iterations_host, void* stream);

/* marching cubes at level 0 + unit-cube transform + orientation fix (source/sdf.py:211-227).
 *   verts [vcap,3] fp32 in model space, faces [fcap,3] int32; counts returned on the host.
 * sync: count read-back. */
int p2s_marching_cubes_dev(const float* vol, int res, float level, float* verts, int64_t vcap,
                           int32_t* faces, int64_t fcap, int64_t* nverts_host, int64_t* nfaces_host,
                           void* stream);

/* ------------------------------------------------------------------ mesh acceptance metric ----- */
/* Area-weighted surface sampling (the sampler behind _chamfer_distance_single_file / _hausdorff_distance_single_file,
 * source/base/evaluation.py:229-238; trimesh.sample.sample_surface without the "even" rejection step -- trimesh is
 * absent, parity unpinned).  verts [V,3] fp32, faces [F,3] int32 -> samples [n,3] fp32, face_ids [n] int32 or NULL.
 * Philox stream keyed by (seed, sample index).  async. */
int p2s_mesh_sample_dev(const float* verts, int64_t V, const int32_t* faces, int64_t F, int64_t n,
                        uint64_t seed, float* samples, int32_t* face_ids, void* stream);

/* Exact nearest neighbour of every a[i] in b (cKDTree.query(a, 1), source/base/evaluation.py:246-250): dist [na]
 * fp32 Euclidean distance, idx [na] int32 (lowest index on ties); either output may be NULL.  async. */
int p2s_nn_distance_dev(const float* a, int64_t na, const float* b, int64_t nb, float* dist, int32_t* idx,
                        void* stream);

/* Both directed sums and maxima of the nearest-neighbour distances between two sample sets:
 * out4_host = { sum a->b, sum b->a, max a->b, max b->a }.  Chamfer (evaluation.py:252-254) = out[0] + out[1];
 * directed Hausdorff (evaluation.py:301-303) = out[2], out[3].  sync: result read-back. */
int p2s_chamfer_hausdorff_dev(const float* a, int64_t na, const float* b, int64_t nb, double* out4_host,
                              void* stream);

/* ------------------------------------------------------------------ training targets ----------- */
/* trimesh.proximity.signed_distance as called by sdf.get_signed_distance (source/sdf.py:318-348) for the query points
 * of make_dataset.py:_get_and_save_query_pts (make_dataset.py:447-478).  Exhaustive and exact: the distance to the
 * nearest triangle is the float64 minimum (an fp32 pass selects the faces to recompute within a stated error bound;
 * ties -> lowest face index); zero-area faces count as segments / points.  Any finite coordinates: the fp32 pass runs
 * in units of a power of two taken from max(|query|_inf, max |vertex coordinate|), so it neither under- nor overflows,
 * and the float64 recompute covers fp32's whole range.  So scaling the mesh and the queries by 2^k scales the distance
 * and the closest point by 2^k bit for bit and keeps the face and the winding number, wherever the scaled inputs and
 * results are normal fp32 numbers (the sign follows the absolute |d| <= 1e-8 rule below).  Sign from the generalised winding number w
 * (float64 solid angles of all faces): dist = +|d| if w > 0.5 or |d| <= 1e-8 (points on the surface are positive, like
 * trimesh), else -|d|; inside is positive.  w equals trimesh's ray-parity inside test on closed, consistently oriented
 * meshes; on meshes with holes or flipped faces the two can disagree.  A query with a non-finite coordinate gives NaN.
 *   verts [V,3] fp32, faces [F,3] int32 (every index in [0, V), else an error; F > 0), query [Q,3] fp32
 *   dist [Q] fp32; closest_face [Q] int32 or NULL; winding [Q] fp32 (w) or NULL.
 * Bitwise deterministic, independent of how the queries are split across calls.  sync: index check read-back. */
int p2s_mesh_signed_distance_dev(const float* verts, int64_t V, const int32_t* faces, int64_t F, const float* query,
                                 int64_t Q, float* dist, int32_t* closest_face, float* winding, void* stream);

/* The unsigned point-to-mesh query: trimesh.proximity.closest_point as called by point_cloud.get_closest_distance_batched
 * (source/base/point_cloud.py:195-218; source/figure/distance_vis.py, and the ground-truth normals of eval_dataset.py).
 * The distance and the face come from the same pass as p2s_mesh_signed_distance_dev without the solid angles: the same
 * fp32 prefilter and float64 recompute band, the same face slabs and the same tie rule (lowest face index), so dist and
 * closest_face equal that function's |dist| and closest_face bit for bit.  The closest point is computed in float64 on
 * the winning face, by the rule that gave its distance: the orthogonal projection onto the face's plane when the query
 * projects inside the face, else the closest point of the nearest edge (the first of ab, bc, ca on equal distances;
 * zero-area faces are their edges), then rounded to fp32 once.  A query with a non-finite coordinate gives NaN for the
 * distance and the point, and face -1.
 *   verts [V,3] fp32, faces [F,3] int32 (every index in [0, V), else an error; F > 0), query [Q,3] fp32
 *   closest_pts [Q,3] fp32 or NULL; dist [Q] fp32; closest_face [Q] int32 or NULL.
 * Bitwise deterministic, independent of how the queries are split across calls.  sync: index check read-back. */
int p2s_mesh_closest_point_dev(const float* verts, int64_t V, const int32_t* faces, int64_t F, const float* query,
                               int64_t Q, float* closest_pts, float* dist, int32_t* closest_face, void* stream);

/* ------------------------------------------------------------------ solid voxelisation --------- */
/* Inside flag of every voxel centre of a res^3 grid over [-1, 1]^3, 2 <= res <= 1024 (the exact-sign volume of
 * make_dataset's 06_mc_gt_exact_sign).  Voxel (ix, iy, iz) has the centre (c(ix), c(iy), c(iz)),
 * c(i) = float(((double)i + 0.5) / res * 2 - 1), the points of p2s_query_points_dev.  It is inside iff the ray from its
 * centre towards +z crosses an odd number of faces.  The rule is watertight: on a closed mesh (every edge shared by
 * exactly two faces) every column is crossed an even number of times, whatever the coordinates:
 *   - x and y are taken in fixed point, X = llrint(double(x) * 2^26), for the vertices and the column centres alike; z
 *     stays fp32.  Every vertex must have |x| < 16, |y| < 16 and a finite z (else an error), so the edge functions below
 *     are exact in int64.
 *   - a column crosses a face iff the face's three projected edge functions E(u -> v) = (u - p) x (v - p), each evaluated
 *     on the edge's canonical vertex order (lower vertex index first) and negated where the face runs the other way,
 *     have the same sign.  So the two faces that share an edge see exactly negated values.
 *   - ties (a column centre on a projected edge or vertex, E == 0) take the sign at the centre moved by (eps, eps^2): the
 *     sign of -(v.y - u.y), or of v.x - u.x when v.y == u.y (a top-left rule).  Every column thus sees one generic
 *     point of the projected mesh.
 *   - faces whose projection has zero area (parallel to z, or with a repeated vertex) cross no column.
 *   - the crossing height is z = (E_bc z_a + E_ca z_b + E_ab z_c) / (E_bc + E_ca + E_ab) in float64 (each E rounded to
 *     float64, sums left to right, no contraction); the crossing flips every voxel of the column with c(iz) < z.
 * The flags are an inside/outside sign only for closed meshes; on other meshes they are the rule's parity.  On a closed
 * mesh the parity is the winding number mod 2: where closed components overlap (winding number 2) a voxel is outside,
 * while p2s_mesh_signed_distance_dev's w > 0.5 calls it inside.
 *   verts [V,3] fp32, faces [F,3] int32 (every index in [0, V), else an error; F = 0 gives all 0)
 *   inside [res^3] uint8: 1 inside, 0 outside, at (ix * res + iy) * res + iz (the order of p2s_query_grid_dev's indices).
 * Bitwise deterministic.  sync: input check read-back. */
int p2s_mesh_inside_grid_dev(const float* verts, int64_t V, const int32_t* faces, int64_t F, int res, uint8_t* inside,
                             void* stream);

/* ------------------------------------------------------------------ input point clouds --------- */
/* Simulated time-of-flight range scans: the BlenSor scans of make_dataset.py:sample_blensor (make_dataset.py:242-380,
 * scanner settings blensor_script_template.py:80-96) merged in model space like _pcd_files_to_pts
 * (make_dataset.py:147-239).  Scanner frame: the scanner sits at the origin and looks along +y; the image's wide axis
 * (res_x columns, lens_angle_w) is z, its rows run along x.  Scan s places the model point p at R_s p + loc_s.  Pixel
 * (row, col), row 0 at +x, col 0 at -z, casts the ray through the pixel centre (v, 1, u) / |(v, 1, u)| with
 *   u = (2 (col + 1/2) / res_x - 1) tan(lens_angle_w / 2),  v = (1 - 2 (row + 1/2) / res_y) tan(lens_angle_h / 2).
 * The ray hits the nearest surface at a distance t in (0, max_distance] (watertight ray-triangle test, no back-face
 * culling, zero-area faces never hit, ties -> lowest face index).  The noisy range is t' = t + noise_mu + noise_sigma z
 * with z standard normal from Philox4x32-10 keyed by (seed, first_scan + s, pixel).  Points are returned in model space,
 * R_s^T (x - loc_s), compacted in (scan, row, col) order.
 *   verts [V,3] fp32, faces [F,3] int32 (every index in [0, V), else an error; F > 0)
 *   poses [S][12] float64 on the device: R_s row-major, then loc_s
 *   pts_noisy [cap,3] fp32; pts_clean [cap,3] fp32 or NULL; face_ids [cap] int32 or NULL; hits_per_scan [S] int32 or NULL
 *   total_host: the number of hits H.  Only the first min(H, cap) hits are written; H <= S * res_x * res_y.
 * Bitwise deterministic and independent of how the scans are split across calls (with first_scan counting on).
 * sync: count read-back. */
typedef struct {
    int32_t res_x, res_y;                        /* 176, 144 */
    float lens_angle_w_deg, lens_angle_h_deg;    /* 43.6, 34.6: full field of view */
    float max_distance;                          /* 10 */
    float noise_mu, noise_sigma;                 /* Gaussian range noise */
    int32_t first_scan;                          /* index of poses[0] in the shape's scan sequence (noise stream) */
} p2s_scan_config;

int p2s_range_scan_dev(const float* verts, int64_t V, const int32_t* faces, int64_t F, const double* poses, int64_t S,
                       const p2s_scan_config* cfg, uint64_t seed, float* pts_noisy, float* pts_clean, int32_t* face_ids,
                       int64_t cap, int32_t* hits_per_scan, int64_t* total_host, void* stream);

/* ------------------------------------------------------------------ mesh cleaning -------------- */
/* The repair of make_dataset.py:_clean_mesh (make_dataset.py:383-413: trimesh's process, remove_degenerate_faces,
 * remove_duplicate_faces, fill_holes, fix_inversion / fix_normals / fix_winding) without the file I/O and the accept /
 * reject decision.  In this order:
 *   1. non-finite: faces that reference a vertex with a non-finite coordinate are dropped.
 *   2. weld (tol.merge = 1e-8): two finite vertices merge iff llround(double(x) * 1e8) is equal for all three
 *      coordinates; the merged vertex keeps the coordinates of its lowest input index.  A finite |coordinate| >= 9e10
 *      is an error (the key overflows int64).
 *   3. degenerate: a face with two equal (welded) indices, or whose float64 altitude over its longest edge
 *      (2 area / longest edge) is <= 1e-8, is dropped.
 *   4. duplicate: faces with the same vertex set, in either orientation; the first is kept.
 *   5. edges: the faces on every undirected edge are counted.  Watertight: every edge has exactly two faces.  The winding
 *      is consistent iff the two faces of every two-face edge traverse it in opposite directions.
 *   6. holes: a boundary loop (a closed chain of one-face edges through vertices of boundary degree 2) of 3 edges gets
 *      one face, of 4 edges two faces split along the diagonal through the loop's lowest vertex.  Fill faces run
 *      opposite to the loop's edge from its lowest vertex v to v's lower boundary neighbour.  Longer loops and loops
 *      through a vertex of boundary degree != 2 stay open.  Step 5 is redone.
 *   7. orientation, only when the winding is inconsistent after 6 (a closed, consistent, all-inverted mesh is not
 *      flipped): components are connected over two-face edges.  A component is orientable iff some choice of face
 *      flips makes all its two-face edges consistent; its faces are then reversed ((a,b,c) -> (c,b,a)) relative to its
 *      lowest face, and the whole component again when its float64 signed volume sum det(v0,v1,v2) / 6 is < 0.
 *      Non-orientable components, and faces without a two-face edge, are left as they came.
 *   8. vertices no output face uses are dropped.
 * Output order: vertices ascending by their lowest merged input index; faces in input order without the dropped ones,
 * then the fill faces ordered by their loop's lowest vertex.  A clean mesh comes back bit-identical.
 * Deviations from trimesh: first-occurrence vertex order (trimesh: hash order; some versions also reorder faces when
 * removing duplicates); the quad diagonal is fixed by the lowest vertex (trimesh: networkx cycle_basis order); loops
 * through non-manifold vertices are not filled; vertices referenced only by dropped faces are dropped here (trimesh
 * keeps them until the mesh is reloaded); the orientation of non-orientable components and of open components with
 * signed volume exactly 0 is not pinned.
 *   verts [V,3] fp32, faces [F,3] int32 (every index in [0, V), else an error)
 *   verts_out [vcap,3] fp32, faces_out [fcap,3] int32: vcap >= V and fcap >= 2 F always suffice; a smaller capacity
 *   that turns out too small is an error, not a truncation.
 * Bitwise deterministic (the signed volumes are reduced in a fixed order, no float atomics).  sync: report read-back. */
typedef struct {
    int64_t vertices_in, faces_in, vertices_out, faces_out;
    int64_t merged_vertices;               /* input vertices welded onto a lower index */
    int64_t unreferenced_vertices;         /* welded vertices (non-finite ones included) no output face uses */
    int64_t nonfinite_faces, degenerate_faces, duplicate_faces;
    int64_t boundary_edges, nonmanifold_edges;    /* after hole filling */
    int64_t holes_filled, faces_added;
    int64_t components, nonorientable_components, faces_reversed;   /* of step 7; 0 when it did not run */
    int32_t watertight_before, winding_consistent_before;            /* after hole filling, before step 7 */
    int32_t watertight, winding_consistent;                          /* of the output */
    double volume;                                                   /* float64 signed volume of the output */
} p2s_clean_report;

int p2s_mesh_clean_dev(const float* verts, int64_t V, const int32_t* faces, int64_t F, float* verts_out, int64_t vcap,
                       int32_t* faces_out, int64_t fcap, p2s_clean_report* report_host, void* stream);

/* ------------------------------------------------------------------ mesh repair (hole filling) -- */
/* The first four filters of the reference's hole_filling_mesh_simp.mlx (dataset_for_deepsdf.py), which it runs through
 * meshlabserver before computing DeepSDF's far-sample distances.  Meshlab's exact choices are not pinned; these are this
 * project's rules, in this order:
 *   1. non-manifold edges, removing faces: every undirected edge with c > 2 faces drops its c - 2 smallest faces by
 *      float64 squared area |(b - a) x (c - a)|^2 (ties: the higher face index is dropped first).  All edges are judged
 *      on the input faces at once; a face dropped by any edge is removed.  Afterwards no edge has more than two faces.
 *   2. non-manifold edges, splitting vertices: a no-op after 1 (no edge has more than two faces), so nothing is done.
 *   3. non-manifold vertices, splitting (VertDispRatio 0): the faces around a vertex are joined into fans over the edges
 *      of that vertex that have two faces.  A vertex with k > 1 fans gets k - 1 copies at the same position: the fan
 *      holding the lowest face index keeps the vertex; the copies are appended after the input vertices in order of
 *      their fan's lowest face index (ties, one face opening fans at two vertices: its corner order 0, 1, 2).
 *   4. close holes (MaxHoleSize, SelfIntersection): after 3 every boundary vertex has exactly two boundary edges, so the
 *      boundary edges form simple loops.  A loop of L <= max_hole_size edges is filled by ear cutting:
 *      - the walk starts at the loop's lowest vertex v towards the neighbour x whose boundary edge runs x -> v in its
 *        face (the lower neighbour when both or neither do), and goes on around the loop; every fill face (prev, tip,
 *        next) follows the walk, so it runs against the boundary edges it closes;
 *      - the plane: the float64 Newell normal n of the walk; u = n x e_k / |n x e_k| for the axis k of smallest |n_k|
 *        (the lowest k on ties), w = (n / |n|) x u; vertex i goes to (p_i . u, p_i . w).  A zero n leaves no valid ear;
 *      - an ear is convex when the 2D cross product of (tip - prev, next - tip) is > 0; convex ears are tried by the
 *        smallest tip angle first (the largest cos of the 2D angle), ties by the lowest tip vertex id, and the first
 *        valid one is cut, until the loop is a triangle, which is cut the same way;
 *      - while more than three loop vertices remain, an ear is not valid when its new edge (next, prev) is already an
 *        edge of the mesh (it would get a third face);
 *      - an ear is not valid when another remaining loop vertex lies inside or on its 2D triangle (it would overlap the
 *        faces beyond the loop's boundary: the planar form of the intersection test), or, with prevent_self_intersection,
 *        when an edge of the ear crosses the interior of a face incident to a loop vertex or of a triangle already
 *        added to this loop, or an edge of such a face crosses the ear's interior.  A crossing is strict: the segment's
 *        ends lie strictly on both sides of the triangle's plane and it passes strictly inside all three edges, each side
 *        a float64 signed volume ((b-a) x (c-a)) . (d-a), taken as 0 when two of its four points coincide.  Coplanar
 *        contact and touching at shared vertices or edges is not a crossing;
 *      - when no convex ear is valid, the faces cut so far are dropped and the loop stays open (counted in
 *        holes_left_open, like the loops longer than max_hole_size).  Triangles added to other loops are not tested.
 *   Decimation to 100 000 faces (the .mlx's last filter) is not done: the repaired mesh is only a signed-distance target.
 * Output order: vertices = the input vertices, then the copies of 3; faces = the faces kept by 1 in input order (with the
 * indices of 3), then the fill faces, loop by loop in order of each loop's lowest vertex id, in cutting order.
 *   verts [V,3] fp32, faces [F,3] int32: every index in [0, V) and three distinct indices per face, else an error.
 *   max_hole_size in [0, 128] (30 in the .mlx); prevent_self_intersection 0/1 (1 in the .mlx).
 *   verts_out [vcap,3] fp32, faces_out [fcap,3] int32: vcap >= V + 3 F and fcap >= 4 F always suffice; a capacity that
 *   turns out too small is an error, not a truncation.
 * Bitwise deterministic (integer atomics only, float64 geometry in a fixed order).  sync: several read-backs. */
typedef struct {
    int64_t vertices_in, faces_in, vertices_out, faces_out;
    int64_t faces_removed;       /* by rule 1 */
    int64_t vertices_split;      /* copies appended by rule 3 */
    int64_t holes_closed;        /* loops filled by rule 4 */
    int64_t holes_left_open;     /* loops longer than max_hole_size, and loops without a valid ear */
    int64_t faces_added;
} p2s_repair_stats;

int p2s_mesh_repair_dev(const float* verts, int64_t V, const int32_t* faces, int64_t F, int32_t max_hole_size,
                        int32_t prevent_self_intersection, float* verts_out, int64_t vcap, int32_t* faces_out, int64_t fcap,
                        p2s_repair_stats* stats_host, void* stream);

/* ------------------------------------------------------------------ screened Poisson baseline --- */
/* Screened Poisson surface reconstruction from oriented points, the SPSR baseline of eval_dataset.py:142-158 (which
 * the reference runs through meshlabserver with poisson.mlx).  The discrete system:
 *   domain  the cube of edge E = scale * (largest extent of the bounding box of all N points), centred on that box,
 *           mapped to [0,1]^3; nodes k in [0, 2^depth]^3, spacing h = 2^-depth
 *   basis   trilinear hat functions B_k, all nodes free (natural boundary); chi is trilinear in every cell
 *   1D      M = int phi_i phi_j (2h/3 on the diagonal, h/3 at both ends, h/6 off it), K = int phi_i' phi_j' (2/h, 1/h at
 *           the ends, -1/h), D(i, j) = int phi_i phi_j' (+-1/2 off the diagonal; -1/2 at node 0, +1/2 at node 2^depth)
 *   L       K(x)M(x)M + M(x)K(x)M + M(x)M(x)K (the 27-point Q1 stencil)
 *   points  normals scaled to unit length; a zero normal drops the point (counted).  Area weight a_p = (4h)^2 / n_c(p),
 *           n_c = the number of kept points in p's cell at depth - 2
 *   V       V_k = sum_p a_p n_p B_k(p) / h^3;  b_j = int V . grad B_j
 *   S       alpha sum_p a_p B(p) B(p)^T, alpha = point_weight * 2^depth
 *   solve   (L + S) chi = b by conjugate gradients preconditioned with one symmetric multigrid V-cycle over depths
 *           depth..2 (exact Galerkin levels, `iters` damped-Jacobi sweeps before and after each coarse correction, 128
 *           sweeps on depth 2); stop at ||b - A chi|| / ||b|| <= 1e-5, after 100 iterations, or when the residual has
 *           not reached a new minimum for 10 iterations.  point_weight 0 makes S = 0 and the system singular (L 1 = 0,
 *           1^T b = 0): chi is then the solution of mean zero over the nodes
 *   iso     sum a_p chi(p) / sum a_p
 * values [(2^depth+1)^3] fp32 = iso - chi at node (i, j, k), index (i R + j) R + k with R = 2^depth + 1: positive inside,
 * zero on the surface, so p2s_marching_cubes_dev(values, R, 0) extracts it; node (i, j, k) is at world position
 * origin + edge (i, j, k) / 2^depth.  values == NULL with vcap == 0 only validates the config and sets grid_res.
 * Deviations from PoissonRecon: a dense grid instead of an adaptive octree (samplesPerNode, fullDepth unused), degree-1
 * instead of degree-2 B-splines, no confidence, and the scaling of alpha is unpinned (PoissonRecon's is not
 * available to compare against).  Errors (not faults): N = 0, non-finite points or normals, zero extent, every normal
 * zero, depth outside [2, 9], scale < 1, point_weight < 0, iters outside [1, 64].
 * Bitwise deterministic (fixed-order sums, no float atomics).  sync: several read-backs (sizes, CG residuals). */
typedef struct {
    int32_t depth;          /* 8 in poisson.mlx */
    float point_weight;     /* 4 */
    float scale;            /* 1.1 */
    int32_t iters;          /* 8: smoothing sweeps per level and half V-cycle */
} p2s_poisson_config;

typedef struct {
    double origin[3];       /* world position of node (0, 0, 0) */
    double edge;            /* world edge of the cube */
    double iso;             /* iso-value of chi (values = iso - chi) */
    double residual;        /* ||b - A chi|| / ||b|| at exit; 0 when b = 0 */
    int64_t grid_res;       /* 2^depth + 1 nodes per axis */
    int64_t points_used, dropped_points;
    int64_t occupied_cells; /* finest cells holding at least one kept point */
    int32_t iterations, reserved;
    float stage_ms[4];      /* CUDA-event times of setup (sort, cells, levels), right-hand side, solve, iso + output */
} p2s_poisson_report;

int p2s_poisson_solve_dev(const float* pts, const float* normals, int64_t N, const p2s_poisson_config* cfg, float* values,
                          int64_t vcap, p2s_poisson_report* report_host, void* stream);

/* ------------------------------------------------------------------ point normals --- */
/* Oriented unit normals of an unstructured point cloud: what meshlab's "Compute normals for point sets" does before the
 * Screened Poisson filter of the reference's normals_poisson.mlx, for clouds that come without a mesh.  Parity with
 * meshlab / vcglib is NOT pinned: neither is part of this project, and meshlab's propagation starts at an arbitrary point
 * without an outward seed.  The rules below are the specification (oracle/normals_oracle.py restates them on the CPU).
 *
 * a. Neighbours.  nbr_ids[i] = the K nearest points of the cloud to point i, point i itself included, by the float64
 *    squared distance (dx*dx + dy*dy) + dz*dz on the fp32 coordinates with every operation rounded (p2s_knn_patch_dev's
 *    semantics), ascending, lowest id first on ties.  3 <= K <= 64, N > K.
 * b. Plane fit.  Float64 centroid and scatter matrix sum (p - centroid)(p - centroid)^T of the K neighbours, eigenvalues
 *    l0 <= l1 <= l2 by cyclic Jacobi.  The fit is degenerate when !(l2 > 0) or l1 - l0 <= 1e-9 * l2 (all neighbours equal,
 *    collinear, or isotropic): the point gets the normal (0, 0, 0) and takes no part in c.  Otherwise the normal is the
 *    unit eigenvector of l0, rounded to fp32, with the sign that makes its component of largest magnitude positive (the
 *    lowest axis on ties, compared on the fp32 values).
 * c. Orientation.
 *    P2S_NORMALS_VIEWPOINT: n is negated when n . (viewpoint - p) < 0 (float64, x then y then z, every operation rounded).
 *    P2S_NORMALS_PROPAGATE (Hoppe et al. 1992): the graph has an edge i-j when j is among nbr_ids[i] or i among
 *    nbr_ids[j], i != j, and both normals are non-zero.  Its cost is c = max(0, 1 - |n_i . n_j|) with
 *    n_i . n_j = (x_i*x_j + y_i*y_j) + z_i*z_j in float64 from the fp32 normals, every operation rounded.  Edges are
 *    totally ordered by (bits of c, min(i, j), max(i, j)), so the minimum spanning forest is unique.  Per component the
 *    root is the point of largest z (lowest id on ties; -0 = +0) and keeps its normal when its z is > 0, is negated when
 *    z < 0, and at z = 0 the same by y, then x.  Every other point is negated when (final normal of its forest parent) .
 *    (its own input normal) < 0, and kept at exactly 0.  Components are oriented independently.  The result is a function
 *    of the input alone (not of the schedule): bitwise identical across runs and streams.
 * Both entry points synchronise `stream` (counts are read back).  Errors (non-zero return, p2s_last_error, nothing written
 * to the outputs): NULL pointers, K outside [3, 64], N <= K, N * K >= 0x7f7f7f7f, an unknown mode, viewpoint mode without
 * a viewpoint, non-finite coordinates, normals or viewpoint, neighbour ids outside [0, N) (the last three checked on the
 * device before any other kernel runs). */
#define P2S_NORMALS_PROPAGATE 0
#define P2S_NORMALS_VIEWPOINT 1

typedef struct {
    int64_t degenerate;     /* points with a zero normal */
    int64_t components;     /* trees of the spanning forest (propagate) */
    int64_t flipped;        /* points whose normal was negated by c */
    int32_t rounds;         /* Boruvka rounds that joined components */
    int32_t sweeps;         /* level sweeps launched over the forest (a multiple of 64) */
    float stage_ms[3];      /* CUDA-event times of a (cell index + neighbours), b, c */
    int32_t reserved;
} p2s_normals_stats;

/* a + b + c.  pts [N,3]; viewpoint: 3 doubles on the host, NULL in propagate mode; normals_out [N,3];
 * nbr_ids_out [N,K] int32 or NULL; stats_host or NULL. */
int p2s_point_normals_dev(const float* pts, int64_t N, int K, int mode, const double* viewpoint, float* normals_out,
                          int32_t* nbr_ids_out, p2s_normals_stats* stats_host, void* stream);
/* c (propagate) alone on caller-supplied normals (unit or zero; any pre-sign) and neighbour ids [N,K], e.g. unoriented
 * normals of another estimator.  parent_out [N] int32 or NULL: the forest parent of every point, a root's own id, -1 for a
 * point without a normal. */
int p2s_orient_normals_dev(const float* pts, const float* normals_in, const int32_t* nbr_ids, int64_t N, int K,
                           float* normals_out, int32_t* parent_out, p2s_normals_stats* stats_host, void* stream);

/* ------------------------------------------------------------------ training-step primitives --- */
/* Row a14 (SURVEY.md section 8a): loss + backward + SGD of source/points_to_surf_train.py:441-461,537-563 with the
 * train-mode BatchNorm of source/points_to_surf_model.py.  Activations are row-major [rows, C] fp32.  The host side
 * (points2surf_b200/train.py) sequences these like the reference's autograd graph.  All async on `stream`. */
/* Accuracy of both GEMMs, per output element, for operands anywhere in fp32's normal range:
 *     |C - C_exact| <= gamma_K sum_k |a_k| |b_k| + 2^-40 K max_k |a_k| max_k |b_k|,   gamma_K = K 2^-24 / (1 - K 2^-24)
 * (K = reduction length, the accumulate form counts the running value as one more term).  Large shapes run on the tensor
 * cores in split precision after scaling every reduction vector by a power of two; the rest, and every shape under
 * P2S_TRAIN_GEMM_FP32=1, on fp32 FMA.
 * C[z][m][n] = act(sum_k A[z][m][k] W[z][n][k] + bias[n])   (torch conv1d(k=1) / linear / bmm forward) */
int p2s_op_gemm_nt(const float* A, int64_t a_stride_z, int lda, const float* W, int64_t w_stride_z,
                   const float* bias, float* C, int64_t c_stride_z, int ldc, int M, int N, int K, int batch,
                   int relu, void* stream);
/* C[z][n][k] (+)= sum_m A[z][m][n] B[z][m][k]               (weight gradient dW = dZ^T X) */
int p2s_op_gemm_tn(const float* A, int64_t a_stride_z, int lda, const float* B, int64_t b_stride_z, int ldb,
                   float* C, int64_t c_stride_z, int ldc, int M, int N, int K, int batch, int accumulate,
                   void* stream);
/* out[z][c][r] = in[z][r][c] */
int p2s_op_transpose(const float* in, float* out, int rows, int cols, int batch, void* stream);
/* s1 = sum x, s2 = sum x^2 over the M rows (f64 [C] each) */
int p2s_op_col_stats(const float* x, int64_t M, int C, double* s1, double* s2, void* stream);
int p2s_op_col_sum(const float* x, int64_t M, int C, double* s1, void* stream);
/* mean, invstd = 1/sqrt(biased var + eps) from the sums of p2s_op_col_stats; running stats updated like torch (unbiased
 * var) when non-NULL.  var = s2/M - (s1/M)^2 cancels once |mean| >> std: BatchNorm uses p2s_op_bn_stats. */
int p2s_op_bn_finalize(const double* s1, const double* s2, int64_t M, int C, float eps, float momentum,
                       float* mean, float* invstd, float* running_mean, float* running_var, void* stream);
/* BatchNorm1d(train) statistics of x [M, C]: mean, invstd and the running stats as p2s_op_bn_finalize, from f64 sums
 * of x - x[0] and (x - x[0])^2 (left in s1, s2, f64 [C] each), so invstd is accurate to ~2^-24 for any |mean| / std */
int p2s_op_bn_stats(const float* x, int64_t M, int C, float eps, float momentum, double* s1, double* s2,
                    float* mean, float* invstd, float* running_mean, float* running_var, void* stream);
/* y = act(gamma (z - mean) invstd + beta) */
int p2s_op_bn_apply(const float* z, int64_t M, int C, const float* mean, const float* invstd,
                    const float* gamma, const float* beta, int relu, float* y, void* stream);
/* dz from dy through act + BatchNorm(train); y = forward output for the ReLU mask or NULL; outputs s1 = dbeta,
 * s2 = dgamma (f64 [C]) */
int p2s_op_bn_backward(const float* dy, const float* z, const float* y, int64_t M, int C, const float* mean,
                       const float* invstd, const float* gamma, double* s1, double* s2, float* dz, void* stream);
/* BatchNorm(train)(+ReLU) fused with the max over the npts points of each query (the conv3 layers): forward from the
 * pre-BN z [B*npts, C] with mean / invstd from p2s_op_col_stats + p2s_op_bn_finalize; backward builds dz directly
 * from dout [B,C] (s1 = dbeta, s2 = dgamma, f64 [C]) */
int p2s_op_bn_maxpool_fwd(const float* z, int64_t B, int npts, int C, const float* mean, const float* invstd,
                          const float* gamma, const float* beta, int relu, float* out, int32_t* arg, void* stream);
int p2s_op_bn_maxpool_bwd(const float* dout, const int32_t* arg, const float* out, const float* z, int64_t B,
                          int npts, int C, const float* mean, const float* invstd, const float* gamma, int relu,
                          double* s1, double* s2, float* dz, void* stream);
/* Eval-mode backward (model.eval(): BatchNorm with mean = running_mean, invstd = 1/sqrt(running_var + eps), constants of
 * the backward, so every row is independent and nothing needs a second pass).
 * BatchNorm(eval)(+ReLU), one pass over the M rows: g = dy masked by y > 0 (y = forward output, NULL without ReLU),
 * dz = gamma invstd g [M, C]; dbeta = sum g, dgamma = sum g (z - mean) invstd, dbias = sum dz (the gradient of the bias of
 * the layer in front), f64 [C] each, overwritten.
 * Per element, with the f64 sums' rounding negligible: |dz - exact| <= 2u |dz|, |dgamma - exact| <= 2u sum |g xhat| +
 * u |dgamma|, |dbias - exact| <= 2u sum |dz| + u |dbias| (u = 2^-24; the last u is the caller's conversion to fp32). */
int p2s_op_bn_eval_backward(const float* dy, const float* z, const float* y, int64_t M, int C, const float* mean,
                            const float* invstd, const float* gamma, double* dbeta, double* dgamma, double* dbias,
                            float* dz, void* stream);
/* BatchNorm(eval)(+ReLU) + max over the npts points, fused with the conv in front of it (z = x W^T + bias, x [B*npts, K],
 * W [C, K], C <= 4096): the backward from dout [B, C] given the forward's arg [B, C] (p2s_op_bn_maxpool_fwd with the
 * running statistics; arg taken on the normalised values, first maximum) and out [B, C] (read for the ReLU mask only,
 * may be NULL without ReLU).  Only the arg row of each (query, channel) carries a gradient, dz[b,c] = gamma invstd
 * dout[b,c] (0 where out <= 0 under ReLU); the dense [B*npts, C] gradient is never formed:
 *     dW[c,:] += sum_b dz[b,c] x[b*npts + arg[b,c], :]                  (gather over B rows, fp32 FMA + fp32 atomics;
 *                                                                       every row is read, so 0 * Inf gives NaN like the dense path)
 *     dx[b*npts + i, :] = sum_{c : arg[b,c] = i} dz[b,c] W[c,:]        (scatter, ascending c, every row written; NULL: skipped)
 *     dbias = sum_b dz, dgamma = sum_b g xhat(arg row), dbeta = sum_b g  (f64 [C], overwritten)
 * dW and dx are within gamma_n sum |dz| |x| (resp. |W|) of the exact sums of the rounded dz (n = terms + 2).  All row
 * offsets are 64-bit, so B * npts * K may exceed 2^31. */
int p2s_op_bn_maxpool_eval_bwd(const float* dout, const int32_t* arg, const float* out, const float* z, const float* x,
                               const float* W, int64_t B, int npts, int C, int K, const float* mean, const float* invstd,
                               const float* gamma, int relu, float* dW, double* dbias, double* dgamma, double* dbeta,
                               float* dx, void* stream);
/* MaxPool1d over the npts points of each query: y [B, npts, C] -> out [B, C], arg [B, C] (first maximum) */
int p2s_op_maxpool_fwd(const float* y, int64_t B, int npts, int C, float* out, int32_t* arg, void* stream);
int p2s_op_maxpool_bwd(const float* dout, const int32_t* arg, int64_t B, int npts, int C, float* dy, void* stream);
/* compute_loss for outputs (imp_surf_magnitude, imp_surf_sign), source/points_to_surf_train.py:550-561 and
 * source/sdf_nn.py:30-40: loss_out (device f64 [2]) = {w_mag * mse(tanh|p0|, tanh|t/r|), w_sign * bce(p1, s)};
 * dpred [B,2] = gradient of their sum (NULL: forward only).  fixed_radius != 0 skips the division by r. */
int p2s_op_loss(const float* pred, const float* target_mag, const float* radius, const float* target_sign,
                int64_t B, float w_mag, float w_sign, int fixed_radius, double* loss_out, float* dpred,
                void* stream);
/* compute_loss for the regression output imp_surf, source/points_to_surf_train.py:541-548 and sdf_nn.calc_loss_distance:
 * loss_out (device f64 [1]) = w * mse(tanh p, tanh(t/r)) with the signed tanh; dpred [B,1] = its gradient (NULL: forward
 * only).  fixed_radius != 0 skips the division by r (radius may then be NULL). */
int p2s_op_loss_distance(const float* pred, const float* target, const float* radius, int64_t B, float w,
                         int fixed_radius, double* loss_out, float* dpred, void* stream);
/* utils.batch_quat_to_rotmat (source/base/utils.py:13-46) forward and backward.  q4 [B,4] is the raw fc3 output of the
 * QSTN; the identity quaternion (1,0,0,0) is added inside (source/points_to_surf_model.py:124-126).  R, dR [B,9]. */
int p2s_op_quat_to_rot(const float* q4, float* R, int64_t B, void* stream);
int p2s_op_quat_to_rot_bwd(const float* q4, const float* dR, int64_t B, float* dq, void* stream);
/* x[b][:] += v[:]  (identity quaternion / identity matrix offsets) */
int p2s_op_add_row(float* x, const float* v, int64_t B, int C, void* stream);
/* out[b][p][:] = in[b][p][:] - q[b][:]  (source/points_to_surf_model.py:303) */
int p2s_op_center(const float* in, const float* q, int64_t B, int npts, float* out, void* stream);
/* y += a x */
int p2s_op_axpy(float* y, const float* x, float a, int64_t n, void* stream);
/* torch.optim.SGD(momentum) update (source/points_to_surf_train.py:406,461) */
int p2s_op_sgd(float* param, const float* grad, float* momentum_buf, int64_t n, float lr, float momentum,
               int first_step, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* P2S_B200_H */
