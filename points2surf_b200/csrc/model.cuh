// Device-resident model: folded fp32 weights (accuracy path) + packed fp16 operand tiles (tensor-core path).
#pragma once
#include "common.cuh"

namespace p2s {

struct Layer {
    const float* W = nullptr;  // [cout][cin] row-major, BN folded
    const float* b = nullptr;  // [cout]
    int cout = 0, cin = 0;
};

struct Stn {  // QSTN (out 4) or STN dim 64 (out 4096): source/points_to_surf_model.py:12-131
    Layer c1, c2, c3, fc1, fc2, fc3;
};

struct Feat {  // PointNetfeat: source/points_to_surf_model.py:134-234
    bool has_qstn = false;
    Stn stn1, stn2;
    Layer conv0a, conv0b, conv1, conv2, conv3;
};

struct TcWeights;  // net_tc.cu

struct Model {
    p2s_model_config cfg{};
    int device = 0;
    float* blob = nullptr;  // device copy of the folded fp32 blob
    size_t blob_floats = 0;
    bool shared_qstn = false;
    Stn point_stn;
    Feat local, global;
    Layer fc1_local, fc1_global, fc2, fc3, fc4;
    // shared-encoder ablation (single_transformer=1, points_to_surf_model.py:253-263,320-323): one PointNetfeat with its
    // own QSTN over cat(patch, sub-sample - q) replaces point_stn / local / global, fc1_enc (1024 -> 1024) replaces
    // fc1_local / fc1_global; those stay empty
    bool single_transformer = false;
    Feat enc;                            // feat_local_global
    Layer fc1_enc;                       // fc1_local_global, bn1_local_global folded

    int precision = P2S_PRECISION_FP32;
    float guard_band = 0.f;
    TcWeights* tc = nullptr;

    cudaStream_t own_stream = nullptr;  // used by the *_host entry points
    DevBuf ws_net;                       // network activations
    DevBuf ws_io;                        // staged host inputs / assembled query batches
    DevBuf ws_misc;
    DevBuf ws_guard;
    DevBuf ws_host;                      // device staging of host-call inputs/outputs
    int64_t* guard_count_dev = nullptr;
    int64_t last_guard_count = 0;
    // deferred guard band (fused pipeline): instead of recomputing inside every batch, forward_tc appends
    // guard_base + i for every flagged query to guard_list; the caller recomputes them all at once
    int32_t* guard_list = nullptr;
    int* guard_list_count = nullptr;
    int64_t guard_list_cap = 0;
    int64_t guard_base = 0;
    float* debug_aux = nullptr;          // optional [B][kAuxStride]: R(9), feat_local_max(1024), feat_global_max(1024);
                                         // shared encoder: R(9), feat_local_global's max(1024), 1024 zeros
};
constexpr int kAuxStride = 2064;
// fg may be null (shared encoder): its 1024 slots are written as zeros
void debug_aux_copy(Model& m, int64_t b0, int64_t Bc, const float* R, const float* fl, const float* fg, cudaStream_t st);

// net_fp32.cu
void forward_fp32(Model& m, const float* patch, const float* sub, const float* query, int64_t B,
                  float* logits, cudaStream_t st);
// net_tc.cu
void tc_build(Model& m);
void tc_destroy(Model& m);
void tc_profile_reset(Model& m, bool on);
void tc_profile_get(Model& m, double* ms, int64_t* launches, double* flops);
void forward_guard(Model& m, const float* patch, const float* sub, const float* query, int64_t B, float* logits, cudaStream_t st);
void forward_tc(Model& m, const float* patch, const float* sub, const float* query, int64_t B,
                float* logits, cudaStream_t st);
// fc_tc.cu
bool fc_tc_supported(int N, int K);
uint8_t* fc_tc_pack(const Layer& L, std::vector<void*>& allocs);
void fc_tc_init();
void launch_fc_tc(const float* A, int lda, const uint8_t* Wimg, const float* bias, float* C, int ldc,
                  int64_t M, int N, int K, bool relu, cudaStream_t st, int pack_img = 0, const float* in_bias = nullptr,
                  bool in_relu = false, const int* a_exp = nullptr, const int* w_exp = nullptr);
uint8_t* fc_tc_pack_raw(const float* W, int N, int K, std::vector<void*>& allocs);
size_t fc_tc_a_image_bytes(int64_t M, int K);
void launch_pack_a(const float* A, int lda, int64_t M, int K, const float* in_bias, bool in_relu, uint8_t* img, cudaStream_t st);
void launch_fc_tc_img(const uint8_t* Aimg, const uint8_t* Wimg, const float* bias, void* C, int ldc, int64_t M, int N, int K,
                      bool relu, cudaStream_t st, int out_mode, int out_kt_total = 0, int out_kt_off = 0);
bool gemm_nt_tc_ok(const float* A, int lda, const float* C, int ldc, int64_t M, int N, int K);
void launch_gemm_nt_tc(const float* A, int lda, const float* W, const float* bias, float* C, int ldc, int64_t M, int N,
                       int K, bool relu, cudaStream_t st);
// split_exp (below) of every row of X[rows][cols] (out[rows])
void launch_split_exp_rows(const float* X, int ld, int64_t rows, int cols, int* out, cudaStream_t st);
// max |x| of every column of X[rows][cols] as float bits (out[cols], zeroed here; cols % 4 == 0, ld % 4 == 0,
// X 16-byte aligned)
void launch_absmax_cols(const float* X, int ld, int64_t rows, int cols, unsigned* out, cudaStream_t st);

// ---- power-of-two operand scaling of the split-precision training GEMMs (fc_tc.cu, gemm_tn_tc.cu)
// hi = fp16(x), lo = fp16(x - hi) keep ~22 bits of x only while both are fp16 normal numbers.  The training operands are
// often far outside that range (the backward pass's dZ shrinks like 1 / batch), so every row (gemm_nt) or column (gemm_tn)
// of an operand is multiplied by 2^s before the split, with s chosen from its largest magnitude `amax` so that the
// scaled maximum lies in [2^15, 65504].  Each output element is a sum over one row / column pair, so the scales factor
// out and the epilogue multiplies by 2^-(s_a + s_b).  An element ~2^-40 below its row's maximum keeps nothing but its
// fp16-subnormal part (half-spacing 2^-25 at a scaled maximum >= 2^15).
__device__ __forceinline__ int split_exp(float amax) {
    if (!(amax > 0.f) || !(amax <= 3.4028235e38f)) return 0;      // zero rows; inf / nan propagate unscaled
    int e;
    const float f = frexpf(amax, &e);                            // amax = f 2^e, f in [0.5, 1)
    return f * 65536.f > 65504.f ? 15 - e : 16 - e;              // s in [-113, 164]
}
// x 2^s without overflow of the factor: two exact power-of-two multiplications (|s| / 2 <= 82)
__device__ __forceinline__ float2 split_factors(int s) {
    const int h = s / 2;
    return make_float2(__int_as_float((127 + h) << 23), __int_as_float((127 + s - h) << 23));
}
// x 2^e rounded once (the epilogue's unscaling): one multiplication while 2^e is a normal float
__device__ __forceinline__ float split_unscale(float x, int e) {
    return (e >= -126 && e <= 127) ? x * __int_as_float((127 + e) << 23) : scalbnf(x, e);
}
// meshdist.cu
void mesh_sample(const float* verts, int64_t V, const int32_t* faces, int64_t F, int64_t n, uint64_t seed,
                 float* samples, int32_t* face_ids, cudaStream_t st);
void nn_distance(const float* a, int64_t na, const float* b, int64_t nb, float* dist, int32_t* idx, cudaStream_t st);
void chamfer_hausdorff(const float* a, int64_t na, const float* b, int64_t nb, double* out4_host, cudaStream_t st);
// meshsdf.cu
void mesh_signed_distance(const float* verts, int64_t V, const int32_t* faces, int64_t F, const float* query, int64_t Q,
                          float* dist, int32_t* closest_face, float* winding, cudaStream_t st);
void mesh_closest_point(const float* verts, int64_t V, const int32_t* faces, int64_t F, const float* query, int64_t Q,
                        float* closest, float* dist, int32_t* closest_face, cudaStream_t st);
// scan.cu
void range_scan(const float* verts, int64_t V, const int32_t* faces, int64_t F, const double* poses, int64_t S,
                const p2s_scan_config& cfg, uint64_t seed, float* pts_noisy, float* pts_clean, int32_t* face_ids,
                int64_t cap, int32_t* hits_per_scan, int64_t* total_host, cudaStream_t st);
// meshclean.cu
void mesh_clean(const float* verts, int64_t V, const int32_t* faces, int64_t F, float* verts_out, int64_t vcap,
                int32_t* faces_out, int64_t fcap, p2s_clean_report* report, cudaStream_t st);
// poisson.cu
void poisson_solve(const float* pts, const float* normals, int64_t N, const p2s_poisson_config& cfg, float* values,
                   int64_t cap, p2s_poisson_report* report, cudaStream_t st);
// normals.cu
void point_normals(const float* pts, int64_t N, int K, int mode, const double* viewpoint, float* normals_out,
                   int32_t* nbr_ids_out, p2s_normals_stats* stats, cudaStream_t st);
void orient_normals(const float* pts, const float* normals_in, const int32_t* nbr_ids, int64_t N, int K, float* normals_out,
                    int32_t* parent_out, p2s_normals_stats* stats, cudaStream_t st);
// gemm_tn_tc.cu
bool gemm_tn_tc_ok(const float* A, int lda, const float* B, int ldb, int64_t M, int N, int K);
void launch_gemm_tn_tc(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int64_t M, int N, int K,
                       cudaStream_t st);
// train_ops.cu
void op_gemm_tn(const float* A, int64_t a_stride_z, int lda, const float* B, int64_t b_stride_z, int ldb, float* C,
                int64_t c_stride_z, int ldc, int M, int N, int K, int batch, bool accumulate, cudaStream_t st);
void op_transpose(const float* in, float* out, int rows, int cols, int batch, cudaStream_t st);
void op_col_stats(const float* x, int64_t M, int C, double* s1, double* s2, cudaStream_t st);
void op_col_sum(const float* x, int64_t M, int C, double* s1, cudaStream_t st);
void op_bn_finalize(const double* s1, const double* s2, int64_t M, int C, float eps, float momentum, float* mean,
                    float* invstd, float* running_mean, float* running_var, cudaStream_t st);
void op_bn_apply(const float* z, int64_t M, int C, const float* mean, const float* invstd, const float* gamma,
                 const float* beta, bool relu, float* y, cudaStream_t st);
void op_bn_backward(const float* dy, const float* z, const float* y_or_null, int64_t M, int C, const float* mean,
                    const float* invstd, const float* gamma, double* s1, double* s2, float* dz, cudaStream_t st);
void op_bn_maxpool_fwd(const float* z, int64_t B, int npts, int C, const float* mean, const float* invstd,
                       const float* gamma, const float* beta, bool relu, float* out, int32_t* arg, cudaStream_t st);
void op_bn_maxpool_bwd(const float* dout, const int32_t* arg, const float* out, const float* z, int64_t B, int npts, int C,
                       const float* mean, const float* invstd, const float* gamma, bool relu, double* s1, double* s2,
                       float* dz, cudaStream_t st);
void op_maxpool_fwd(const float* y, int64_t B, int npts, int C, float* out, int32_t* arg, cudaStream_t st);
void op_maxpool_bwd(const float* dout, const int32_t* arg, int64_t B, int npts, int C, float* dy, cudaStream_t st);
void op_loss(const float* pred, const float* target_mag, const float* radius, const float* target_sign, int64_t B,
             float w_mag, float w_sign, bool fixed_radius, double* loss_out, float* dpred, cudaStream_t st);
void op_loss_distance(const float* pred, const float* target, const float* radius, int64_t B, float w, bool fixed_radius,
                      double* loss_out, float* dpred, cudaStream_t st);
void op_quat_to_rot_bwd(const float* q4, const float* dR, int64_t B, float* dq, cudaStream_t st);
void op_add_row(float* x, const float* v, int64_t B, int C, cudaStream_t st);
void op_sgd(float* p, const float* g, float* buf, int64_t n, float lr, float momentum, bool first, cudaStream_t st);
void op_axpy(float* y, const float* x, float a, int64_t n, cudaStream_t st);
void op_center(const float* in, const float* q, int64_t B, int npts, float* out, cudaStream_t st);
// dispatch (api.cu)
void forward(Model& m, const float* patch, const float* sub, const float* query, int64_t B,
             float* logits, cudaStream_t st);

// small shared kernels (net_fp32.cu), also used by the TC path for the per-query FC tails
void launch_gemm_nt(const float* A, int64_t a_stride_z, int lda, const float* W, int64_t w_stride_z,
                    const float* bias, float* C, int64_t c_stride_z, int ldc, int M, int N, int K,
                    int batch, bool relu, cudaStream_t st);
void launch_gemm_nt_colmax(const float* A, int64_t a_stride_z, int lda, const float* W, float* out,
                           int M, int N, int K, int batch, cudaStream_t st);
void launch_fill(float* p, int64_t n, float v, cudaStream_t st);
void launch_bias_act(float* x, const float* bias, int64_t rows, int cols, bool relu, cudaStream_t st);
void launch_quat_to_rot(const float* q4, float* R, int64_t B, cudaStream_t st);
void launch_add_identity64(float* T, int64_t B, cudaStream_t st);

}  // namespace p2s
