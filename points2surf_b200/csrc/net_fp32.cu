// fp32 CUDA-core implementation of PointsToSurfModel.forward (source/points_to_surf_model.py:296-352).
// This is the accuracy path: plain FMA in fp32, layer by layer, in the reference's operation order.
// It backs P2S_PRECISION_FP32 and the guard-band recompute of the tensor-core path.
#include "model.cuh"

namespace p2s {

// ------------------------------------------------------------------------------------------------
// Batched NT GEMM:  C[z][m][n] = act( sum_k A[z][m][k] * W[z][n][k] + bias[n] )
// 64x64x16 tiles, 256 threads, 4x4 outputs per thread.
// COLMAX: instead of storing C, reduce max over the valid rows m and atomically max into out[z][n].
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
    if (v >= 0.f) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
    else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

template <bool VEC, bool COLMAX>
__global__ void __launch_bounds__(256)
gemm_nt_kernel(const float* __restrict__ A, int64_t a_stride_z, int lda,
               const float* __restrict__ W, int64_t w_stride_z, const float* __restrict__ bias,
               float* __restrict__ C, int64_t c_stride_z, int ldc, int M, int N, int K, int relu) {
    constexpr int BM = 64, BN = 64, BK = 16;
    __shared__ float As[BK][BM + 4];
    __shared__ float Ws[BK][BN + 4];
    __shared__ float red[16][BN];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int z = blockIdx.z;
    const float* Az = A + (int64_t)z * a_stride_z;
    const float* Wz = W + (int64_t)z * w_stride_z;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < K; k0 += BK) {
        if (VEC) {
            const int r = tid >> 2, kq = (tid & 3) * 4;
            float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vw = va;
            if (m0 + r < M && k0 + kq < K) va = *reinterpret_cast<const float4*>(Az + (int64_t)(m0 + r) * lda + k0 + kq);
            if (n0 + r < N && k0 + kq < K) vw = *reinterpret_cast<const float4*>(Wz + (int64_t)(n0 + r) * K + k0 + kq);
            As[kq + 0][r] = va.x; As[kq + 1][r] = va.y; As[kq + 2][r] = va.z; As[kq + 3][r] = va.w;
            Ws[kq + 0][r] = vw.x; Ws[kq + 1][r] = vw.y; Ws[kq + 2][r] = vw.z; Ws[kq + 3][r] = vw.w;
        } else {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int e = tid + i * 256, r = e >> 4, k = e & 15;
                As[k][r] = (m0 + r < M && k0 + k < K) ? Az[(int64_t)(m0 + r) * lda + k0 + k] : 0.f;
                Ws[k][r] = (n0 + r < N && k0 + k < K) ? Wz[(int64_t)(n0 + r) * K + k0 + k] : 0.f;
            }
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float a[4], w[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = As[k][ty * 4 + i];
#pragma unroll
            for (int j = 0; j < 4; ++j) w[j] = Ws[k][tx * 4 + j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
        }
        __syncthreads();
    }

    if (!COLMAX) {
        float* Cz = C + (int64_t)z * c_stride_z;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int m = m0 + ty * 4 + i;
            if (m >= M) continue;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int n = n0 + tx * 4 + j;
                if (n >= N) continue;
                float v = acc[i][j] + (bias ? bias[n] : 0.f);
                if (relu) v = fmaxf(v, 0.f);
                Cz[(int64_t)m * ldc + n] = v;
            }
        }
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float v = -INFINITY;
#pragma unroll
            for (int i = 0; i < 4; ++i)
                if (m0 + ty * 4 + i < M) v = fmaxf(v, acc[i][j]);
            red[ty][tx * 4 + j] = v;
        }
        __syncthreads();
        if (tid < BN) {
            float v = red[0][tid];
#pragma unroll
            for (int r = 1; r < 16; ++r) v = fmaxf(v, red[r][tid]);
            if (n0 + tid < N) atomic_max_float(C + (int64_t)z * c_stride_z + n0 + tid, v);
        }
    }
}


// ------------------------------------------------------------------------------------------------
// Larger-tile variant for the shapes that carry the FLOPs (K % 16 == 0, 16-byte aligned rows):
// 128 x BN x 16 tiles, 256 threads, 8 x (BN/16) outputs per thread, double-buffered shared memory,
// global loads of the next tile overlapped with the FMAs of the current one.
// ------------------------------------------------------------------------------------------------
template <int BN, bool COLMAX>
__global__ void __launch_bounds__(256)
gemm128_nt_kernel(const float* __restrict__ A, int64_t a_stride_z, int lda,
                  const float* __restrict__ W, int64_t w_stride_z, const float* __restrict__ bias,
                  float* __restrict__ C, int64_t c_stride_z, int ldc, int M, int N, int K, int relu) {
    constexpr int BM = 128, BK = 16, NJ = BN / 64;          // NJ column groups of 4 per thread (64 apart)
    constexpr int LDA_S = BM + 4, LDB_S = BN + 4;
    __shared__ __align__(16) float As[2][BK][LDA_S];
    __shared__ __align__(16) float Bs[2][BK][LDB_S];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int z = blockIdx.z;
    const float* Az = A + (int64_t)z * a_stride_z;
    const float* Wz = W + (int64_t)z * w_stride_z;
    // global -> register staging: A tile 128 x 16 = 512 float4 (2 per thread), B tile BN x 16 = BN*4 float4
    const int lr = tid >> 2, lk = (tid & 3) * 4;             // row 0..63, k offset
    float4 ra[2], rb[BN / 64];
    auto load_tile = [&](int k0) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int r = m0 + lr + i * 64;
            ra[i] = (r < M) ? *reinterpret_cast<const float4*>(Az + (int64_t)r * lda + k0 + lk) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int i = 0; i < BN / 64; ++i) {
            const int r = n0 + lr + i * 64;
            rb[i] = (r < N) ? *reinterpret_cast<const float4*>(Wz + (int64_t)r * K + k0 + lk) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    auto store_tile = [&](int b) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int r = lr + i * 64;
            As[b][lk + 0][r] = ra[i].x; As[b][lk + 1][r] = ra[i].y; As[b][lk + 2][r] = ra[i].z; As[b][lk + 3][r] = ra[i].w;
        }
#pragma unroll
        for (int i = 0; i < BN / 64; ++i) {
            const int r = lr + i * 64;
            Bs[b][lk + 0][r] = rb[i].x; Bs[b][lk + 1][r] = rb[i].y; Bs[b][lk + 2][r] = rb[i].z; Bs[b][lk + 3][r] = rb[i].w;
        }
    };
    float acc[8][NJ * 4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < NJ * 4; ++j) acc[i][j] = 0.f;

    load_tile(0);
    store_tile(0);
    __syncthreads();
    const int nk = K / BK;
    for (int kt = 0; kt < nk; ++kt) {
        const int b = kt & 1;
        if (kt + 1 < nk) load_tile((kt + 1) * BK);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float a[8], w[NJ * 4];
            const float4 a0 = *reinterpret_cast<const float4*>(&As[b][k][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[b][k][64 + ty * 4]);
            a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
                const float4 w4 = *reinterpret_cast<const float4*>(&Bs[b][k][j * 64 + tx * 4]);
                w[j * 4 + 0] = w4.x; w[j * 4 + 1] = w4.y; w[j * 4 + 2] = w4.z; w[j * 4 + 3] = w4.w;
            }
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < NJ * 4; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
        }
        if (kt + 1 < nk) store_tile(b ^ 1);
        __syncthreads();
    }

    if (!COLMAX) {
        float* Cz = C + (int64_t)z * c_stride_z;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int m = m0 + (i >> 2) * 64 + ty * 4 + (i & 3);
            if (m >= M) continue;
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
                const int n = n0 + j * 64 + tx * 4;
                float v[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    v[e] = acc[i][j * 4 + e] + ((bias && n + e < N) ? bias[n + e] : 0.f);
                    if (relu) v[e] = fmaxf(v[e], 0.f);
                }
                if (n + 3 < N && (ldc & 3) == 0) *reinterpret_cast<float4*>(Cz + (int64_t)m * ldc + n) = make_float4(v[0], v[1], v[2], v[3]);
                else
                    for (int e = 0; e < 4; ++e)
                        if (n + e < N) Cz[(int64_t)m * ldc + n + e] = v[e];
            }
        }
    } else {
        float* red = &As[0][0][0];          // [16][BN] floats <= 2*16*132
        __syncthreads();
#pragma unroll
        for (int j = 0; j < NJ * 4; ++j) {
            float v = -INFINITY;
#pragma unroll
            for (int i = 0; i < 8; ++i)
                if (m0 + (i >> 2) * 64 + ty * 4 + (i & 3) < M) v = fmaxf(v, acc[i][j]);
            red[ty * BN + (j >> 2) * 64 + tx * 4 + (j & 3)] = v;
        }
        __syncthreads();
        if (tid < BN) {
            float v = red[tid];
#pragma unroll
            for (int r = 1; r < 16; ++r) v = fmaxf(v, red[r * BN + tid]);
            if (n0 + tid < N) atomic_max_float(C + (int64_t)z * c_stride_z + n0 + tid, v);
        }
    }
}

static bool gemm128_ok(const float* A, int64_t a_stride_z, int lda, const float* W, int64_t w_stride_z, int N, int K) {
    return (K % 16 == 0) && (lda % 4 == 0) && (a_stride_z % 4 == 0) && (w_stride_z % 4 == 0) &&
           ((uintptr_t)A % 16 == 0) && ((uintptr_t)W % 16 == 0) && (N >= 64);
}

void launch_gemm_nt(const float* A, int64_t a_stride_z, int lda, const float* W, int64_t w_stride_z,
                    const float* bias, float* C, int64_t c_stride_z, int ldc, int M, int N, int K,
                    int batch, bool relu, cudaStream_t st) {
    if (M <= 0 || batch <= 0) return;
    if (gemm128_ok(A, a_stride_z, lda, W, w_stride_z, N, K) && M >= 64) {
        if (N >= 128) {
            dim3 g((unsigned)cdiv(M, 128), (unsigned)cdiv(N, 128), (unsigned)batch);
            P2S_LAUNCH((gemm128_nt_kernel<128, false>), g, 256, 0, st, A, a_stride_z, lda, W, w_stride_z, bias, C, c_stride_z, ldc, M, N, K, relu ? 1 : 0);
        } else {
            dim3 g((unsigned)cdiv(M, 128), (unsigned)cdiv(N, 64), (unsigned)batch);
            P2S_LAUNCH((gemm128_nt_kernel<64, false>), g, 256, 0, st, A, a_stride_z, lda, W, w_stride_z, bias, C, c_stride_z, ldc, M, N, K, relu ? 1 : 0);
        }
        return;
    }
    dim3 grid((unsigned)cdiv(M, 64), (unsigned)cdiv(N, 64), (unsigned)batch);
    const bool vec = (K % 4 == 0) && (lda % 4 == 0) && (a_stride_z % 4 == 0) && (w_stride_z % 4 == 0) &&
                     ((uintptr_t)A % 16 == 0) && ((uintptr_t)W % 16 == 0);
    if (vec) P2S_LAUNCH((gemm_nt_kernel<true, false>), grid, 256, 0, st, A, a_stride_z, lda, W, w_stride_z, bias, C, c_stride_z, ldc, M, N, K, relu ? 1 : 0);
    else P2S_LAUNCH((gemm_nt_kernel<false, false>), grid, 256, 0, st, A, a_stride_z, lda, W, w_stride_z, bias, C, c_stride_z, ldc, M, N, K, relu ? 1 : 0);
}

// out[z][n] = max_m sum_k A[z][m][k] W[n][k]   (out must be pre-filled with -inf)
void launch_gemm_nt_colmax(const float* A, int64_t a_stride_z, int lda, const float* W, float* out,
                           int M, int N, int K, int batch, cudaStream_t st) {
    if (M <= 0 || batch <= 0) return;
    if (gemm128_ok(A, a_stride_z, lda, W, 0, N, K) && N >= 128) {
        dim3 g((unsigned)cdiv(M, 128), (unsigned)cdiv(N, 128), (unsigned)batch);
        P2S_LAUNCH((gemm128_nt_kernel<128, true>), g, 256, 0, st, A, a_stride_z, lda, W, (int64_t)0, nullptr, out, (int64_t)N, N, M, N, K, 0);
        return;
    }
    dim3 grid((unsigned)cdiv(M, 64), (unsigned)cdiv(N, 64), (unsigned)batch);
    const bool vec = (K % 4 == 0) && (lda % 4 == 0) && (a_stride_z % 4 == 0) &&
                     ((uintptr_t)A % 16 == 0) && ((uintptr_t)W % 16 == 0);
    if (vec) P2S_LAUNCH((gemm_nt_kernel<true, true>), grid, 256, 0, st, A, a_stride_z, lda, W, (int64_t)0, nullptr, out, (int64_t)N, N, M, N, K, 0);
    else P2S_LAUNCH((gemm_nt_kernel<false, true>), grid, 256, 0, st, A, a_stride_z, lda, W, (int64_t)0, nullptr, out, (int64_t)N, N, M, N, K, 0);
}

// ------------------------------------------------------------------------------------------------
// small element-wise kernels
// ------------------------------------------------------------------------------------------------
__global__ void fill_kernel(float* p, int64_t n, float v) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}
__global__ void debug_aux_kernel(float* aux, int64_t b0, int64_t Bc, const float* R, const float* fl, const float* fg) {
    int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= Bc * kAuxStride) return;
    int64_t b = e / kAuxStride;
    int j = (int)(e % kAuxStride);
    float v = 0.f;
    if (j < 9) v = R ? R[b * 9 + j] : (j % 4 == 0 ? 1.f : 0.f);
    else if (j < 9 + 1024) v = fl[b * 1024 + (j - 9)];
    else if (j < 9 + 2048) v = fg ? fg[b * 1024 + (j - 9 - 1024)] : 0.f;
    aux[(b0 + b) * kAuxStride + j] = v;
}
void debug_aux_copy(Model& m, int64_t b0, int64_t Bc, const float* R, const float* fl, const float* fg, cudaStream_t st) {
    if (!m.debug_aux || Bc <= 0) return;
    P2S_LAUNCH(debug_aux_kernel, (unsigned)cdiv(Bc * kAuxStride, 256), 256, 0, st, m.debug_aux, b0, Bc, R, fl, fg);
}

void launch_fill(float* p, int64_t n, float v, cudaStream_t st) {
    if (n <= 0) return;
    P2S_LAUNCH(fill_kernel, (unsigned)cdiv(n, 256), 256, 0, st, p, n, v);
}

__global__ void bias_act_kernel(float* x, const float* __restrict__ bias, int64_t total, int cols, int relu) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    float v = x[i] + bias[i % cols];
    if (relu) v = fmaxf(v, 0.f);
    x[i] = v;
}
void launch_bias_act(float* x, const float* bias, int64_t rows, int cols, bool relu, cudaStream_t st) {
    int64_t total = rows * cols;
    if (total <= 0) return;
    P2S_LAUNCH(bias_act_kernel, (unsigned)cdiv(total, 256), 256, 0, st, x, bias, total, cols, relu ? 1 : 0);
}

// source/base/utils.py:13-46 with q = fc3(x) + [1,0,0,0] (points_to_surf_model.py:124-126)
__global__ void quat_to_rot_kernel(const float* __restrict__ q4, float* __restrict__ R, int64_t B) {
    int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    float q[4] = {q4[b * 4 + 0] + 1.f, q4[b * 4 + 1], q4[b * 4 + 2], q4[b * 4 + 3]};
    float s = 2.f / (q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    float h[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) h[i][j] = q[i] * q[j];
    float* o = R + b * 9;
    o[0] = 1.f - (h[2][2] + h[3][3]) * s;
    o[1] = (h[1][2] - h[3][0]) * s;
    o[2] = (h[1][3] + h[2][0]) * s;
    o[3] = (h[1][2] + h[3][0]) * s;
    o[4] = 1.f - (h[1][1] + h[3][3]) * s;
    o[5] = (h[2][3] - h[1][0]) * s;
    o[6] = (h[1][3] - h[2][0]) * s;
    o[7] = (h[2][3] + h[1][0]) * s;
    o[8] = 1.f - (h[1][1] + h[2][2]) * s;
}
void launch_quat_to_rot(const float* q4, float* R, int64_t B, cudaStream_t st) {
    P2S_LAUNCH(quat_to_rot_kernel, (unsigned)cdiv(B, 128), 128, 0, st, q4, R, B);
}

__global__ void add_identity64_kernel(float* T, int64_t B) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < B * 64) T[(i / 64) * 4096 + (i % 64) * 65] += 1.f;
}
void launch_add_identity64(float* T, int64_t B, cudaStream_t st) {
    P2S_LAUNCH(add_identity64_kernel, (unsigned)cdiv(B * 64, 256), 256, 0, st, T, B);
}

// out[b][i][:] = R[b] * in[b][i][:]  (torch.bmm(trans, x), model.py:328-329); R may be null (copy)
// `center` (optional [B,3]) is subtracted first (model.py:303).
__global__ void transform_points_kernel(const float* __restrict__ in, const float* __restrict__ center,
                                        const float* __restrict__ R, float* __restrict__ out,
                                        int64_t B, int n_in, int n_out, int out_off) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * n_in) return;
    int64_t b = i / n_in;
    int p = (int)(i % n_in);
    float x = in[i * 3 + 0], y = in[i * 3 + 1], z = in[i * 3 + 2];
    if (center) { x -= center[b * 3 + 0]; y -= center[b * 3 + 1]; z -= center[b * 3 + 2]; }
    float ox = x, oy = y, oz = z;
    if (R) {
        const float* r = R + b * 9;
        ox = r[0] * x + r[1] * y + r[2] * z;
        oy = r[3] * x + r[4] * y + r[5] * z;
        oz = r[6] * x + r[7] * y + r[8] * z;
    }
    float* o = out + ((int64_t)b * n_out + out_off + p) * 3;
    o[0] = ox; o[1] = oy; o[2] = oz;
}
static void transform_points(const float* in, const float* center, const float* R, float* out,
                             int64_t B, int n_in, int n_out, int out_off, cudaStream_t st) {
    P2S_LAUNCH(transform_points_kernel, (unsigned)cdiv(B * n_in, 256), 256, 0, st, in, center, R, out, B, n_in, n_out, out_off);
}

// ------------------------------------------------------------------------------------------------
// forward orchestration
// ------------------------------------------------------------------------------------------------
namespace {

struct Ws {  // activations for one chunk of Bc queries
    float *xall, *patch_r, *sub_r, *bufH, *bufA, *bufB, *g, *f1, *f2, *q4, *R, *T, *fb_local, *fb_global, *cat, *h3, *h4;
};

// point-wise layer on a flat [rows, cin] matrix
void conv(const Layer& L, const float* in, float* out, int64_t rows, bool relu, cudaStream_t st) {
    launch_gemm_nt(in, 0, L.cin, L.W, 0, L.b, out, 0, L.cout, (int)rows, L.cout, L.cin, 1, relu, st);
}

// conv3 (128 -> 1024) fused with the max over the n points of each query; bias (+ReLU) after the max
void conv_max(const Layer& L, const float* in, float* out, int64_t Bc, int n, bool relu, cudaStream_t st) {
    launch_fill(out, Bc * L.cout, -INFINITY, st);
    launch_gemm_nt_colmax(in, (int64_t)n * L.cin, L.cin, L.W, out, n, L.cout, L.cin, (int)Bc, st);
    launch_bias_act(out, L.b, Bc, L.cout, relu, st);
}

void fc(const Layer& L, const float* in, float* out, int64_t Bc, bool relu, cudaStream_t st) {
    launch_gemm_nt(in, 0, L.cin, L.W, 0, L.b, out, 0, L.cout, (int)Bc, L.cout, L.cin, 1, relu, st);
}

// QSTN / STN: x [Bc, n, cin] -> out [Bc, 4 | 4096]
void stn(const Stn& s, const float* x, int64_t Bc, int n, Ws& w, float* out, cudaStream_t st) {
    conv(s.c1, x, w.bufA, Bc * n, true, st);
    conv(s.c2, w.bufA, w.bufB, Bc * n, true, st);
    conv_max(s.c3, w.bufB, w.g, Bc, n, true, st);
    fc(s.fc1, w.g, w.f1, Bc, true, st);
    fc(s.fc2, w.f1, w.f2, Bc, true, st);
    fc(s.fc3, w.f2, out, Bc, false, st);
}

// PointNetfeat.forward: pts [Bc, n, 3] (already transformed) -> fmax [Bc,1024]
void feat(const Feat& f, const float* pts, int64_t Bc, int n, Ws& w, float* fmax, cudaStream_t st) {
    conv(f.conv0a, pts, w.bufA, Bc * n, true, st);
    conv(f.conv0b, w.bufA, w.bufH, Bc * n, true, st);
    stn(f.stn2, w.bufH, Bc, n, w, w.T, st);
    launch_add_identity64(w.T, Bc, st);
    // x = bmm(trans2, x): per query y = T x  -> batched NT gemm with W = T[b]
    launch_gemm_nt(w.bufH, (int64_t)n * 64, 64, w.T, 4096, nullptr, w.bufA, (int64_t)n * 64, 64, n, 64, 64, (int)Bc, false, st);
    conv(f.conv1, w.bufA, w.bufB, Bc * n, true, st);
    conv(f.conv2, w.bufB, w.bufA, Bc * n, true, st);
    conv_max(f.conv3, w.bufA, fmax, Bc, n, false, st);
}

}  // namespace

void forward_fp32(Model& m, const float* patch, const float* sub, const float* query, int64_t B,
                  float* logits, cudaStream_t st) {
    const int P = m.cfg.points_per_patch, S = m.cfg.sub_sample_size, PS = P + S;
    const int64_t Bc_max = 1024;
    // carve the workspace
    size_t per_q = (size_t)PS * 3 * 3 + (size_t)PS * (64 + 128 + 128) + 1024 * 3 + 512 * 3 + 256 + 4 + 9 + 4096 + 1024 + 256 + 128 + 64;
    float* base = m.ws_net.as<float>(per_q * Bc_max);
    Ws w;
    float* p = base;
    auto take = [&](size_t n) { float* r = p; p += (n * Bc_max + 3) / 4 * 4; return r; };
    w.xall = take((size_t)PS * 3); w.patch_r = take((size_t)P * 3); w.sub_r = take((size_t)S * 3);
    w.bufH = take((size_t)PS * 64); w.bufA = take((size_t)PS * 128); w.bufB = take((size_t)PS * 128);
    w.g = take(1024); w.f1 = take(512); w.f2 = take(256); w.q4 = take(4); w.R = take(9); w.T = take(4096);
    w.fb_local = take(1024); w.fb_global = take(1024); w.cat = take(1024); w.h3 = take(256); w.h4 = take(128);

    for (int64_t b0 = 0; b0 < B; b0 += Bc_max) {
        const int64_t Bc = (B - b0 < Bc_max) ? (B - b0) : Bc_max;
        const float* pa = patch + b0 * P * 3;
        const float* su = sub + b0 * S * 3;
        const float* qu = query + b0 * 3;
        const float* R_local = nullptr;
        if (m.single_transformer) {
            // shared encoder (model.py:320-323): x = cat(patch, shape - q); feat_local_global's QSTN sees and rotates all
            // P + S points (model.py:180-184); the rotated points go to bufB, which feat() reads only in its first layer,
            // before its STN64 reuses the buffer
            transform_points(pa, nullptr, nullptr, w.xall, Bc, P, PS, 0, st);
            transform_points(su, qu, nullptr, w.xall, Bc, S, PS, P, st);
            stn(m.enc.stn1, w.xall, Bc, PS, w, w.q4, st);
            launch_quat_to_rot(w.q4, w.R, Bc, st);
            transform_points(pa, nullptr, w.R, w.bufB, Bc, P, PS, 0, st);
            transform_points(su, qu, w.R, w.bufB, Bc, S, PS, P, st);
            float* fmax = w.fb_local;
            feat(m.enc, w.bufB, Bc, PS, w, fmax, st);
            debug_aux_copy(m, b0, Bc, w.R, fmax, nullptr, st);
            fc(m.fc1_enc, fmax, w.cat, Bc, true, st);                  // fc1_local_global + bn + ReLU (model.py:323)
            fc(m.fc2, w.cat, w.h3, Bc, true, st);
            fc(m.fc3, w.h3, w.h4, Bc, true, st);
            fc(m.fc4, w.h4, logits + b0 * m.fc4.cout, Bc, false, st);
            continue;
        }
        if (m.shared_qstn) {
            // feats = cat(patch, shape - q); trans = QSTN(feats)   (model.py:303,325-331)
            transform_points(pa, nullptr, nullptr, w.xall, Bc, P, PS, 0, st);
            transform_points(su, qu, nullptr, w.xall, Bc, S, PS, P, st);
            stn(m.point_stn, w.xall, Bc, PS, w, w.q4, st);
            launch_quat_to_rot(w.q4, w.R, Bc, st);
            transform_points(su, qu, w.R, w.sub_r, Bc, S, S, 0, st);
            transform_points(pa, nullptr, w.R, w.patch_r, Bc, P, P, 0, st);
        } else {
            transform_points(su, qu, nullptr, w.sub_r, Bc, S, S, 0, st);
            if (m.global.has_qstn) {
                // feat_global.stn1 on the centred sub-sample; the patch is rotated by it too (model.py:180-184,337-339)
                stn(m.global.stn1, w.sub_r, Bc, S, w, w.q4, st);
                launch_quat_to_rot(w.q4, w.R, Bc, st);
                transform_points(su, qu, w.R, w.sub_r, Bc, S, S, 0, st);
                R_local = w.R;
            }
            transform_points(pa, nullptr, R_local, w.patch_r, Bc, P, P, 0, st);
        }
        feat(m.global, w.sub_r, Bc, S, w, w.fb_global, st);
        feat(m.local, w.patch_r, Bc, P, w, w.fb_local, st);
        debug_aux_copy(m, b0, Bc, (m.shared_qstn || m.global.has_qstn) ? w.R : nullptr, w.fb_local, w.fb_global, st);
        // cat(local, global) after fc1_* + ReLU  (model.py:335,343,346)
        launch_gemm_nt(w.fb_local, 0, 1024, m.fc1_local.W, 0, m.fc1_local.b, w.cat, 0, 1024, (int)Bc, 512, 1024, 1, true, st);
        launch_gemm_nt(w.fb_global, 0, 1024, m.fc1_global.W, 0, m.fc1_global.b, w.cat + 512, 0, 1024, (int)Bc, 512, 1024, 1, true, st);
        fc(m.fc2, w.cat, w.h3, Bc, true, st);
        fc(m.fc3, w.h3, w.h4, Bc, true, st);
        fc(m.fc4, w.h4, logits + b0 * m.fc4.cout, Bc, false, st);   // logits [B][output_dim]
    }
}

}  // namespace p2s
