// K13: screened Poisson surface reconstruction (Kazhdan & Hoppe 2013) on a dense trilinear grid -- the SPSR baseline of
// eval_dataset.py:142-158, which the reference runs through meshlabserver and poisson.mlx.  The discrete system and the
// deviations from PoissonRecon are stated in include/p2s_b200.h; oracle/poisson_oracle.py assembles the same system
// with SciPy sparse matrices.
//   1. poisson_bbox_kernel: bounding box, non-finite and zero-normal counts (fixed-grid partials, finished on the host)
//   2. poisson_key_kernel + stable radix sort: points by the Morton key of their finest cell, so that every cell of
//      every depth is a contiguous run; points with a zero normal get a key past every cell and sort last
//   3. area weights a_p = (4h)^2 / n_c(p): n_c by a run-length encoding of the keys at depth d-2, found by binary search
//   4. poisson_fine_cells_kernel: per occupied finest cell, over its run in sorted order, the 36 values of
//      alpha sum a_p B B^T and the 24 of sum a_p n_p B; every coarser level's cell matrices from the <= 8 children by
//      P_c^T S P_c (exactly the screening term of the coarser basis, so the hierarchy is Galerkin)
//   5. V at the nodes by a gather over the <= 8 incident cells; b_j = sum_k V_k . (D M M, M D M, M M D)(k, j)
//   6. conjugate gradients preconditioned by one symmetric V-cycle: `iters` damped-Jacobi sweeps before and after the
//      coarse correction on every level (D = diag L + row sums of S), kCoarseSweeps sweeps on the 5^3 nodes of depth 2;
//      L is the matrix-free 27-point Q1 stencil, restriction P^T and prolongation P gather from the nested grid
//   7. point_weight 0 (singular): chi -= mean(chi).  iso = sum a_p chi(p) / sum a_p; the output is iso - chi (positive
//      inside) in fp32
// No float atomics: every sum runs in a fixed order, so the output is bitwise identical across runs.
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <vector>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <cub/device/device_scan.cuh>

namespace p2s {

namespace {

constexpr int kRedBlocks = 512;       // fixed grid of every reduction: partial sums in a fixed order
constexpr int kRedThreads = 256;
constexpr int kCoarseDepth = 2;       // coarsest multigrid level: 5^3 nodes
constexpr int kCoarseSweeps = 128;    // damped-Jacobi sweeps of the coarsest level (one thread block)
constexpr double kOmega = 2.0 / 3.0;  // Jacobi damping; lambda_max(D^-1 A) <= 1.5 for the Q1 stencil plus S
constexpr double kRelTol = 1e-5;      // stop at ||b - A chi|| / ||b|| <= kRelTol ...
constexpr int kMaxIters = 100;        // ... or after kMaxIters iterations ...
constexpr int kStallIters = 10;       // ... or when the residual has not reached a new minimum for kStallIters

enum { OP_APPLY, OP_RESIDUAL, OP_JACOBI };
enum { SC_RZ0, SC_RZ1, SC_PQ, SC_RR, SC_AREA, SC_ACHI, SC_XSUM, SC_COUNT };

// ---- Morton keys, 9 bits per axis: x in bit 3k+2, y in 3k+1, z in 3k; the parent cell's key is key >> 3
__host__ __device__ __forceinline__ uint32_t spread3(uint32_t v) {
    v &= 0x3ffu;
    v = (v | (v << 16)) & 0x030000FFu;
    v = (v | (v << 8)) & 0x0300F00Fu;
    v = (v | (v << 4)) & 0x030C30C3u;
    v = (v | (v << 2)) & 0x09249249u;
    return v;
}
__host__ __device__ __forceinline__ uint32_t compact3(uint32_t v) {
    v &= 0x09249249u;
    v = (v ^ (v >> 2)) & 0x030C30C3u;
    v = (v ^ (v >> 4)) & 0x0300F00Fu;
    v = (v ^ (v >> 8)) & 0x030000FFu;
    v = (v ^ (v >> 16)) & 0x3ffu;
    return v;
}
__device__ __forceinline__ int64_t dense_cell(uint32_t key, int n) {
    return ((int64_t)compact3(key >> 2) * n + compact3(key >> 1)) * n + compact3(key);
}
__device__ __forceinline__ int64_t nid(int i, int j, int l, int R) { return ((int64_t)i * R + j) * R + l; }

// upper-triangle index of (a, b) in a symmetric 8x8 matrix stored as 36 values
__host__ __device__ __forceinline__ int tri8(int a, int b) {
    if (a > b) { const int t = a; a = b; b = t; }
    return a * 8 - a * (a - 1) / 2 + (b - a);
}

// 1D integrals of the hat functions on nodes 0..n (spacing h = 1/n): mass M, stiffness K, D(i, j) = int phi_i phi_j'
__device__ __forceinline__ double mass1(int i, int j, int n, double h) {
    return i != j ? h / 6.0 : ((i == 0 || i == n) ? h / 3.0 : 2.0 * h / 3.0);
}
__device__ __forceinline__ double stiff1(int i, int j, int n, double h) {
    return i != j ? -1.0 / h : ((i == 0 || i == n) ? 1.0 / h : 2.0 / h);
}
__device__ __forceinline__ double deriv1(int i, int j, int n) {
    return j > i ? 0.5 : (j < i ? -0.5 : (i == 0 ? -0.5 : (i == n ? 0.5 : 0.0)));
}

// the grid coordinate u * 2^depth of a point, u = (p - origin) / edge in [0, 1]^3, and its finest cell
struct Frame {
    double o[3], edge;
    int n;
};
__device__ __forceinline__ double grid_coord(float p, const Frame& f, int a) { return ((double)p - f.o[a]) / f.edge * f.n; }
__device__ __forceinline__ int cell_of(double g, int n) { return min(max((int)floor(g), 0), n - 1); }

struct LevelView {
    int n;                  // cells per axis (2^depth); nodes 0..n per axis
    const int32_t* slot;    // [n^3] cell -> row of S, -1 when the cell holds no point
    const double* S;        // [cells][36] upper triangle of the cell's screening matrix
    const double* invD;     // [(n+1)^3] 1 / (diag L + row sum of S)
    double m_end, m_mid, m_off, k_end, k_mid, k_off;   // the entries of the 1D M and K (mass1 / stiff1)
};

// the row of the 1D M and K at node i: entries to nodes i-1, i, i+1 (0 beyond the ends), and the three node indices
// clamped into range (their entries are 0 where clamped)
__device__ __forceinline__ void row1(const LevelView& L, int i, double m[3], double k[3], int q[3]) {
    const bool end = i == 0 || i == L.n;
    m[0] = i > 0 ? L.m_off : 0.0;
    m[1] = end ? L.m_end : L.m_mid;
    m[2] = i < L.n ? L.m_off : 0.0;
    k[0] = i > 0 ? L.k_off : 0.0;
    k[1] = end ? L.k_end : L.k_mid;
    k[2] = i < L.n ? L.k_off : 0.0;
    q[0] = max(i - 1, 0);
    q[1] = i;
    q[2] = min(i + 1, L.n);
}

// (L + S) x at node (i, j, l): the 27-point stencil of K(x)M(x)M + M(x)K(x)M + M(x)M(x)K, then the screening rows of
// the <= 8 occupied cells around the node
__device__ __forceinline__ double apply_node(const LevelView& L, const double* __restrict__ x, int i, int j, int l) {
    const int n = L.n, R = n + 1;
    double mx[3], kx[3], my[3], ky[3], mz[3], kz[3];
    int qx[3], qy[3], qz[3];
    row1(L, i, mx, kx, qx);
    row1(L, j, my, ky, qy);
    row1(L, l, mz, kz, qz);
    double acc = 0.0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int b = 0; b < 3; ++b) {
            const double mxy = mx[a] * my[b], kmxy = kx[a] * my[b] + mx[a] * ky[b];
            const double* xr = x + ((int64_t)qx[a] * R + qy[b]) * R;
#pragma unroll
            for (int c = 0; c < 3; ++c) acc += (kmxy * mz[c] + mxy * kz[c]) * xr[qz[c]];
        }
    }
#pragma unroll
    for (int o = 0; o < 8; ++o) {
        const int cx = i - (o & 1), cy = j - ((o >> 1) & 1), cz = l - (o >> 2);
        if (cx < 0 || cy < 0 || cz < 0 || cx >= n || cy >= n || cz >= n) continue;
        const int s = L.slot[((int64_t)cx * n + cy) * n + cz];
        if (s < 0) continue;
        const double* S = L.S + (int64_t)s * 36;
#pragma unroll
        for (int m = 0; m < 8; ++m) acc += S[tri8(o, m)] * x[nid(cx + (m & 1), cy + ((m >> 1) & 1), cz + (m >> 2), R)];
    }
    return acc;
}

// node index -> (i, j, l) in 32-bit arithmetic (513^3 < 2^32)
__device__ __forceinline__ void node_ijl(int64_t v, int R, int& i, int& j, int& l) {
    const uint32_t u = (uint32_t)v, r = (uint32_t)R, t = u / r;
    l = (int)(u - t * r);
    j = (int)(t % r);
    i = (int)(t / r);
}

template <int OP>
__global__ void __launch_bounds__(256)
poisson_level_kernel(LevelView L, const double* __restrict__ x, const double* __restrict__ b, double* __restrict__ out) {
    const int R = L.n + 1;
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= (int64_t)R * R * R) return;
    int i, j, l;
    node_ijl(v, R, i, j, l);
    const double ax = apply_node(L, x, i, j, l);
    if (OP == OP_APPLY) out[v] = ax;
    else if (OP == OP_RESIDUAL) out[v] = b[v] - ax;
    else out[v] = x[v] + kOmega * L.invD[v] * (b[v] - ax);
}

// first Jacobi sweep from x = 0
__global__ void __launch_bounds__(256)
poisson_jacobi0_kernel(const double* __restrict__ invD, const double* __restrict__ b, int64_t nn, double* __restrict__ x) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v < nn) x[v] = kOmega * invD[v] * b[v];
}

// b_coarse = P^T r_fine: coarse node K gathers the fine nodes 2K + (-1, 0, 1)^3 with weights (1/2, 1, 1/2) per axis
__global__ void __launch_bounds__(256)
poisson_restrict_kernel(int nc, const double* __restrict__ rf, double* __restrict__ bc) {
    const int Rc = nc + 1, nf = 2 * nc, Rf = nf + 1;
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= (int64_t)Rc * Rc * Rc) return;
    int I, J, K;
    node_ijl(v, Rc, I, J, K);
    double acc = 0.0;
    for (int a = -1; a <= 1; ++a) {
        const int i = 2 * I + a;
        if (i < 0 || i > nf) continue;
        for (int b = -1; b <= 1; ++b) {
            const int j = 2 * J + b;
            if (j < 0 || j > nf) continue;
            const double wab = (a ? 0.5 : 1.0) * (b ? 0.5 : 1.0);
            for (int c = -1; c <= 1; ++c) {
                const int k = 2 * K + c;
                if (k < 0 || k > nf) continue;
                acc += wab * (c ? 0.5 : 1.0) * rf[nid(i, j, k, Rf)];
            }
        }
    }
    bc[v] = acc;
}

// x_fine += P x_coarse: an even fine index has one coarse parent (weight 1), an odd one two (1/2 each)
__global__ void __launch_bounds__(256)
poisson_prolong_add_kernel(int nc, const double* __restrict__ xc, double* __restrict__ xf) {
    const int Rc = nc + 1, Rf = 2 * nc + 1;
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= (int64_t)Rf * Rf * Rf) return;
    int i, j, l;
    node_ijl(v, Rf, i, j, l);
    const int i0 = i >> 1, j0 = j >> 1, l0 = l >> 1;
    const int ni = (i & 1) + 1, nj = (j & 1) + 1, nl = (l & 1) + 1;
    double acc = 0.0;
    for (int a = 0; a < ni; ++a)
        for (int b = 0; b < nj; ++b)
            for (int c = 0; c < nl; ++c) acc += xc[nid(i0 + a, j0 + b, l0 + c, Rc)];
    xf[v] += acc / (double)(ni * nj * nl);
}

// coarsest level: kCoarseSweeps damped-Jacobi sweeps from x = 0 in one block, the iterate in shared memory
__global__ void __launch_bounds__(128)
poisson_coarse_kernel(LevelView L, const double* __restrict__ b, double* __restrict__ x) {
    constexpr int R = (1 << kCoarseDepth) + 1, NN = R * R * R;
    __shared__ double buf[2][NN];
    const int t = threadIdx.x;
    const int i = t / (R * R), j = (t / R) % R, l = t % R;
    double bt = 0.0, dt = 0.0;
    if (t < NN) {
        bt = b[t];
        dt = L.invD[t];
        buf[0][t] = kOmega * dt * bt;
    }
    __syncthreads();
    int cur = 0;
    for (int s = 1; s < kCoarseSweeps; ++s) {
        if (t < NN) buf[cur ^ 1][t] = buf[cur][t] + kOmega * dt * (bt - apply_node(L, buf[cur], i, j, l));
        __syncthreads();
        cur ^= 1;
    }
    if (t < NN) x[t] = buf[cur][t];
}

// ---- fixed-order reductions: kRedBlocks partials (grid-stride, tree in shared memory), then one block over them
__device__ __forceinline__ double block_sum(double v, double* sh) {
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int w = blockDim.x / 2; w > 0; w >>= 1) {
        if ((int)threadIdx.x < w) sh[threadIdx.x] += sh[threadIdx.x + w];
        __syncthreads();
    }
    return sh[0];
}

// partial[block] = sum a_i b_i (b == nullptr: sum a_i)
__global__ void __launch_bounds__(kRedThreads)
poisson_dot_kernel(const double* __restrict__ a, const double* __restrict__ b, int64_t n, double* __restrict__ partial) {
    __shared__ double sh[kRedThreads];
    double s = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * kRedThreads + threadIdx.x; i < n; i += (int64_t)kRedBlocks * kRedThreads)
        s += b ? a[i] * b[i] : a[i];
    const double r = block_sum(s, sh);
    if (threadIdx.x == 0) partial[blockIdx.x] = r;
}

__global__ void __launch_bounds__(kRedBlocks) poisson_finish_kernel(const double* __restrict__ partial, double* out) {
    __shared__ double sh[kRedBlocks];
    const double r = block_sum(partial[threadIdx.x], sh);
    if (threadIdx.x == 0) *out = r;
}

__global__ void __launch_bounds__(256)
poisson_cg_x_kernel(const double* __restrict__ sc, int rz, const double* __restrict__ p, const double* __restrict__ q,
                    double* __restrict__ x, double* __restrict__ r, int64_t nn) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nn) return;
    const double pq = sc[SC_PQ];
    const double alpha = pq > 0.0 ? sc[rz] / pq : 0.0;   // breakdown: no step, the stall rule ends the iteration
    x[v] += alpha * p[v];
    r[v] -= alpha * q[v];
}

__global__ void __launch_bounds__(256)
poisson_cg_p_kernel(const double* __restrict__ sc, int rz_old, int rz_new, const double* __restrict__ z,
                    double* __restrict__ p, int64_t nn) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nn) return;
    const double beta = sc[rz_old] > 0.0 ? sc[rz_new] / sc[rz_old] : 0.0;
    p[v] = z[v] + beta * p[v];
}

// x -= mean(x), the sum in sc[SC_XSUM]
__global__ void __launch_bounds__(256)
poisson_sub_mean_kernel(const double* __restrict__ sc, double* __restrict__ x, int64_t nn) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v < nn) x[v] -= sc[SC_XSUM] / (double)nn;
}

// ---- points
// per block: min / max of the finite points, counts of non-finite points or normals and of zero normals
__global__ void __launch_bounds__(kRedThreads)
poisson_bbox_kernel(const float* __restrict__ pts, const float* __restrict__ nrm, int64_t N, float* __restrict__ box,
                    int64_t* __restrict__ counts) {
    __shared__ float sh[kRedThreads];
    __shared__ int64_t shc[kRedThreads];
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    int64_t bad = 0, zero = 0;
    for (int64_t i = (int64_t)blockIdx.x * kRedThreads + threadIdx.x; i < N; i += (int64_t)kRedBlocks * kRedThreads) {
        const float p0 = pts[3 * i], p1 = pts[3 * i + 1], p2 = pts[3 * i + 2];
        const float n0 = nrm[3 * i], n1 = nrm[3 * i + 1], n2 = nrm[3 * i + 2];
        const bool fin = isfinite(p0) && isfinite(p1) && isfinite(p2) && isfinite(n0) && isfinite(n1) && isfinite(n2);
        if (!fin) { ++bad; continue; }
        zero += (n0 == 0.f && n1 == 0.f && n2 == 0.f) ? 1 : 0;
        lo[0] = fminf(lo[0], p0); lo[1] = fminf(lo[1], p1); lo[2] = fminf(lo[2], p2);
        hi[0] = fmaxf(hi[0], p0); hi[1] = fmaxf(hi[1], p1); hi[2] = fmaxf(hi[2], p2);
    }
    const int t = threadIdx.x;
    for (int k = 0; k < 6; ++k) {
        sh[t] = k < 3 ? lo[k] : hi[k - 3];
        __syncthreads();
        for (int w = kRedThreads / 2; w > 0; w >>= 1) {
            if (t < w) sh[t] = k < 3 ? fminf(sh[t], sh[t + w]) : fmaxf(sh[t], sh[t + w]);
            __syncthreads();
        }
        if (t == 0) box[blockIdx.x * 6 + k] = sh[0];
        __syncthreads();
    }
    for (int k = 0; k < 2; ++k) {
        shc[t] = k == 0 ? bad : zero;
        __syncthreads();
        for (int w = kRedThreads / 2; w > 0; w >>= 1) {
            if (t < w) shc[t] += shc[t + w];
            __syncthreads();
        }
        if (t == 0) counts[blockIdx.x * 2 + k] = shc[0];
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256)
poisson_key_kernel(const float* __restrict__ pts, const float* __restrict__ nrm, int64_t N, Frame f, int depth,
                   uint32_t* __restrict__ keys, int32_t* __restrict__ idx) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const bool zero = nrm[3 * i] == 0.f && nrm[3 * i + 1] == 0.f && nrm[3 * i + 2] == 0.f;
    uint32_t c[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) c[a] = (uint32_t)cell_of(grid_coord(pts[3 * i + a], f, a), f.n);
    keys[i] = zero ? (1u << (3 * depth)) : (spread3(c[0]) << 2 | spread3(c[1]) << 1 | spread3(c[2]));
    idx[i] = (int32_t)i;
}

// sorted point p: grid coordinates g [3][Nk] and unit normal un [3][Nk] (SoA)
__global__ void __launch_bounds__(256)
poisson_gather_kernel(const int32_t* __restrict__ order, int64_t Nk, const float* __restrict__ pts,
                      const float* __restrict__ nrm, Frame f, double* __restrict__ g, double* __restrict__ un) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= Nk) return;
    const int64_t i = order[p];
    const double n0 = nrm[3 * i], n1 = nrm[3 * i + 1], n2 = nrm[3 * i + 2];
    const double len = sqrt(n0 * n0 + n1 * n1 + n2 * n2);
#pragma unroll
    for (int a = 0; a < 3; ++a) g[a * Nk + p] = grid_coord(pts[3 * i + a], f, a);
    un[p] = n0 / len;
    un[Nk + p] = n1 / len;
    un[2 * Nk + p] = n2 / len;
}

__global__ void __launch_bounds__(256)
poisson_shift_kernel(const uint32_t* __restrict__ in, int64_t n, int shift, uint32_t* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[i] >> shift;
}

// a_p = (4h)^2 / (number of points in p's cell at depth d - 2)
__global__ void __launch_bounds__(256)
poisson_area_kernel(const uint32_t* __restrict__ keys, int64_t Nk, int shift, const uint32_t* __restrict__ ukey,
                    const int32_t* __restrict__ cnt, int nruns, double a_num, double* __restrict__ area) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= Nk) return;
    const uint32_t k = keys[p] >> shift;
    int lo = 0, hi = nruns - 1;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (ukey[mid] < k) lo = mid + 1;
        else hi = mid;
    }
    area[p] = a_num / (double)cnt[lo];
}

// per occupied finest cell, over its points in sorted order: S = alpha sum a_p B B^T (36) and W = sum a_p n_p B (8 x 3)
__global__ void __launch_bounds__(128)
poisson_fine_cells_kernel(const uint32_t* __restrict__ ukey, const int32_t* __restrict__ start,
                          const int32_t* __restrict__ cnt, int ncell, int n, const double* __restrict__ g,
                          const double* __restrict__ un, const double* __restrict__ area, int64_t Nk, double alpha,
                          int32_t* __restrict__ slot, double* __restrict__ S, double* __restrict__ W) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= ncell) return;
    const uint32_t key = ukey[c];
    slot[dense_cell(key, n)] = c;
    const double cx = compact3(key >> 2), cy = compact3(key >> 1), cz = compact3(key);
    double s[36], w[24];
#pragma unroll
    for (int k = 0; k < 36; ++k) s[k] = 0.0;
#pragma unroll
    for (int k = 0; k < 24; ++k) w[k] = 0.0;
    const int64_t p0 = start[c], p1 = p0 + cnt[c];
    for (int64_t p = p0; p < p1; ++p) {
        const double tx = g[p] - cx, ty = g[Nk + p] - cy, tz = g[2 * Nk + p] - cz;
        const double bx[2] = {1.0 - tx, tx}, by[2] = {1.0 - ty, ty}, bz[2] = {1.0 - tz, tz};
        double bm[8];
#pragma unroll
        for (int m = 0; m < 8; ++m) bm[m] = bx[m & 1] * by[(m >> 1) & 1] * bz[m >> 2];
        const double ap = area[p], ca = alpha * ap;
        const double an[3] = {ap * un[p], ap * un[Nk + p], ap * un[2 * Nk + p]};
#pragma unroll
        for (int m = 0; m < 8; ++m)
#pragma unroll
            for (int k = 0; k < 3; ++k) w[m * 3 + k] += an[k] * bm[m];
#pragma unroll
        for (int a = 0; a < 8; ++a)
#pragma unroll
            for (int b = a; b < 8; ++b) s[tri8(a, b)] += ca * (bm[a] * bm[b]);
    }
#pragma unroll
    for (int k = 0; k < 36; ++k) S[(int64_t)c * 36 + k] = s[k];
#pragma unroll
    for (int k = 0; k < 24; ++k) W[(int64_t)c * 24 + k] = w[k];
}

// the coarse basis at a child corner: child corner m of child e sits at (e + m) / 2 of the coarse cell per axis
__device__ __forceinline__ double child_weight(int e, int m, int M) {
    double w = 1.0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double q = 0.5 * (((e >> a) & 1) + ((m >> a) & 1));
        w *= ((M >> a) & 1) ? q : 1.0 - q;
    }
    return w;
}

// coarse cell matrix = sum over the occupied children (in child order) of P_c^T S_child P_c
__global__ void __launch_bounds__(128)
poisson_coarse_cells_kernel(const uint32_t* __restrict__ ukey, int ncell, int n, LevelView fine,
                            int32_t* __restrict__ slot, double* __restrict__ S) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= ncell) return;
    const uint32_t key = ukey[c];
    slot[dense_cell(key, n)] = c;
    double acc[36];
#pragma unroll
    for (int k = 0; k < 36; ++k) acc[k] = 0.0;
    for (int e = 0; e < 8; ++e) {
        const int s = fine.slot[dense_cell((key << 3) | (uint32_t)(((e & 1) << 2) | (e & 2) | ((e >> 2) & 1)), 2 * n)];
        if (s < 0) continue;
        const double* Sf = fine.S + (int64_t)s * 36;
#pragma unroll
        for (int A = 0; A < 8; ++A) {
            double u[8];
#pragma unroll
            for (int mp = 0; mp < 8; ++mp) {
                double t = 0.0;
#pragma unroll
                for (int m = 0; m < 8; ++m) t += child_weight(e, m, A) * Sf[tri8(m, mp)];
                u[mp] = t;
            }
#pragma unroll
            for (int B = A; B < 8; ++B) {
                double t = 0.0;
#pragma unroll
                for (int mp = 0; mp < 8; ++mp) t += u[mp] * child_weight(e, mp, B);
                acc[tri8(A, B)] += t;
            }
        }
    }
#pragma unroll
    for (int k = 0; k < 36; ++k) S[(int64_t)c * 36 + k] = acc[k];
}

__global__ void __launch_bounds__(256) poisson_invdiag_kernel(LevelView L, double* __restrict__ invD) {
    const int n = L.n, R = n + 1;
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= (int64_t)R * R * R) return;
    int i, j, l;
    node_ijl(v, R, i, j, l);
    const double h = 1.0 / n;
    const double mi = mass1(i, i, n, h), mj = mass1(j, j, n, h), ml = mass1(l, l, n, h);
    double d = stiff1(i, i, n, h) * mj * ml + mi * stiff1(j, j, n, h) * ml + mi * mj * stiff1(l, l, n, h);
    for (int o = 0; o < 8; ++o) {
        const int cx = i - (o & 1), cy = j - ((o >> 1) & 1), cz = l - (o >> 2);
        if (cx < 0 || cy < 0 || cz < 0 || cx >= n || cy >= n || cz >= n) continue;
        const int s = L.slot[((int64_t)cx * n + cy) * n + cz];
        if (s < 0) continue;
        for (int m = 0; m < 8; ++m) d += L.S[(int64_t)s * 36 + tri8(o, m)];
    }
    invD[v] = 1.0 / d;
}

// V_k = sum over the incident occupied cells of their corner sums, / h^3  -> V [3][nodes]
__global__ void __launch_bounds__(256)
poisson_vfield_kernel(int n, const int32_t* __restrict__ slot, const double* __restrict__ W, double* __restrict__ V) {
    const int R = n + 1;
    const int64_t nn = (int64_t)R * R * R;
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nn) return;
    int i, j, l;
    node_ijl(v, R, i, j, l);
    const double inv_h3 = (double)n * n * n;
    double acc[3] = {0.0, 0.0, 0.0};
    for (int o = 0; o < 8; ++o) {
        const int cx = i - (o & 1), cy = j - ((o >> 1) & 1), cz = l - (o >> 2);
        if (cx < 0 || cy < 0 || cz < 0 || cx >= n || cy >= n || cz >= n) continue;
        const int s = slot[((int64_t)cx * n + cy) * n + cz];
        if (s < 0) continue;
#pragma unroll
        for (int k = 0; k < 3; ++k) acc[k] += W[(int64_t)s * 24 + o * 3 + k];
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) V[k * nn + v] = acc[k] * inv_h3;
}

// b_j = sum_k V_k . (D(k_x, j_x) M M, M D(k_y, j_y) M, M M D(k_z, j_z)) over the 27 nodes k around j
__global__ void __launch_bounds__(256) poisson_rhs_kernel(int n, const double* __restrict__ V, double* __restrict__ b) {
    const int R = n + 1;
    const int64_t nn = (int64_t)R * R * R;
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nn) return;
    int i, j, l;
    node_ijl(v, R, i, j, l);
    const double h = 1.0 / n;
    double acc = 0.0;
    for (int a = (i > 0 ? -1 : 0); a <= (i < n ? 1 : 0); ++a) {
        const double mx = mass1(i + a, i, n, h), dx = deriv1(i + a, i, n);
        for (int b = (j > 0 ? -1 : 0); b <= (j < n ? 1 : 0); ++b) {
            const double my = mass1(j + b, j, n, h), dy = deriv1(j + b, j, n);
            for (int c = (l > 0 ? -1 : 0); c <= (l < n ? 1 : 0); ++c) {
                const double mz = mass1(l + c, l, n, h), dz = deriv1(l + c, l, n);
                const int64_t k = nid(i + a, j + b, l + c, R);
                acc += V[k] * (dx * my * mz) + V[nn + k] * (mx * dy * mz) + V[2 * nn + k] * (mx * my * dz);
            }
        }
    }
    b[v] = acc;
}

// chi at every sorted point (trilinear in its finest cell)
__global__ void __launch_bounds__(256)
poisson_point_chi_kernel(const double* __restrict__ g, int64_t Nk, int n, const double* __restrict__ chi,
                         double* __restrict__ out) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= Nk) return;
    const int R = n + 1;
    int c[3];
    double t[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double ga = g[a * Nk + p];
        c[a] = cell_of(ga, n);
        t[a] = ga - c[a];
    }
    double acc = 0.0;
#pragma unroll
    for (int m = 0; m < 8; ++m) {
        const double w = ((m & 1) ? t[0] : 1.0 - t[0]) * (((m >> 1) & 1) ? t[1] : 1.0 - t[1]) * ((m >> 2) ? t[2] : 1.0 - t[2]);
        acc += w * chi[nid(c[0] + (m & 1), c[1] + ((m >> 1) & 1), c[2] + (m >> 2), R)];
    }
    out[p] = acc;
}

__global__ void __launch_bounds__(256)
poisson_output_kernel(const double* __restrict__ chi, const double* __restrict__ sc, int64_t nn, float* __restrict__ out) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nn) return;
    const double iso = sc[SC_ACHI] / sc[SC_AREA];
    out[v] = (float)(iso - chi[v]);
}

// ---- host side
struct Level {
    int n = 0;
    int64_t nn = 0, ncell = 0;
    uint32_t* ukey = nullptr;
    int32_t* slot = nullptr;
    double *S = nullptr, *invD = nullptr, *x = nullptr, *b = nullptr, *r = nullptr, *t = nullptr;
    LevelView view() const {   // the expressions of mass1 / stiff1
        const double h = 1.0 / n;
        return LevelView{n, slot, S, invD, h / 3.0, 2.0 * h / 3.0, h / 6.0, 1.0 / h, 2.0 / h, -1.0 / h};
    }
};

struct Solver {
    std::vector<Level> lv;   // by depth
    int depth = 0, nu = 0;
    double* partial = nullptr;
    double* sc = nullptr;
    cudaStream_t st = nullptr;

    void dot(const double* a, const double* b, int64_t n, int slot_out) {
        P2S_LAUNCH(poisson_dot_kernel, kRedBlocks, kRedThreads, 0, st, a, b, n, partial);
        P2S_LAUNCH(poisson_finish_kernel, 1, kRedBlocks, 0, st, partial, sc + slot_out);
    }
    template <int OP>
    void level_op(const Level& L, const double* x, const double* b, double* out) {
        P2S_LAUNCH(poisson_level_kernel<OP>, grid1d(L.nn, 256), 256, 0, st, L.view(), x, b, out);
    }
    // x = V-cycle(b) on level l
    void vcycle(int l, const double* b, double* x) {
        const Level& L = lv[l];
        if (l == kCoarseDepth) {
            P2S_LAUNCH(poisson_coarse_kernel, 1, 128, 0, st, L.view(), b, x);
            return;
        }
        // 2 nu - 1 ping-pong swaps follow the first sweep, so starting in t leaves the result in x
        double *cur = L.t, *oth = x;
        P2S_LAUNCH(poisson_jacobi0_kernel, grid1d(L.nn, 256), 256, 0, st, L.invD, b, L.nn, cur);
        for (int s = 1; s < nu; ++s) {
            level_op<OP_JACOBI>(L, cur, b, oth);
            std::swap(cur, oth);
        }
        level_op<OP_RESIDUAL>(L, cur, b, L.r);
        const Level& C = lv[l - 1];
        P2S_LAUNCH(poisson_restrict_kernel, grid1d(C.nn, 256), 256, 0, st, C.n, L.r, C.b);
        vcycle(l - 1, C.b, C.x);
        P2S_LAUNCH(poisson_prolong_add_kernel, grid1d(L.nn, 256), 256, 0, st, C.n, C.x, cur);
        for (int s = 0; s < nu; ++s) {
            level_op<OP_JACOBI>(L, cur, b, oth);
            std::swap(cur, oth);
        }
        if (cur != x) P2S_CUDA(cudaMemcpyAsync(x, cur, (size_t)L.nn * sizeof(double), cudaMemcpyDeviceToDevice, st));
    }
};

}  // namespace

void poisson_solve(const float* pts, const float* nrm, int64_t N, const p2s_poisson_config& cfg, float* values,
                   int64_t cap, p2s_poisson_report* rep, cudaStream_t st) {
    P2S_CHECK(cfg.depth >= 2 && cfg.depth <= 9, "depth must be in [2, 9]");
    P2S_CHECK(std::isfinite(cfg.point_weight) && cfg.point_weight >= 0.f, "point_weight must be finite and >= 0");
    P2S_CHECK(std::isfinite(cfg.scale) && cfg.scale >= 1.f, "scale must be finite and >= 1");
    P2S_CHECK(cfg.iters >= 1 && cfg.iters <= 64, "iters must be in [1, 64]");
    const int d = cfg.depth, n = 1 << d, R = n + 1;
    const int64_t nn = (int64_t)R * R * R;
    std::memset(rep, 0, sizeof(*rep));
    rep->grid_res = R;
    if (!values && cap == 0) return;   // size query
    P2S_CHECK(values && cap >= nn, "values must hold (2^depth + 1)^3 floats");
    P2S_CHECK(pts && nrm, "null argument");
    P2S_CHECK(N > 0, "no points");
    P2S_CHECK(N < (1ll << 31) - 1, "too many points for 32-bit indices");

    cudaEvent_t ev[5];
    for (auto& e : ev) P2S_CUDA(cudaEventCreate(&e));
    struct EvGuard {
        cudaEvent_t* e;
        ~EvGuard() { for (int k = 0; k < 5; ++k) cudaEventDestroy(e[k]); }
    } evg{ev};
    P2S_CUDA(cudaEventRecord(ev[0], st));
    static thread_local std::vector<Workspace> t_ws;
    Workspace& ws = for_device(t_ws).begin(st);

    // 1. bounding box and input checks
    float* box = ws.get<float>(kRedBlocks * 6);
    int64_t* counts = ws.get<int64_t>(kRedBlocks * 2);
    P2S_LAUNCH(poisson_bbox_kernel, kRedBlocks, kRedThreads, 0, st, pts, nrm, N, box, counts);
    const std::vector<float> hbox = read_back(box, kRedBlocks * 6, st);
    const std::vector<int64_t> hcnt = read_back(counts, kRedBlocks * 2, st);
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    int64_t bad = 0, dropped = 0;
    for (int b = 0; b < kRedBlocks; ++b) {
        for (int a = 0; a < 3; ++a) {
            lo[a] = std::min(lo[a], hbox[b * 6 + a]);
            hi[a] = std::max(hi[a], hbox[b * 6 + 3 + a]);
        }
        bad += hcnt[b * 2];
        dropped += hcnt[b * 2 + 1];
    }
    P2S_CHECK(bad == 0, "non-finite point or normal");
    const int64_t Nk = N - dropped;
    P2S_CHECK(Nk > 0, "every normal has zero length");
    double ext = 0.0;
    for (int a = 0; a < 3; ++a) ext = std::max(ext, (double)hi[a] - (double)lo[a]);
    P2S_CHECK(ext > 0.0, "all points are identical (zero extent)");
    Frame f;
    f.edge = (double)cfg.scale * ext;
    f.n = n;
    for (int a = 0; a < 3; ++a) f.o[a] = 0.5 * ((double)lo[a] + (double)hi[a]) - 0.5 * f.edge;
    for (int a = 0; a < 3; ++a) rep->origin[a] = f.o[a];
    rep->edge = f.edge;
    rep->points_used = Nk;
    rep->dropped_points = dropped;

    // 2. sort by the Morton key of the finest cell
    uint32_t* key_in = ws.get<uint32_t>(N);
    uint32_t* key = ws.get<uint32_t>(N);
    int32_t* idx_in = ws.get<int32_t>(N);
    int32_t* order = ws.get<int32_t>(N);
    P2S_LAUNCH(poisson_key_kernel, grid1d(N, 256), 256, 0, st, pts, nrm, N, f, d, key_in, idx_in);
    cub_run(ws, 1, [&](void* t, size_t& b) {
        return cub::DeviceRadixSort::SortPairs(t, b, key_in, key, idx_in, order, (int)N, 0, 3 * d + 1, st);
    });
    double* g = ws.get<double>(3 * Nk);
    double* un = ws.get<double>(3 * Nk);
    P2S_LAUNCH(poisson_gather_kernel, grid1d(Nk, 256), 256, 0, st, order, Nk, pts, nrm, f, g, un);

    // 3. area weights from the point count of the depth d-2 cell
    int32_t* d_num = ws.get<int32_t>(1);
    uint32_t* skey = ws.get<uint32_t>(Nk);
    uint32_t* ukey_dens = ws.get<uint32_t>(Nk);
    int32_t* cnt_dens = ws.get<int32_t>(Nk);
    double* area = ws.get<double>(Nk);
    P2S_LAUNCH(poisson_shift_kernel, grid1d(Nk, 256), 256, 0, st, key, Nk, 6, skey);
    cub_run(ws, 1, [&](void* t, size_t& b) {
        return cub::DeviceRunLengthEncode::Encode(t, b, skey, ukey_dens, cnt_dens, d_num, (int)Nk, st);
    });
    const int ndens = read_back(d_num, 1, st)[0];
    P2S_LAUNCH(poisson_area_kernel, grid1d(Nk, 256), 256, 0, st, key, Nk, 6, ukey_dens, cnt_dens, ndens, 16.0 / ((double)n * n),
               area);

    // 4. cells of every level
    Solver sv;
    sv.st = st;
    sv.depth = d;
    sv.nu = cfg.iters;
    sv.lv.resize(d + 1);
    sv.partial = ws.get<double>(kRedBlocks);
    sv.sc = ws.get<double>(SC_COUNT);
    const double alpha = (double)cfg.point_weight * (double)n;
    int32_t* cell_cnt = ws.get<int32_t>(Nk);
    int32_t* cell_start = ws.get<int32_t>(Nk);
    double* W = nullptr;
    for (int l = d; l >= kCoarseDepth; --l) {
        Level& L = sv.lv[l];
        L.n = 1 << l;
        L.nn = (int64_t)(L.n + 1) * (L.n + 1) * (L.n + 1);
        const int64_t ncells_dense = (int64_t)L.n * L.n * L.n;
        if (l == d) {
            L.ukey = ws.get<uint32_t>(Nk);
            cub_run(ws, 1, [&](void* t, size_t& b) {
                return cub::DeviceRunLengthEncode::Encode(t, b, key, L.ukey, cell_cnt, d_num, (int)Nk, st);
            });
        } else {
            const Level& F = sv.lv[l + 1];
            L.ukey = ws.get<uint32_t>(F.ncell);
            P2S_LAUNCH(poisson_shift_kernel, grid1d(F.ncell, 256), 256, 0, st, F.ukey, F.ncell, 3, skey);
            cub_run(ws, 1, [&](void* t, size_t& b) {
                return cub::DeviceRunLengthEncode::Encode(t, b, skey, L.ukey, cell_cnt, d_num, (int)F.ncell, st);
            });
        }
        L.ncell = read_back(d_num, 1, st)[0];
        L.slot = ws.get<int32_t>(ncells_dense);
        L.S = ws.get<double>(L.ncell * 36);
        P2S_CUDA(cudaMemsetAsync(L.slot, 0xff, (size_t)ncells_dense * sizeof(int32_t), st));
        if (l == d) {
            cub_run(ws, 1, [&](void* t, size_t& b) {
                return cub::DeviceScan::ExclusiveSum(t, b, cell_cnt, cell_start, (int)L.ncell, st);
            });
            W = ws.get<double>(L.ncell * 24);
            P2S_LAUNCH(poisson_fine_cells_kernel, (unsigned)cdiv(L.ncell, 128), 128, 0, st, L.ukey, cell_start, cell_cnt,
                       (int)L.ncell, L.n, g, un, area, Nk, alpha, L.slot, L.S, W);
            rep->occupied_cells = L.ncell;
        } else {
            P2S_LAUNCH(poisson_coarse_cells_kernel, (unsigned)cdiv(L.ncell, 128), 128, 0, st, L.ukey, (int)L.ncell, L.n,
                       sv.lv[l + 1].view(), L.slot, L.S);
        }
        L.invD = ws.get<double>(L.nn);
        P2S_LAUNCH(poisson_invdiag_kernel, grid1d(L.nn, 256), 256, 0, st, L.view(), L.invD);
        L.t = ws.get<double>(L.nn);
        L.r = ws.get<double>(L.nn);
        if (l < d) {
            L.x = ws.get<double>(L.nn);
            L.b = ws.get<double>(L.nn);
        }
    }
    P2S_CUDA(cudaEventRecord(ev[1], st));

    // 5. right-hand side
    const Level& Fl = sv.lv[d];
    double* V = ws.get<double>(3 * nn);
    double* B = ws.get<double>(nn);
    P2S_LAUNCH(poisson_vfield_kernel, grid1d(nn, 256), 256, 0, st, n, Fl.slot, W, V);
    P2S_LAUNCH(poisson_rhs_kernel, grid1d(nn, 256), 256, 0, st, n, V, B);
    P2S_CUDA(cudaEventRecord(ev[2], st));

    // 6. MG-preconditioned CG from chi = 0
    double* X = ws.get<double>(nn);
    double* Rr = ws.get<double>(nn);
    double* Z = ws.get<double>(nn);
    double* P = ws.get<double>(nn);
    double* Q = ws.get<double>(nn);
    P2S_CUDA(cudaMemsetAsync(X, 0, (size_t)nn * sizeof(double), st));
    P2S_CUDA(cudaMemcpyAsync(Rr, B, (size_t)nn * sizeof(double), cudaMemcpyDeviceToDevice, st));
    sv.dot(B, B, nn, SC_RR);
    const double bb = read_back(sv.sc + SC_RR, 1, st)[0];
    int it = 0;
    double residual = 0.0;
    if (bb > 0.0) {
        int rz = SC_RZ0;
        sv.vcycle(d, Rr, Z);
        sv.dot(Rr, Z, nn, rz);
        P2S_CUDA(cudaMemcpyAsync(P, Z, (size_t)nn * sizeof(double), cudaMemcpyDeviceToDevice, st));
        double best = INFINITY;
        int stall = 0;
        while (it < kMaxIters) {
            sv.level_op<OP_APPLY>(Fl, P, nullptr, Q);
            sv.dot(P, Q, nn, SC_PQ);
            P2S_LAUNCH(poisson_cg_x_kernel, grid1d(nn, 256), 256, 0, st, sv.sc, rz, P, Q, X, Rr, nn);
            sv.dot(Rr, Rr, nn, SC_RR);
            ++it;
            const double rel = std::sqrt(read_back(sv.sc + SC_RR, 1, st)[0] / bb);
            if (!(rel > kRelTol)) break;   // converged (or not a number: stop)
            if (rel < best) {
                best = rel;
                stall = 0;
            } else if (++stall >= kStallIters) {
                break;
            }
            sv.vcycle(d, Rr, Z);
            sv.dot(Rr, Z, nn, rz ^ 1);
            P2S_LAUNCH(poisson_cg_p_kernel, grid1d(nn, 256), 256, 0, st, sv.sc, rz, rz ^ 1, Z, P, nn);
            rz ^= 1;
        }
        sv.level_op<OP_RESIDUAL>(Fl, X, B, Rr);   // report the true residual, not the recursive one
        sv.dot(Rr, Rr, nn, SC_RR);
        residual = std::sqrt(read_back(sv.sc + SC_RR, 1, st)[0] / bb);
    }
    // point_weight 0: S = 0 and L 1 = 0, so chi is only defined up to a constant, which CG leaves wherever the V-cycles
    // put it; take the solution of mean zero so that chi and iso are defined (values = iso - chi does not change)
    if (alpha == 0.0) {
        sv.dot(X, nullptr, nn, SC_XSUM);
        P2S_LAUNCH(poisson_sub_mean_kernel, grid1d(nn, 256), 256, 0, st, sv.sc, X, nn);
    }
    rep->iterations = it;
    rep->residual = residual;
    P2S_CUDA(cudaEventRecord(ev[3], st));

    // 7. iso-value and output
    double* chi_p = ws.get<double>(Nk);
    P2S_LAUNCH(poisson_point_chi_kernel, grid1d(Nk, 256), 256, 0, st, g, Nk, n, X, chi_p);
    sv.dot(area, nullptr, Nk, SC_AREA);
    sv.dot(area, chi_p, Nk, SC_ACHI);
    P2S_LAUNCH(poisson_output_kernel, grid1d(nn, 256), 256, 0, st, X, sv.sc, nn, values);
    P2S_CUDA(cudaEventRecord(ev[4], st));
    const std::vector<double> s2 = read_back(sv.sc + SC_AREA, 2, st);
    rep->iso = s2[1] / s2[0];
    for (int k = 0; k < 4; ++k) P2S_CUDA(cudaEventElapsedTime(&rep->stage_ms[k], ev[k], ev[k + 1]));
}

}  // namespace p2s
