// Oriented normals of an unstructured point cloud (rules in include/p2s_b200.h, "Point normals").
//   a. nrm_knn_kernel: the K nearest points of every point (itself included), exact: k smallest float64 distances on
//      the fp32 coordinates, ascending, lowest id on ties -- the semantics of knn_patch_kernel.  That kernel is
//      exhaustive and its fast path needs queries closer together than a quarter of the k-th distance, which cloud
//      points with K ~ 10 never are; this one walks the cloud's cell index (cloud_index_build, assemble.cu): one thread
//      per point in cell order, its own cell first, then every cell whose tight box is not farther than the current
//      K-th distance.  The box bound is computed with the same rounded operations as the distances, so it never
//      exceeds the distance of a point inside the box and pruning loses nothing.
//   b. nrm_fit_kernel: float64 centroid and scatter matrix of the K neighbours, cyclic Jacobi, eigenvector of the
//      smallest eigenvalue, rounded to fp32, deterministic pre-sign.
//   c. orientation.  viewpoint: one kernel.  propagate: the minimum spanning forest of the symmetrised kNN graph under
//      the total order (cost bits, min id, max id), which is unique, then signs along it from each component's root.
//        - nrm_edge_kernel writes one entry per (point, neighbour slot); two stable radix sorts put them in the total
//          order, so an edge's rank is a 32-bit integer (both copies of a mutual pair are adjacent and name the same edge)
//        - Boruvka rounds: nrm_findmin_kernel (atomicMin of the rank per component), nrm_hook_kernel (every component
//          hooks onto the other side of its edge; of a mutual pair the lower id stays root), ceil(log2 N) + 1 pointer
//          jumps, nrm_flat_kernel checks that every label is a root.  The host reads the hook count back after every
//          round and stops at the first round without one; more than ceil(log2 N) + 1 rounds is an error.
//        - roots by 64-bit atomicMax of (z, -id); level-synchronous sweeps over the forest edges set (parent, flip) of
//          every point in one 32-bit word.  The host reads the visited count back every 64 sweeps; more than N sweeps,
//          or a forest that does not reach every point, is an error.
//      The forest and the signs are functions of the input alone: integer atomics only, and which sweep reaches a point
//      does not change what it receives.
#include "common.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cmath>

namespace p2s {

namespace {

constexpr int kT = 256;
constexpr int kMaxK = 64;
constexpr int kCells = kCloudGrid * kCloudGrid * kCloudGrid;
constexpr unsigned long long kNoEdge = ~0ull;
constexpr int kNoRank = 0x7f7f7f7f;          // what cudaMemset(0x7f) leaves in an int
constexpr int kSweepBatch = 64;

// flags[0]: non-finite values in a (and b), flags[1]: ids outside [0, N)
__global__ void __launch_bounds__(kT)
nrm_check_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t nf, const int32_t* __restrict__ ids,
                 int64_t nids, int N, unsigned* __restrict__ flags) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool nonfinite = false, bad = false;
    if (i < nf) nonfinite = !isfinite(a[i]) || (b && !isfinite(b[i]));
    if (ids && i < nids) { const int32_t x = ids[i]; bad = x < 0 || x >= N; }
    const unsigned n0 = __popc(__ballot_sync(0xffffffffu, nonfinite)), n1 = __popc(__ballot_sync(0xffffffffu, bad));
    if ((threadIdx.x & 31) == 0) {
        if (n0) atomicAdd(&flags[0], n0);
        if (n1) atomicAdd(&flags[1], n1);
    }
}

// cKDTree's squared distance: (dx*dx + dy*dy) + dz*dz in float64, every operation rounded (dist2_f64 of assemble.cu)
__device__ __forceinline__ double d2_rn(double dx, double dy, double dz) {
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

__global__ void __launch_bounds__(128)
nrm_knn_kernel(const CloudIndex ix, int N, int K, int32_t* __restrict__ ids_out) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;      // position in cell order
    if (t >= N) return;
    const float* __restrict__ spts = ix.spts;
    const double qx = spts[t * 3 + 0], qy = spts[t * 3 + 1], qz = spts[t * 3 + 2];
    double kd[kMaxK];
    int ki[kMaxK];
    int n = 0;
    auto scan_cell = [&](int c) {
        const int end = ix.start[c + 1];
        for (int j = ix.start[c]; j < end; ++j) {
            const double d = d2_rn((double)spts[j * 3 + 0] - qx, (double)spts[j * 3 + 1] - qy, (double)spts[j * 3 + 2] - qz);
            const int id = ix.perm[j];
            if (n == K && !(d < kd[K - 1] || (d == kd[K - 1] && id < ki[K - 1]))) continue;
            int p = n < K ? n++ : K - 1;
            while (p > 0 && (kd[p - 1] > d || (kd[p - 1] == d && ki[p - 1] > id))) { kd[p] = kd[p - 1]; ki[p] = ki[p - 1]; --p; }
            kd[p] = d; ki[p] = id;
        }
    };
    int lo = 0, hi = kCells;                                  // own cell: the last c with start[c] <= t
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (ix.start[mid] <= t) lo = mid; else hi = mid; }
    const int own = lo;
    scan_cell(own);
    for (int c = 0; c < kCells; ++c) {
        if (c == own || ix.start[c + 1] == ix.start[c]) continue;
        if (n == K) {
            const float* __restrict__ b = ix.cbox + c * 6;
            const double bx = fmax(fmax((double)b[0] - qx, qx - (double)b[3]), 0.0);
            const double by = fmax(fmax((double)b[1] - qy, qy - (double)b[4]), 0.0);
            const double bz = fmax(fmax((double)b[2] - qz, qz - (double)b[5]), 0.0);
            if (d2_rn(bx, by, bz) > kd[K - 1]) continue;
        }
        scan_cell(c);
    }
    int32_t* __restrict__ o = ids_out + (int64_t)ix.perm[t] * K;
    for (int s = 0; s < K; ++s) o[s] = ki[s];
}

// one Jacobi rotation that zeroes a[P][Q] of the symmetric matrix a (upper triangle kept); v accumulates the rotations
template <int P, int Q>
__device__ __forceinline__ void jacobi_rotate(double (&a)[3][3], double (&v)[3][3]) {
    constexpr int R = 3 - P - Q;
    const double apq = a[P][Q];
    if (apq == 0.0) return;
    const double theta = (a[Q][Q] - a[P][P]) / (2.0 * apq);
    const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
    const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
    a[P][P] -= t * apq;
    a[Q][Q] += t * apq;
    a[P][Q] = 0.0;
    // a[R][P], a[R][Q] live in the upper triangle at (min, max)
    double& arp = a[R < P ? R : P][R < P ? P : R];
    double& arq = a[R < Q ? R : Q][R < Q ? Q : R];
    const double rp = arp, rq = arq;
    arp = c * rp - s * rq;
    arq = s * rp + c * rq;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double vp = v[k][P], vq = v[k][Q];
        v[k][P] = c * vp - s * vq;
        v[k][Q] = s * vp + c * vq;
    }
}

__global__ void __launch_bounds__(kT)
nrm_fit_kernel(const float* __restrict__ pts, const int32_t* __restrict__ ids, int N, int K, float* __restrict__ normals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int32_t* __restrict__ nb = ids + (int64_t)i * K;
    double mx = 0.0, my = 0.0, mz = 0.0;
    for (int s = 0; s < K; ++s) { const int j = nb[s]; mx += pts[j * 3 + 0]; my += pts[j * 3 + 1]; mz += pts[j * 3 + 2]; }
    mx /= K; my /= K; mz /= K;
    double a[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    for (int s = 0; s < K; ++s) {
        const int j = nb[s];
        const double dx = pts[j * 3 + 0] - mx, dy = pts[j * 3 + 1] - my, dz = pts[j * 3 + 2] - mz;
        a[0][0] += dx * dx; a[0][1] += dx * dy; a[0][2] += dx * dz;
        a[1][1] += dy * dy; a[1][2] += dy * dz; a[2][2] += dz * dz;
    }
    double v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int sweep = 0; sweep < 10; ++sweep) {
        jacobi_rotate<0, 1>(a, v);
        jacobi_rotate<0, 2>(a, v);
        jacobi_rotate<1, 2>(a, v);
    }
    const double e0 = a[0][0], e1 = a[1][1], e2 = a[2][2];
    const int m = (e0 <= e1 && e0 <= e2) ? 0 : (e1 <= e2 ? 1 : 2);
    const double l0 = m == 0 ? e0 : (m == 1 ? e1 : e2);
    const double r0 = m == 0 ? e1 : e0, r1 = m == 2 ? e1 : e2;          // the other two
    const double l1 = fmin(r0, r1), l2 = fmax(r0, r1);
    float nx = 0.f, ny = 0.f, nz = 0.f;
    if (l2 > 0.0 && l1 - l0 > 1e-9 * l2) {
        const double x = m == 0 ? v[0][0] : (m == 1 ? v[0][1] : v[0][2]);
        const double y = m == 0 ? v[1][0] : (m == 1 ? v[1][1] : v[1][2]);
        const double z = m == 0 ? v[2][0] : (m == 1 ? v[2][1] : v[2][2]);
        const double inv = 1.0 / sqrt(x * x + y * y + z * z);
        nx = (float)(x * inv); ny = (float)(y * inv); nz = (float)(z * inv);
        // pre-sign: the component of largest magnitude (lowest axis on ties) is positive
        float big = nx;
        if (fabsf(ny) > fabsf(big)) big = ny;
        if (fabsf(nz) > fabsf(big)) big = nz;
        if (big < 0.f) { nx = -nx; ny = -ny; nz = -nz; }
    }
    normals[i * 3 + 0] = nx; normals[i * 3 + 1] = ny; normals[i * 3 + 2] = nz;
}

__device__ __forceinline__ bool nonzero3(const float* __restrict__ n, int i) {
    return n[i * 3 + 0] != 0.f || n[i * 3 + 1] != 0.f || n[i * 3 + 2] != 0.f;
}

// n_i . n_j in float64, x then y then z, every operation rounded (the products of two floats are exact)
__device__ __forceinline__ double dot_rn(const float* __restrict__ n, int i, int j) {
    return __dadd_rn(__dadd_rn(__dmul_rn((double)n[i * 3 + 0], (double)n[j * 3 + 0]),
                               __dmul_rn((double)n[i * 3 + 1], (double)n[j * 3 + 1])),
                     __dmul_rn((double)n[i * 3 + 2], (double)n[j * 3 + 2]));
}

__global__ void __launch_bounds__(kT)
nrm_viewpoint_kernel(const float* __restrict__ pts, const float* __restrict__ nin, int N, double vx, double vy, double vz,
                     float* __restrict__ nout, unsigned long long* __restrict__ ctr) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const double nx = nin[i * 3 + 0], ny = nin[i * 3 + 1], nz = nin[i * 3 + 2];
    const double d = __dadd_rn(__dadd_rn(__dmul_rn(nx, vx - (double)pts[i * 3 + 0]), __dmul_rn(ny, vy - (double)pts[i * 3 + 1])),
                               __dmul_rn(nz, vz - (double)pts[i * 3 + 2]));
    const bool flip = d < 0.0;
    const float s = flip ? -1.f : 1.f;
    nout[i * 3 + 0] = s * nin[i * 3 + 0]; nout[i * 3 + 1] = s * nin[i * 3 + 1]; nout[i * 3 + 2] = s * nin[i * 3 + 2];
    if (flip) atomicAdd(&ctr[3], 1ull);
    if (!nonzero3(nin, i)) atomicAdd(&ctr[4], 1ull);
}

// entry e = (point i, slot s): the undirected edge {i, ids[e]} as (min << 32 | max) and its cost's bits; kNoEdge for a
// self loop or an end without a normal
__global__ void __launch_bounds__(kT)
nrm_edge_kernel(const float* __restrict__ normals, const int32_t* __restrict__ ids, int N, int K,
                unsigned long long* __restrict__ mm, unsigned long long* __restrict__ cost) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)N * K) return;
    const int i = (int)(e / K), j = ids[e];
    unsigned long long m = kNoEdge, c = kNoEdge;
    if (j != i && nonzero3(normals, i) && nonzero3(normals, j)) {
        const unsigned lo = (unsigned)min(i, j), hi = (unsigned)max(i, j);
        m = ((unsigned long long)lo << 32) | hi;
        c = (unsigned long long)__double_as_longlong(fmax(__dsub_rn(1.0, fabs(dot_rn(normals, i, j))), 0.0));
    }
    mm[e] = m; cost[e] = c;
}

__global__ void __launch_bounds__(kT) nrm_init_kernel(int N, int32_t* __restrict__ comp, int32_t* __restrict__ fe) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v < N) { comp[v] = v; fe[v] = -1; }
}

__global__ void __launch_bounds__(kT)
nrm_findmin_kernel(const unsigned long long* __restrict__ mm, int64_t M, const int32_t* __restrict__ comp, int* __restrict__ best) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= M) return;
    const unsigned long long m = mm[r];
    if (m == kNoEdge) return;
    const int cu = comp[(int)(m >> 32)], cv = comp[(int)(m & 0xffffffffu)];
    if (cu == cv) return;
    atomicMin(&best[cu], (int)r);
    atomicMin(&best[cv], (int)r);
}

// link = comp after this round's hooks (comp itself is read by every thread and stays as it is)
__global__ void __launch_bounds__(kT)
nrm_hook_kernel(const unsigned long long* __restrict__ mm, int N, const int32_t* __restrict__ comp, const int* __restrict__ best,
                int32_t* __restrict__ link, int32_t* __restrict__ fe, unsigned long long* __restrict__ ctr) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= N) return;
    const int c = comp[v];
    link[v] = c;
    if (c != v) return;
    const int r = best[v];
    if (r == kNoRank) return;
    const unsigned long long m = mm[r];
    const int cu = comp[(int)(m >> 32)], cv = comp[(int)(m & 0xffffffffu)];
    const int other = cu == v ? cv : cu;
    if (best[other] == r && v < other) return;      // both chose this edge: the lower id stays root
    link[v] = other;
    fe[v] = r;
    atomicAdd(&ctr[0], 1ull);
}

__global__ void __launch_bounds__(kT) nrm_jump_kernel(int N, int32_t* comp) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= N) return;
    const int p = comp[v], g = comp[p];
    if (g != p) comp[v] = g;
}

__global__ void __launch_bounds__(kT) nrm_flat_kernel(int N, const int32_t* __restrict__ comp, unsigned long long* __restrict__ ctr) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= N) return;
    const int p = comp[v];
    if (comp[p] != p) atomicAdd(&ctr[1], 1ull);
}

// per component the point of largest z, lowest id on ties: atomicMax of (ordered z bits, ~id)
__global__ void __launch_bounds__(kT)
nrm_rootkey_kernel(const float* __restrict__ pts, const float* __restrict__ normals, int N, const int32_t* __restrict__ comp,
                   unsigned long long* __restrict__ rootkey) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= N || !nonzero3(normals, v)) return;
    const unsigned b = __float_as_uint(pts[v * 3 + 2] + 0.0f);          // + 0: -0 and +0 are the same height
    const unsigned z = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
    atomicMax(&rootkey[comp[v]], ((unsigned long long)z << 32) | (0xffffffffu - (unsigned)v));
}

// state[v] = (parent << 1) | flip, -1 = not reached.  A root is its own parent and points up: z > 0, else y, else x.
__global__ void __launch_bounds__(kT)
nrm_root_kernel(const float* __restrict__ normals, int N, const int32_t* __restrict__ comp,
                const unsigned long long* __restrict__ rootkey, int32_t* __restrict__ state, unsigned long long* __restrict__ ctr) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= N || comp[v] != v || !nonzero3(normals, v)) return;
    const int root = (int)(0xffffffffu - (unsigned)(rootkey[v] & 0xffffffffu));
    const float x = normals[root * 3 + 0], y = normals[root * 3 + 1], z = normals[root * 3 + 2];
    const float lead = z != 0.f ? z : (y != 0.f ? y : x);
    state[root] = (root << 1) | (lead < 0.f ? 1 : 0);
    atomicAdd(&ctr[2], 1ull);
}

__global__ void __launch_bounds__(kT)
nrm_sweep_kernel(const unsigned long long* __restrict__ mm, const int32_t* __restrict__ fe, const float* __restrict__ normals, int N,
                 volatile int32_t* state, unsigned long long* __restrict__ ctr) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= N) return;
    const int r = fe[c];
    if (r < 0) return;
    const unsigned long long m = mm[r];
    const int u = (int)(m >> 32), v = (int)(m & 0xffffffffu);
    const int su = state[u], sv = state[v];
    if ((su >= 0) == (sv >= 0)) return;
    const int parent = su >= 0 ? u : v, child = su >= 0 ? v : u;
    const double d = dot_rn(normals, parent, child);
    const bool pflip = ((su >= 0 ? su : sv) & 1) != 0;
    state[child] = (parent << 1) | ((pflip ? -d : d) < 0.0 ? 1 : 0);     // d == 0: the child keeps its sign
    atomicAdd(&ctr[5], 1ull);
}

__global__ void __launch_bounds__(kT)
nrm_apply_kernel(const float* __restrict__ nin, int N, const int32_t* __restrict__ state, float* __restrict__ nout,
                 int32_t* __restrict__ parent_out, unsigned long long* __restrict__ ctr) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= N) return;
    const bool valid = nonzero3(nin, v);
    const int s = state[v];
    if (valid && s < 0) { atomicAdd(&ctr[1], 1ull); return; }
    const bool flip = valid && (s & 1);
    const float sg = flip ? -1.f : 1.f;
    nout[v * 3 + 0] = sg * nin[v * 3 + 0]; nout[v * 3 + 1] = sg * nin[v * 3 + 1]; nout[v * 3 + 2] = sg * nin[v * 3 + 2];
    if (parent_out) parent_out[v] = valid ? (s >> 1) : -1;
    if (flip) atomicAdd(&ctr[3], 1ull);
    if (!valid) atomicAdd(&ctr[4], 1ull);
}

int ceil_log2(int64_t n) { int l = 0; while (((int64_t)1 << l) < n) ++l; return l; }

void check_inputs(Workspace& ws, const float* pts, const float* normals, const int32_t* ids, int64_t N, int K, cudaStream_t st) {
    unsigned* flags = ws.get<unsigned>(2);
    P2S_CUDA(cudaMemsetAsync(flags, 0, 2 * sizeof(unsigned), st));
    const int64_t n = std::max<int64_t>(3 * N, ids ? N * K : 0);
    P2S_LAUNCH(nrm_check_kernel, grid1d(n, kT), kT, 0, st, pts, normals, 3 * N, ids, N * K, (int)N, flags);
    const std::vector<unsigned> h = read_back(flags, 2, st);
    P2S_CHECK(h[0] == 0, "non-finite point coordinate or normal");
    P2S_CHECK(h[1] == 0, "neighbour id outside [0, N)");
}

void check_sizes(int64_t N, int K) {
    P2S_CHECK(K >= 3 && K <= kMaxK, "K must be in [3, 64]");
    P2S_CHECK(N > K, "point normals need N > K");
    P2S_CHECK(N < (1 << 30) && N * K < kNoRank, "cloud too large");
}

// ctr: [0] hooks, [1] internal errors, [2] components, [3] flipped, [4] points without a normal, [5] points reached by sweeps
void orient_propagate(Workspace& ws, const float* pts, const float* nin, const int32_t* ids, int64_t N, int K, float* nout,
                      int32_t* parent_out, unsigned long long* ctr, p2s_normals_stats* stats, cudaStream_t st) {
    const int n = (int)N;
    const int64_t M = N * K;
    unsigned long long* mm = ws.get<unsigned long long>(M);
    unsigned long long* cost = ws.get<unsigned long long>(M);
    unsigned long long* mm_s = ws.get<unsigned long long>(M);
    unsigned long long* cost_s = ws.get<unsigned long long>(M);
    int32_t* comp = ws.get<int32_t>(N);
    int32_t* link = ws.get<int32_t>(N);
    int32_t* fe = ws.get<int32_t>(N);
    int* best = ws.get<int>(N);
    int32_t* state = ws.get<int32_t>(N);
    unsigned long long* rootkey = ws.get<unsigned long long>(N);
    P2S_LAUNCH(nrm_edge_kernel, grid1d(M, kT), kT, 0, st, nin, ids, n, K, mm, cost);
    // total order (cost, min, max): stable LSD passes, ends first
    cub_run(ws, 8, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, mm, mm_s, cost, cost_s, M, 0, 64, st); });
    cub_run(ws, 8, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, cost_s, cost, mm_s, mm, M, 0, 64, st); });
    P2S_LAUNCH(nrm_init_kernel, grid1d(N, kT), kT, 0, st, n, comp, fe);
    const int jumps = ceil_log2(N) + 1, max_rounds = ceil_log2(N) + 1;
    unsigned long long hooks = 0;
    int rounds = 0;
    for (;; ++rounds) {
        P2S_CUDA(cudaMemsetAsync(best, 0x7f, (size_t)N * sizeof(int), st));
        P2S_LAUNCH(nrm_findmin_kernel, grid1d(M, kT), kT, 0, st, mm, M, comp, best);
        P2S_LAUNCH(nrm_hook_kernel, grid1d(N, kT), kT, 0, st, mm, n, comp, best, link, fe, ctr);
        std::swap(comp, link);
        for (int j = 0; j < jumps; ++j) P2S_LAUNCH(nrm_jump_kernel, grid1d(N, kT), kT, 0, st, n, comp);
        P2S_LAUNCH(nrm_flat_kernel, grid1d(N, kT), kT, 0, st, n, comp, ctr);
        const std::vector<unsigned long long> h = read_back(ctr, 2, st);
        P2S_CHECK(h[1] == 0, "normal orientation: component labels did not flatten");
        if (h[0] == hooks) break;
        hooks = h[0];
        P2S_CHECK(rounds < max_rounds, "normal orientation: more Boruvka rounds than ceil(log2 N) + 1");
    }
    P2S_CUDA(cudaMemsetAsync(rootkey, 0, (size_t)N * sizeof(unsigned long long), st));
    P2S_CUDA(cudaMemsetAsync(state, 0xff, (size_t)N * sizeof(int32_t), st));
    P2S_LAUNCH(nrm_rootkey_kernel, grid1d(N, kT), kT, 0, st, pts, nin, n, comp, rootkey);
    P2S_LAUNCH(nrm_root_kernel, grid1d(N, kT), kT, 0, st, nin, n, comp, rootkey, state, ctr);
    unsigned long long reached = 0;
    int64_t sweeps = 0;
    for (;;) {
        for (int s = 0; s < kSweepBatch; ++s) P2S_LAUNCH(nrm_sweep_kernel, grid1d(N, kT), kT, 0, st, mm, fe, nin, n, state, ctr);
        sweeps += kSweepBatch;
        const unsigned long long now = read_back(ctr + 5, 1, st)[0];
        if (now == reached) break;
        reached = now;
        P2S_CHECK(sweeps <= N + kSweepBatch, "normal orientation: more sweeps than points");
    }
    P2S_LAUNCH(nrm_apply_kernel, grid1d(N, kT), kT, 0, st, nin, n, state, nout, parent_out, ctr);
    const std::vector<unsigned long long> h = read_back(ctr, 6, st);
    P2S_CHECK(h[1] == 0, "normal orientation: the forest does not reach every point");
    if (stats) {
        stats->components = (int64_t)h[2]; stats->flipped = (int64_t)h[3]; stats->degenerate = (int64_t)h[4];
        stats->rounds = rounds; stats->sweeps = (int32_t)sweeps;
    }
}

void orient_viewpoint(const float* pts, const float* nin, int64_t N, const double* vp, float* nout, unsigned long long* ctr,
                      p2s_normals_stats* stats, cudaStream_t st) {
    P2S_LAUNCH(nrm_viewpoint_kernel, grid1d(N, kT), kT, 0, st, pts, nin, (int)N, vp[0], vp[1], vp[2], nout, ctr);
    const std::vector<unsigned long long> h = read_back(ctr, 6, st);
    if (stats) { stats->flipped = (int64_t)h[3]; stats->degenerate = (int64_t)h[4]; }
}

unsigned long long* counters(Workspace& ws, cudaStream_t st) {
    unsigned long long* ctr = ws.get<unsigned long long>(6);
    P2S_CUDA(cudaMemsetAsync(ctr, 0, 6 * sizeof(unsigned long long), st));
    return ctr;
}

// CUDA-event stage times for the stats; no events without stats
struct StageEvents {
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    bool on;
    cudaStream_t st;
    StageEvents(bool enabled, cudaStream_t s) : on(enabled), st(s) {
        if (on) for (auto& e : ev) P2S_CUDA(cudaEventCreate(&e));
    }
    ~StageEvents() { for (auto& e : ev) if (e) cudaEventDestroy(e); }
    void mark(int i) { if (on) P2S_CUDA(cudaEventRecord(ev[i], st)); }
    void read(float* ms) {
        if (!on) return;
        P2S_CUDA(cudaEventSynchronize(ev[3]));
        for (int i = 0; i < 3; ++i) P2S_CUDA(cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]));
    }
};

}  // namespace

void point_normals(const float* pts, int64_t N, int K, int mode, const double* viewpoint, float* normals_out,
                   int32_t* nbr_ids_out, p2s_normals_stats* stats, cudaStream_t st) {
    check_sizes(N, K);
    P2S_CHECK(mode == P2S_NORMALS_PROPAGATE || mode == P2S_NORMALS_VIEWPOINT, "unknown orientation mode");
    P2S_CHECK(mode != P2S_NORMALS_VIEWPOINT || viewpoint, "viewpoint mode needs a viewpoint");
    if (viewpoint) P2S_CHECK(std::isfinite(viewpoint[0]) && std::isfinite(viewpoint[1]) && std::isfinite(viewpoint[2]), "non-finite viewpoint");
    static thread_local std::vector<Workspace> t_ws;
    Workspace& ws = for_device(t_ws).begin(st);
    check_inputs(ws, pts, nullptr, nullptr, N, K, st);
    if (stats) *stats = p2s_normals_stats{};
    StageEvents ev(stats != nullptr, st);
    int32_t* ids = nbr_ids_out ? nbr_ids_out : ws.get<int32_t>(N * K);
    float* fit = ws.get<float>(3 * N);
    unsigned long long* ctr = counters(ws, st);
    ev.mark(0);
    const CloudIndex* ix = cloud_index_build(pts, N, st);
    P2S_LAUNCH(nrm_knn_kernel, grid1d(N, 128), 128, 0, st, *ix, (int)N, K, ids);
    ev.mark(1);
    P2S_LAUNCH(nrm_fit_kernel, grid1d(N, kT), kT, 0, st, pts, ids, (int)N, K, fit);
    ev.mark(2);
    if (mode == P2S_NORMALS_VIEWPOINT) orient_viewpoint(pts, fit, N, viewpoint, normals_out, ctr, stats, st);
    else orient_propagate(ws, pts, fit, ids, N, K, normals_out, nullptr, ctr, stats, st);
    ev.mark(3);
    if (stats) ev.read(stats->stage_ms);
}

void orient_normals(const float* pts, const float* normals_in, const int32_t* nbr_ids, int64_t N, int K, float* normals_out,
                    int32_t* parent_out, p2s_normals_stats* stats, cudaStream_t st) {
    check_sizes(N, K);
    static thread_local std::vector<Workspace> t_ws;
    Workspace& ws = for_device(t_ws).begin(st);
    check_inputs(ws, pts, normals_in, nbr_ids, N, K, st);
    if (stats) *stats = p2s_normals_stats{};
    StageEvents ev(stats != nullptr, st);
    unsigned long long* ctr = counters(ws, st);
    ev.mark(0); ev.mark(1); ev.mark(2);
    orient_propagate(ws, pts, normals_in, nbr_ids, N, K, normals_out, parent_out, ctr, stats, st);
    ev.mark(3);
    if (stats) ev.read(stats->stage_ms);
}

}  // namespace p2s
