// K11: simulated time-of-flight range scans -- the input point clouds (04_pts) that make_dataset.py:sample_blensor makes
// with BlenSor (make_dataset.py:242-380, scanner settings blensor_script_template.py:80-96), merged in model space like
// _pcd_files_to_pts (make_dataset.py:147-239).  Scanner model (include/p2s_b200.h): origin, looking along +y, 176 x 144
// rays through the pixel centres of a uniform image-plane grid, the nearest hit within max_distance, Gaussian range
// noise.  Exhaustive and exact, no BVH:
//   1. scan_check_kernel: every face index in [0, V) (else an error, read back) and the vertex bounding box
//   2. scan_cull_kernel: every (scan, pixel) ray, moved into model space with R^T, against the bounding box (slab test,
//      padded so that it never rejects a ray that hits a face); CUB select compacts the survivors in (scan, pixel) order
//   3. scan_cast_kernel: one surviving ray per thread, tiles of faces staged in shared memory, faces in ascending
//      order.  Watertight ray-triangle test (Woop, Benthin & Wald 2013) in float64 with explicitly rounded products,
//      so that the edge function of an edge shared by two faces is the same number (negated) in both: a ray through a
//      shared edge or vertex cannot pass between them.  Nearest t in (0, max_distance], strict <: lowest face on ties.
//      Zero-area faces (float64 cross product of the edges exactly 0) are never hit.
//   4. CUB select compacts the hits in (scan, pixel) order; scan_emit_kernel writes the noisy and noise-free points,
//      the faces and the hits per scan (integer atomics only).
// Every ray and every noise value is a function of (pose, pixel) and (seed, first_scan + scan, pixel) alone, so the
// output is bitwise identical across runs and for any split of the scans across calls.
#include "common.cuh"
#include <cmath>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

namespace p2s {

namespace {

constexpr int kThreads = 128;   // rays per CTA
constexpr int kTile = 128;      // faces per shared-memory tile (one staged per thread)

struct ScanParams {
    int res_x, res_y, npix, first_scan;
    double tan_w, tan_h;        // tan(lens angle / 2)
    double tmax;                // max_distance
    double mu, sigma;           // range noise
    uint64_t seed;
    double lo[3], hi[3];        // padded bounding box (cull only)
};

// model-space ray of pixel `pix` of the scan with pose p (R row-major, loc).  Every product and sum is rounded
// explicitly, in the order oracle/scan_oracle.py uses, so that the CPU restatement computes the same rays.
__device__ __forceinline__ void scan_ray(const double* __restrict__ p, int pix, const ScanParams& P, double o[3],
                                         double d[3]) {
    const int row = pix / P.res_x, col = pix - row * P.res_x;
    const double u = __dmul_rn(__dsub_rn(__ddiv_rn(__dmul_rn(2.0, (double)col + 0.5), (double)P.res_x), 1.0), P.tan_w);
    const double v = __dmul_rn(__dsub_rn(1.0, __ddiv_rn(__dmul_rn(2.0, (double)row + 0.5), (double)P.res_y)), P.tan_h);
    const double n = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(u, u), 1.0), __dmul_rn(v, v)));
    // the wide image axis (columns, u) is z, the rows (v) run along x
    const double s0 = __ddiv_rn(v, n), s1 = __ddiv_rn(1.0, n), s2 = __ddiv_rn(u, n);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        // d = R^T s, o = -R^T loc
        d[i] = __dadd_rn(__dadd_rn(__dmul_rn(p[i], s0), __dmul_rn(p[3 + i], s1)), __dmul_rn(p[6 + i], s2));
        o[i] = -__dadd_rn(__dadd_rn(__dmul_rn(p[i], p[9]), __dmul_rn(p[3 + i], p[10])), __dmul_rn(p[6 + i], p[11]));
    }
}

// float -> unsigned key that orders like the float (for atomicMin / atomicMax of the bounding box)
__device__ __forceinline__ unsigned float_key(float x) {
    const unsigned u = __float_as_uint(x);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ inline float key_float(unsigned k) {
    const unsigned u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    float x;
    memcpy(&x, &u, 4);
    return x;
}

// flags: [0] out-of-range face indices, [1..3] min key, [4..6] max key
__global__ void __launch_bounds__(256)
scan_check_kernel(const float* __restrict__ verts, int64_t V, const int32_t* __restrict__ faces, int64_t F,
                  unsigned* __restrict__ flags) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool bad = false;
    if (i < 3 * F) {
        const int32_t x = faces[i];
        bad = x < 0 || x >= V;
    }
    const unsigned nbad = __popc(__ballot_sync(0xffffffffu, bad));
    if ((threadIdx.x & 31) == 0 && nbad) atomicAdd(flags, nbad);
    if (i < V) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const unsigned key = float_key(verts[3 * i + k]);
            atomicMin(flags + 1 + k, key);
            atomicMax(flags + 4 + k, key);
        }
    }
}

__global__ void __launch_bounds__(256)
scan_cull_kernel(const double* __restrict__ poses, int64_t nrays, ScanParams P, uint8_t* __restrict__ flag) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nrays) return;
    const int s = (int)(r / P.npix), pix = (int)(r - (int64_t)s * P.npix);
    double o[3], d[3];
    scan_ray(poses + 12 * s, pix, P, o, d);
    double tn = 0.0, tf = P.tmax;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double inv = 1.0 / d[k];   // +-inf on an axis-parallel ray; fmin / fmax drop the NaN of 0 * inf
        double t0 = (P.lo[k] - o[k]) * inv, t1 = (P.hi[k] - o[k]) * inv;
        if (t0 > t1) { const double x = t0; t0 = t1; t1 = x; }
        tn = fmax(tn, t0);
        tf = fmin(tf, t1);
    }
    flag[r] = tn <= tf;
}

// component k of (x, y, z) without a dynamically indexed local array
template <class T>
__device__ __forceinline__ double pick(int k, T x, T y, T z) { return k == 0 ? x : (k == 1 ? y : z); }

__global__ void __launch_bounds__(kThreads)
scan_cast_kernel(const float* __restrict__ verts, const int32_t* __restrict__ faces, int64_t F,
                 const double* __restrict__ poses, ScanParams P, const int32_t* __restrict__ rays, int n,
                 double* __restrict__ t_out, int32_t* __restrict__ face_out, uint8_t* __restrict__ hit) {
    __shared__ float sv[9][kTile];
    __shared__ unsigned char szero[kTile];
    const int i = blockIdx.x * kThreads + threadIdx.x;
    int kx = 0, ky = 1, kz = 2;
    double Sx = 0.0, Sy = 0.0, Sz = 0.0, ox = 0.0, oy = 0.0, oz = 0.0;
    if (i < n) {
        const int r = rays[i];
        const int s = r / P.npix;
        double o[3], d[3];
        scan_ray(poses + 12 * s, r - s * P.npix, P, o, d);
        // shear frame: kz = the largest |d| component (first on ties), (kx, ky) swapped when d[kz] < 0 to keep the
        // winding of the projected triangles
        kz = fabs(d[1]) > fabs(d[0]) ? 1 : 0;
        if (fabs(d[2]) > fabs(pick(kz, d[0], d[1], d[2]))) kz = 2;
        kx = kz == 2 ? 0 : kz + 1;
        ky = kx == 2 ? 0 : kx + 1;
        const double dz = pick(kz, d[0], d[1], d[2]);
        if (dz < 0.0) { const int x = kx; kx = ky; ky = x; }
        Sx = __ddiv_rn(pick(kx, d[0], d[1], d[2]), dz);
        Sy = __ddiv_rn(pick(ky, d[0], d[1], d[2]), dz);
        Sz = __ddiv_rn(1.0, dz);
        ox = pick(kx, o[0], o[1], o[2]); oy = pick(ky, o[0], o[1], o[2]); oz = pick(kz, o[0], o[1], o[2]);
    }
    double best = INFINITY;
    int32_t best_face = -1;
    for (int64_t t0 = 0; t0 < F; t0 += kTile) {
        const int cnt = (int)min((int64_t)kTile, F - t0);
        __syncthreads();
        if (threadIdx.x < cnt) {
            const int64_t f = t0 + threadIdx.x;
            float c[9];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const int64_t vi = faces[3 * f + k];
                c[3 * k] = verts[3 * vi]; c[3 * k + 1] = verts[3 * vi + 1]; c[3 * k + 2] = verts[3 * vi + 2];
            }
#pragma unroll
            for (int k = 0; k < 9; ++k) sv[k][threadIdx.x] = c[k];
            // zero area: the float64 cross product of the edges is exactly 0 (as in meshsdf.cu)
            const double ux = (double)c[3] - c[0], uy = (double)c[4] - c[1], uz = (double)c[5] - c[2];
            const double wx = (double)c[6] - c[0], wy = (double)c[7] - c[1], wz = (double)c[8] - c[2];
            const double nx = __dsub_rn(__dmul_rn(uy, wz), __dmul_rn(uz, wy));
            const double ny = __dsub_rn(__dmul_rn(uz, wx), __dmul_rn(ux, wz));
            const double nz = __dsub_rn(__dmul_rn(ux, wy), __dmul_rn(uy, wx));
            szero[threadIdx.x] = nx == 0.0 && ny == 0.0 && nz == 0.0;
        }
        __syncthreads();
        if (i >= n) continue;
        for (int k = 0; k < cnt; ++k) {
            if (szero[k]) continue;
            // vertices relative to the origin in the permuted frame, then sheared onto the ray (z along the ray)
            const double az = __dsub_rn(pick(kz, sv[0][k], sv[1][k], sv[2][k]), oz);
            const double bz = __dsub_rn(pick(kz, sv[3][k], sv[4][k], sv[5][k]), oz);
            const double cz = __dsub_rn(pick(kz, sv[6][k], sv[7][k], sv[8][k]), oz);
            const double Ax = __dsub_rn(__dsub_rn(pick(kx, sv[0][k], sv[1][k], sv[2][k]), ox), __dmul_rn(Sx, az));
            const double Ay = __dsub_rn(__dsub_rn(pick(ky, sv[0][k], sv[1][k], sv[2][k]), oy), __dmul_rn(Sy, az));
            const double Bx = __dsub_rn(__dsub_rn(pick(kx, sv[3][k], sv[4][k], sv[5][k]), ox), __dmul_rn(Sx, bz));
            const double By = __dsub_rn(__dsub_rn(pick(ky, sv[3][k], sv[4][k], sv[5][k]), oy), __dmul_rn(Sy, bz));
            const double Cx = __dsub_rn(__dsub_rn(pick(kx, sv[6][k], sv[7][k], sv[8][k]), ox), __dmul_rn(Sx, cz));
            const double Cy = __dsub_rn(__dsub_rn(pick(ky, sv[6][k], sv[7][k], sv[8][k]), oy), __dmul_rn(Sy, cz));
            // scaled barycentric coordinates (edge functions); on a shared edge the two faces see -U and U exactly
            const double U = __dsub_rn(__dmul_rn(Cx, By), __dmul_rn(Cy, Bx));
            const double V = __dsub_rn(__dmul_rn(Ax, Cy), __dmul_rn(Ay, Cx));
            const double W = __dsub_rn(__dmul_rn(Bx, Ay), __dmul_rn(By, Ax));
            if ((U < 0.0 || V < 0.0 || W < 0.0) && (U > 0.0 || V > 0.0 || W > 0.0)) continue;   // no back-face culling
            const double det = __dadd_rn(__dadd_rn(U, V), W);
            if (det == 0.0) continue;
            const double T = __dadd_rn(__dadd_rn(__dmul_rn(U, __dmul_rn(Sz, az)), __dmul_rn(V, __dmul_rn(Sz, bz))),
                                       __dmul_rn(W, __dmul_rn(Sz, cz)));
            const double t = __ddiv_rn(T, det);
            if (t > 0.0 && t <= P.tmax && t < best) { best = t; best_face = (int32_t)(t0 + k); }
        }
    }
    if (i < n) {
        t_out[i] = best;
        face_out[i] = best_face;
        hit[i] = best_face >= 0;
    }
}

// grid over all H hits; writes the first min(H, cap)
__global__ void __launch_bounds__(256)
scan_emit_kernel(const double* __restrict__ poses, ScanParams P, const int32_t* __restrict__ rays,
                 const int32_t* __restrict__ hitsel, int H, int64_t cap, const double* __restrict__ t_ray,
                 const int32_t* __restrict__ face_ray, float* __restrict__ noisy, float* __restrict__ clean,
                 int32_t* __restrict__ face_ids, int32_t* __restrict__ hits_per_scan) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= H) return;
    const int ri = hitsel[j];
    const int r = rays[ri];
    const int s = r / P.npix, pix = r - s * P.npix;
    if (hits_per_scan) atomicAdd(hits_per_scan + s, 1);
    if (j >= cap) return;
    double o[3], d[3];
    scan_ray(poses + 12 * s, pix, P, o, d);
    const double t = t_ray[ri];
    // Box-Muller on one Philox block keyed by (seed, scan, pixel): u1 in (0, 1), u2 in [0, 1)
    uint32_t b[4];
    philox4x32_10((uint32_t)P.seed, (uint32_t)(P.seed >> 32), (uint32_t)(P.first_scan + s), (uint32_t)pix, 0u,
                  0x2545f491u, b);
    const double u1 = ((double)b[0] + 0.5) * 2.3283064365386963e-10;
    const double u2 = (double)b[1] * 2.3283064365386963e-10;
    const double z = sqrt(-2.0 * log(u1)) * cospi(2.0 * u2);
    const double tn = t + P.mu + P.sigma * z;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        noisy[3 * (int64_t)j + k] = (float)(o[k] + d[k] * tn);
        if (clean) clean[3 * (int64_t)j + k] = (float)(o[k] + d[k] * t);
    }
    if (face_ids) face_ids[j] = face_ray[ri];
}

}  // namespace

void range_scan(const float* verts, int64_t V, const int32_t* faces, int64_t F, const double* poses, int64_t S,
                const p2s_scan_config& cfg, uint64_t seed, float* pts_noisy, float* pts_clean, int32_t* face_ids,
                int64_t cap, int32_t* hits_per_scan, int64_t* total_host, cudaStream_t st) {
    P2S_CHECK(V > 0 && F > 0, "empty mesh");
    P2S_CHECK(V <= INT32_MAX && F <= INT32_MAX / 3, "mesh too large for int32 indices");
    P2S_CHECK(S >= 0 && cap >= 0, "negative size");
    P2S_CHECK(cfg.res_x > 0 && cfg.res_y > 0, "scanner resolution must be positive");
    P2S_CHECK(cfg.lens_angle_w_deg > 0.f && cfg.lens_angle_w_deg < 180.f && cfg.lens_angle_h_deg > 0.f &&
                  cfg.lens_angle_h_deg < 180.f, "lens angles must lie in (0, 180) degrees");
    P2S_CHECK(cfg.max_distance > 0.f && std::isfinite(cfg.max_distance), "max_distance must be positive and finite");
    P2S_CHECK(cfg.noise_sigma >= 0.f && std::isfinite(cfg.noise_sigma) && std::isfinite(cfg.noise_mu),
              "noise_sigma must be >= 0 and finite, noise_mu finite");
    P2S_CHECK(cfg.first_scan >= 0, "first_scan must be >= 0");
    const int64_t npix = (int64_t)cfg.res_x * cfg.res_y;
    P2S_CHECK(npix <= INT32_MAX && S * npix <= INT32_MAX, "too many rays for one call (S * res_x * res_y >= 2^31)");
    static thread_local std::vector<Workspace> t_ws;
    Workspace& ws = for_device(t_ws).begin(st);
    unsigned* flags = ws.get<unsigned>(7);
    unsigned init[7] = {0u, ~0u, ~0u, ~0u, 0u, 0u, 0u};
    P2S_CUDA(cudaMemcpyAsync(flags, init, sizeof(init), cudaMemcpyHostToDevice, st));
    const int64_t nchk = std::max(3 * F, V);
    P2S_LAUNCH(scan_check_kernel, (unsigned)cdiv(nchk, 256), 256, 0, st, verts, V, faces, F, flags);
    const std::vector<unsigned> h = read_back(flags, 7, st);
    P2S_CHECK(h[0] == 0, "face index outside [0, V)");
    ScanParams P;
    P.res_x = cfg.res_x; P.res_y = cfg.res_y; P.npix = (int)npix; P.first_scan = cfg.first_scan;
    P.tan_w = std::tan((double)cfg.lens_angle_w_deg * (M_PI / 360.0));
    P.tan_h = std::tan((double)cfg.lens_angle_h_deg * (M_PI / 360.0));
    P.tmax = cfg.max_distance; P.mu = cfg.noise_mu; P.sigma = cfg.noise_sigma; P.seed = seed;
    double scale = 0.0;
    for (int k = 0; k < 3; ++k) {
        P.lo[k] = key_float(h[1 + k]);
        P.hi[k] = key_float(h[4 + k]);
        P2S_CHECK(std::isfinite(P.lo[k]) && std::isfinite(P.hi[k]), "non-finite vertex coordinate");
        scale = std::max(scale, std::max(std::fabs(P.lo[k]), std::fabs(P.hi[k])));
    }
    // padding far above the rounding of the slab test: the cull never drops a ray that reaches a face
    const double pad = 1e-6 * scale + 1e-30;
    for (int k = 0; k < 3; ++k) { P.lo[k] -= pad; P.hi[k] += pad; }
    if (hits_per_scan && S > 0) P2S_CUDA(cudaMemsetAsync(hits_per_scan, 0, (size_t)S * sizeof(int32_t), st));
    *total_host = 0;
    if (S == 0) return;
    const int nrays = (int)(S * npix);

    cub::CountingInputIterator<int32_t> counting(0);
    int* d_num = ws.get<int>(1);
    uint8_t* ray_flag = ws.get<uint8_t>(nrays);
    int32_t* rays = ws.get<int32_t>(nrays);
    P2S_LAUNCH(scan_cull_kernel, (unsigned)cdiv(nrays, 256), 256, 0, st, poses, (int64_t)nrays, P, ray_flag);
    cub_run(ws, 2, [&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, counting, ray_flag, rays, d_num, nrays, st); });
    const int n = read_back(d_num, 1, st)[0];
    if (n == 0) return;

    double* t_ray = ws.get<double>(n);
    int32_t* face_ray = ws.get<int32_t>(n);
    uint8_t* hit = ws.get<uint8_t>(n);
    int32_t* hitsel = ws.get<int32_t>(n);
    P2S_LAUNCH(scan_cast_kernel, (unsigned)cdiv(n, kThreads), kThreads, 0, st, verts, faces, F, poses, P, rays, n, t_ray,
               face_ray, hit);
    cub_run(ws, 2, [&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, counting, hit, hitsel, d_num, n, st); });
    const int H = read_back(d_num, 1, st)[0];
    *total_host = H;
    if (H == 0) return;
    P2S_CHECK(cap == 0 || pts_noisy, "null output with cap > 0");
    P2S_LAUNCH(scan_emit_kernel, (unsigned)cdiv(H, 256), 256, 0, st, poses, P, rays, hitsel, H, cap, t_ray, face_ray,
               pts_noisy, pts_clean, face_ids, hits_per_scan);
}

}  // namespace p2s
