// K10: ground-truth signed distances from query points to a triangle mesh -- the training targets that
// make_dataset.py:_get_and_save_query_pts writes to 05_query_dist (sdf.get_signed_distance, source/sdf.py:318-348, which
// calls trimesh.proximity.signed_distance; trimesh is absent here).  Exhaustive and exact, no BVH:
//   1. mesh_check_kernel: every face index in [0, V) (else an error, read back) and the largest |vertex coordinate|
//      (the scale of the fp32 error bound below)
//   2. meshsdf_slab_kernel: grid (query blocks, face slabs); every CTA stages tiles of its slab's triangles in shared
//      memory, one query per thread, faces in ascending order.  Per face:
//        - squared distance in fp32, in units of the query's power-of-two scale; every face whose fp32 value lies
//          within kRelTol / the eps(scale) bound of the running fp32 minimum is recomputed in float64 and the float64
//          minimum kept (strict <: lowest face on ties).  Degenerate and sliver faces (|n|^2 < 2^-10 * longest edge^4)
//          skip the fp32 value and always go to float64, and so do faces too small for fp32 at that scale.
//        - float64 solid angle (Van Oosterom & Strackee 1983) summed into the slab's winding-number partial; zero-area
//          faces contribute 0.
//      -> per (slab, query): float64 d^2, face, float64 winding partial.  Slab boundaries depend on F only.
//   3. meshsdf_finalize_kernel: slabs in ascending order (min d^2, strict <; winding sum) -> signed distance.
// No float atomics anywhere: results are bitwise identical across runs and for any split of the query array.
//
// The unsigned query (p2s_mesh_closest_point_dev: trimesh.proximity.closest_point for point_cloud.
// get_closest_distance_batched, source/base/point_cloud.py:195-218) is the same slab kernel compiled without the solid
// angles (meshsdf_slab_kernel<false>), so its distances and faces are the signed path's bit for bit; its finalize
// recomputes the closest point of the winning face in float64 (tri_dist2 with a point output) and rounds it once.
//
// Sign: inside iff the generalised winding number w (Jacobson et al. 2013) > 0.5, inside is positive like trimesh;
// |d| <= 1e-8 counts as on the surface and is positive (trimesh's tol.merge).  On a closed, consistently oriented mesh
// w is 1 inside and 0 outside.  On a mesh with holes or inconsistent orientation w is fractional and can disagree with
// trimesh's ray-parity test; the caller orients the mesh outward (points2surf_b200/sdf.py flips it when its signed
// volume is negative, the global part of trimesh's fix_normals).
#include "common.cuh"
#include <cmath>

namespace p2s {

namespace {

constexpr int kThreads = 128;      // queries per CTA
constexpr int kTile = 128;         // faces per shared-memory tile (one staged per thread)
constexpr int kMaxSlabs = 32;      // face slabs per query block
constexpr int64_t kChunk = 1 << 18;   // queries per launch pair (bounds the per-slab partials to 20 B * 32 * 2^18)

// fp32 error budget of the candidate test.  The fp32 squared distance of a well-shaped face (|n| >= 2^-5 * longest
// edge^2, so that the fp32 normal is accurate to ~2^5 u) differs from the float64 one by far less than
// 2^-10 * d^2 + 2 d eps + eps^2 with eps = 2^-12 * (|p|_inf + max |vertex coordinate|): the coordinate differences
// carry u * scale, the normal direction 2^5 u, and the rest is a handful of roundings.  The face with the exact minimum
// therefore always passes `d2f <= best32 + tol(best32)` (tol covers the error on both sides).
// The argument needs every fp32 value to be a normal number: |n|^2 ~ l^4 and h^2 ~ l^4 d^2 leave fp32's range for
// coordinates beyond ~2^31 or below ~2^-31.  So the fp32 pass runs in units of 2^e, the power of two with
// max(|p|_inf, max |vertex coordinate|) in [2^(e-1), 2^e) (e clamped to [-126, 126]): every operand is then at most 1
// in magnitude (4 beyond 2^126), no value
// overflows, and the arithmetic is the unit-scale one bit for bit (scaling by a power of two is exact).  A face whose
// fp32 |n|^2 falls below kMinNN in those units (an edge below ~2^-22 of the scale) goes to float64, so underflow never
// moves an fp32 value by more than 2^-50, far inside eps^2 >= 2^-26.
constexpr float kRelTol = 1.0f / 1024.0f;
constexpr float kEpsScale = 1.0f / 4096.0f;
constexpr float kMinNN = 0x1p-100f;

enum : unsigned char { kZeroArea = 1, kForce64 = 2 };

// squared distance from p to the segment [a, b] (a point when a == b); the closest point a + t (b - a) into cp when
// cp is not null
template <class T>
__device__ __forceinline__ T seg_dist2(T px, T py, T pz, T ax, T ay, T az, T bx, T by, T bz, T* cp = nullptr) {
    const T ux = bx - ax, uy = by - ay, uz = bz - az;
    const T wx = px - ax, wy = py - ay, wz = pz - az;
    const T uu = ux * ux + uy * uy + uz * uz;
    T t = uu > T(0) ? (ux * wx + uy * wy + uz * wz) / uu : T(0);
    t = t < T(0) ? T(0) : (t > T(1) ? T(1) : t);
    const T dx = wx - t * ux, dy = wy - t * uy, dz = wz - t * uz;
    if (cp) { cp[0] = ax + t * ux; cp[1] = ay + t * uy; cp[2] = az + t * uz; }
    return dx * dx + dy * dy + dz * dz;
}

// squared distance from p to the triangle (a, b, c): the plane distance when p projects inside the triangle, else the
// nearest edge.  A zero-area face is its three edges (a segment or a point).  When cp is not null, the point that gives
// this distance goes to cp: the projection onto the plane, or the closest point of the first nearest edge in the order
// ab, bc, ca.  With cp null the arithmetic is exactly the distance-only one.  |n|^2 goes to nn_out when it is not null.
template <class T>
__device__ __forceinline__ T tri_dist2(T px, T py, T pz, T ax, T ay, T az, T bx, T by, T bz, T cx, T cy, T cz,
                                       bool zero_area, T* cp = nullptr, T* nn_out = nullptr) {
    if (!zero_area) {
        const T abx = bx - ax, aby = by - ay, abz = bz - az;
        const T acx = cx - ax, acy = cy - ay, acz = cz - az;
        const T nx = aby * acz - abz * acy, ny = abz * acx - abx * acz, nz = abx * acy - aby * acx;
        const T nn = nx * nx + ny * ny + nz * nz;
        if (nn_out) *nn_out = nn;
        const T apx = px - ax, apy = py - ay, apz = pz - az;
        const T bpx = px - bx, bpy = py - by, bpz = pz - bz;
        const T cpx = px - cx, cpy = py - cy, cpz = pz - cz;
        const T bcx = cx - bx, bcy = cy - by, bcz = cz - bz;
        const T cax = ax - cx, cay = ay - cy, caz = az - cz;
        // p is on the inner side of edge (v, v') iff ((v' - v) x (p - v)) . n >= 0
        const T e0 = (aby * apz - abz * apy) * nx + (abz * apx - abx * apz) * ny + (abx * apy - aby * apx) * nz;
        const T e1 = (bcy * bpz - bcz * bpy) * nx + (bcz * bpx - bcx * bpz) * ny + (bcx * bpy - bcy * bpx) * nz;
        const T e2 = (cay * cpz - caz * cpy) * nx + (caz * cpx - cax * cpz) * ny + (cax * cpy - cay * cpx) * nz;
        if (nn > T(0) && e0 >= T(0) && e1 >= T(0) && e2 >= T(0)) {
            const T h = nx * apx + ny * apy + nz * apz;
            if (cp) {
                const T s = h / nn;
                cp[0] = px - s * nx; cp[1] = py - s * ny; cp[2] = pz - s * nz;
            }
            return h * h / nn;
        }
    }
    if (!cp) {
        T d = seg_dist2(px, py, pz, ax, ay, az, bx, by, bz);
        d = fmin(d, seg_dist2(px, py, pz, bx, by, bz, cx, cy, cz));
        return fmin(d, seg_dist2(px, py, pz, cx, cy, cz, ax, ay, az));
    }
    T e[3];
    T d = seg_dist2(px, py, pz, ax, ay, az, bx, by, bz, cp);
    const T d1 = seg_dist2(px, py, pz, bx, by, bz, cx, cy, cz, e);
    if (d1 < d) { d = d1; cp[0] = e[0]; cp[1] = e[1]; cp[2] = e[2]; }
    const T d2 = seg_dist2(px, py, pz, cx, cy, cz, ax, ay, az, e);
    if (d2 < d) { d = d2; cp[0] = e[0]; cp[1] = e[1]; cp[2] = e[2]; }
    return d;
}

// kZeroArea / kForce64 of the face with corners c = (a, b, c)
__device__ __forceinline__ unsigned char face_flags(const float* c) {
    // zero area: the float64 cross product of the edges is exactly 0 (no FMA contraction, so that the CPU restatement
    // makes the same decision)
    const double ux = (double)c[3] - c[0], uy = (double)c[4] - c[1], uz = (double)c[5] - c[2];
    const double wx = (double)c[6] - c[0], wy = (double)c[7] - c[1], wz = (double)c[8] - c[2];
    const double nx = __dsub_rn(__dmul_rn(uy, wz), __dmul_rn(uz, wy));
    const double ny = __dsub_rn(__dmul_rn(uz, wx), __dmul_rn(ux, wz));
    const double nz = __dsub_rn(__dmul_rn(ux, wy), __dmul_rn(uy, wx));
    const double nn = nx * nx + ny * ny + nz * nz;
    const double vx = (double)c[6] - c[3], vy = (double)c[7] - c[4], vz = (double)c[8] - c[5];
    const double l2 = fmax(ux * ux + uy * uy + uz * uz, fmax(wx * wx + wy * wy + wz * wz, vx * vx + vy * vy + vz * vz));
    const bool zero = nx == 0.0 && ny == 0.0 && nz == 0.0;
    return zero ? (kZeroArea | kForce64) : (nn < (1.0 / 1024.0) * l2 * l2 ? kForce64 : 0);
}

__device__ __forceinline__ void load_face(const float* __restrict__ verts, const int32_t* __restrict__ faces, int64_t f,
                                          float* c) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int64_t vi = faces[3 * f + k];
        c[3 * k] = verts[3 * vi]; c[3 * k + 1] = verts[3 * vi + 1]; c[3 * k + 2] = verts[3 * vi + 2];
    }
}

__global__ void __launch_bounds__(256)
mesh_check_kernel(const float* __restrict__ verts, int64_t V, const int32_t* __restrict__ faces, int64_t F,
                  unsigned* __restrict__ flags) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool bad = false;
    unsigned m = 0;
    if (i < 3 * F) {
        const int32_t x = faces[i];
        bad = x < 0 || x >= V;
    }
    if (i < 3 * V) m = __float_as_uint(fabsf(verts[i]));   // non-negative floats order like their bits; NaN sorts last
    const unsigned nbad = __popc(__ballot_sync(0xffffffffu, bad));
    m = __reduce_max_sync(0xffffffffu, m);
    if ((threadIdx.x & 31) == 0) {
        if (nbad) atomicAdd(flags, nbad);
        atomicMax(flags + 1, m);
    }
}

// grid (ceil(Q / kThreads), slabs): slab s covers faces [s * slab_len, min(F, (s + 1) * slab_len)).
// kWinding = false is the unsigned query: the same distances and faces, no solid angles, part_wind unused.
template <bool kWinding>
__global__ void __launch_bounds__(kThreads)
meshsdf_slab_kernel(const float* __restrict__ verts, const int32_t* __restrict__ faces, int64_t F, int64_t slab_len,
                    const float* __restrict__ query, int64_t Q, float vmax, double* __restrict__ part_d2,
                    int32_t* __restrict__ part_face, double* __restrict__ part_wind) {
    __shared__ float sv[9][kTile];
    __shared__ unsigned char sflag[kTile];
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    float px = 0.f, py = 0.f, pz = 0.f;
    if (i < Q) { px = query[3 * i]; py = query[3 * i + 1]; pz = query[3 * i + 2]; }
    const double qx = px, qy = py, qz = pz;
    // the fp32 pass in units of 2^e (above): s = 2^-e, e clamped so that s is a normal number
    const float pmax = fmaxf(fabsf(px), fmaxf(fabsf(py), fabsf(pz)));
    int e = 0;
    if (isfinite(pmax)) frexpf(fmaxf(pmax, vmax), &e);
    e = max(-126, min(126, e));
    const float s = __int_as_float((127 - e) << 23);
    const double s2 = (double)s * s;
    const float spx = px * s, spy = py * s, spz = pz * s;
    const float eps = kEpsScale * (pmax * s + vmax * s);
    float best32 = INFINITY, thr = INFINITY;
    double best64 = INFINITY, wind = 0.0;
    int32_t best_face = -1;
    const int64_t f0 = (int64_t)blockIdx.y * slab_len, f1 = min(F, f0 + slab_len);
    for (int64_t t = f0; t < f1; t += kTile) {
        const int cnt = (int)min((int64_t)kTile, f1 - t);
        __syncthreads();
        if (threadIdx.x < cnt) {
            float c[9];
            load_face(verts, faces, t + threadIdx.x, c);
#pragma unroll
            for (int k = 0; k < 9; ++k) sv[k][threadIdx.x] = c[k];
            sflag[threadIdx.x] = face_flags(c);
        }
        __syncthreads();
        if (i >= Q) continue;
        for (int k = 0; k < cnt; ++k) {
            const unsigned char fl = sflag[k];
            const float ax = sv[0][k], ay = sv[1][k], az = sv[2][k];
            const float bx = sv[3][k], by = sv[4][k], bz = sv[5][k];
            const float cx = sv[6][k], cy = sv[7][k], cz = sv[8][k];
            const bool zero = fl & kZeroArea;
            float d2f = 0.f;
            bool force = fl & kForce64;
            if (!force) {
                float nn;
                d2f = tri_dist2<float>(spx, spy, spz, ax * s, ay * s, az * s, bx * s, by * s, bz * s, cx * s, cy * s,
                                       cz * s, false, nullptr, &nn);
                force = !(nn >= kMinNN);
            }
            if (force || d2f <= thr) {
                const double d2 = tri_dist2<double>(qx, qy, qz, ax, ay, az, bx, by, bz, cx, cy, cz, zero);
                if (d2 < best64) { best64 = d2; best_face = (int32_t)(t + k); }
                if (force) d2f = (float)(d2 * s2);
                if (d2f < best32) {
                    best32 = d2f;
                    thr = best32 + kRelTol * best32 + 2.f * sqrtf(best32) * eps + eps * eps;
                }
            }
            if (kWinding && !zero) {
                const double Ax = ax - qx, Ay = ay - qy, Az = az - qz;
                const double Bx = bx - qx, By = by - qy, Bz = bz - qz;
                const double Cx = cx - qx, Cy = cy - qy, Cz = cz - qz;
                const double la = sqrt(Ax * Ax + Ay * Ay + Az * Az);
                const double lb = sqrt(Bx * Bx + By * By + Bz * Bz);
                const double lc = sqrt(Cx * Cx + Cy * Cy + Cz * Cz);
                const double det = Ax * (By * Cz - Bz * Cy) + Ay * (Bz * Cx - Bx * Cz) + Az * (Bx * Cy - By * Cx);
                const double den = la * lb * lc + (Ax * Bx + Ay * By + Az * Bz) * lc + (Bx * Cx + By * Cy + Bz * Cz) * la +
                                   (Cx * Ax + Cy * Ay + Cz * Az) * lb;
                wind += atan2(det, den);   // half the solid angle of the face seen from q
            }
        }
    }
    if (i < Q) {
        const int64_t o = (int64_t)blockIdx.y * Q + i;
        part_d2[o] = best64;
        part_face[o] = best_face;
        if (kWinding) part_wind[o] = wind;
    }
}

__global__ void __launch_bounds__(256)
meshsdf_finalize_kernel(const double* __restrict__ part_d2, const int32_t* __restrict__ part_face,
                        const double* __restrict__ part_wind, int slabs, int64_t Q, float* __restrict__ dist,
                        int32_t* __restrict__ closest_face, float* __restrict__ winding) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Q) return;
    double bd = INFINITY, w = 0.0;
    int32_t bf = -1;
    for (int s = 0; s < slabs; ++s) {
        const double d = part_d2[(int64_t)s * Q + i];
        if (d < bd) { bd = d; bf = part_face[(int64_t)s * Q + i]; }   // strict <: the lower slab (lower face) wins ties
        w += part_wind[(int64_t)s * Q + i];
    }
    w *= 0.15915494309189533577;   // sum of half solid angles / (2 pi) = sum of solid angles / (4 pi)
    const double d = sqrt(bd);
    float out = (float)d;
    if (bf < 0) out = NAN;                       // a non-finite query coordinate
    else if (!(w > 0.5 || d <= 1e-8)) out = -out;
    dist[i] = out;
    if (closest_face) closest_face[i] = bf;
    if (winding) winding[i] = (float)w;
}

// slabs in ascending order (min d^2, strict <) -> unsigned distance, face, and the closest point: tri_dist2's point on
// the winning face in float64, rounded to fp32 once
__global__ void __launch_bounds__(256)
mesh_closest_finalize_kernel(const double* __restrict__ part_d2, const int32_t* __restrict__ part_face, int slabs,
                             int64_t Q, const float* __restrict__ verts, const int32_t* __restrict__ faces,
                             const float* __restrict__ query, float* __restrict__ closest, float* __restrict__ dist,
                             int32_t* __restrict__ closest_face) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Q) return;
    double bd = INFINITY;
    int32_t bf = -1;
    for (int s = 0; s < slabs; ++s) {
        const double d = part_d2[(int64_t)s * Q + i];
        if (d < bd) { bd = d; bf = part_face[(int64_t)s * Q + i]; }   // strict <: the lower slab (lower face) wins ties
    }
    dist[i] = bf < 0 ? NAN : (float)sqrt(bd);   // bf < 0: a non-finite query coordinate
    if (closest_face) closest_face[i] = bf;
    if (!closest) return;
    double cp[3] = {NAN, NAN, NAN};
    if (bf >= 0) {
        float c[9];
        load_face(verts, faces, bf, c);
        tri_dist2<double>(query[3 * i], query[3 * i + 1], query[3 * i + 2], c[0], c[1], c[2], c[3], c[4], c[5], c[6], c[7],
                          c[8], face_flags(c) & kZeroArea, cp);
    }
    closest[3 * i] = (float)cp[0]; closest[3 * i + 1] = (float)cp[1]; closest[3 * i + 2] = (float)cp[2];
}

// kSigned: signed distance (+ winding); else unsigned distance (+ closest point)
template <bool kSigned>
void mesh_query(const float* verts, int64_t V, const int32_t* faces, int64_t F, const float* query, int64_t Q,
                float* dist, int32_t* closest_face, float* winding, float* closest, cudaStream_t st) {
    P2S_CHECK(V > 0 && F > 0, "empty mesh");
    P2S_CHECK(V <= INT32_MAX && F <= INT32_MAX / 3, "mesh too large for int32 indices");
    static thread_local std::vector<Workspace> t_ws;   // one per instantiation: signed distance, closest point
    Workspace& ws = for_device(t_ws).begin(st);
    unsigned* flags = ws.get<unsigned>(2);   // [0] out-of-range face indices, [1] max |vertex coordinate| (bits)
    P2S_CUDA(cudaMemsetAsync(flags, 0, 2 * sizeof(unsigned), st));
    const int64_t n = 3 * std::max(V, F);
    P2S_LAUNCH(mesh_check_kernel, (unsigned)cdiv(n, 256), 256, 0, st, verts, V, faces, F, flags);
    const std::vector<unsigned> h = read_back(flags, 2, st);
    P2S_CHECK(h[0] == 0, "face index outside [0, V)");
    float vmax;
    memcpy(&vmax, &h[1], 4);
    P2S_CHECK(std::isfinite(vmax), "non-finite vertex coordinate");
    if (Q <= 0) return;
    // slab boundaries are a function of F alone: the per-slab partials, and so the results, do not depend on Q
    const int64_t slab_len = std::max<int64_t>(kTile, cdiv(cdiv(F, kMaxSlabs), kTile) * kTile);
    const int slabs = (int)cdiv(F, slab_len);
    const int64_t qc = std::min(Q, kChunk);
    double* d2 = ws.get<double>(slabs * qc);
    int32_t* fc = ws.get<int32_t>(slabs * qc);
    double* wn = kSigned ? ws.get<double>(slabs * qc) : nullptr;
    for (int64_t q0 = 0; q0 < Q; q0 += kChunk) {
        const int64_t nq = std::min(kChunk, Q - q0);
        P2S_LAUNCH(meshsdf_slab_kernel<kSigned>, dim3((unsigned)cdiv(nq, kThreads), (unsigned)slabs), kThreads, 0, st, verts,
                   faces, F, slab_len, query + 3 * q0, nq, vmax, d2, fc, wn);
        if (kSigned)
            P2S_LAUNCH(meshsdf_finalize_kernel, (unsigned)cdiv(nq, 256), 256, 0, st, d2, fc, wn, slabs, nq, dist + q0,
                       closest_face ? closest_face + q0 : nullptr, winding ? winding + q0 : nullptr);
        else
            P2S_LAUNCH(mesh_closest_finalize_kernel, (unsigned)cdiv(nq, 256), 256, 0, st, d2, fc, slabs, nq, verts, faces,
                       query + 3 * q0, closest ? closest + 3 * q0 : nullptr, dist + q0,
                       closest_face ? closest_face + q0 : nullptr);
    }
}

}  // namespace

void mesh_signed_distance(const float* verts, int64_t V, const int32_t* faces, int64_t F, const float* query, int64_t Q,
                          float* dist, int32_t* closest_face, float* winding, cudaStream_t st) {
    mesh_query<true>(verts, V, faces, F, query, Q, dist, closest_face, winding, nullptr, st);
}

void mesh_closest_point(const float* verts, int64_t V, const int32_t* faces, int64_t F, const float* query, int64_t Q,
                        float* closest, float* dist, int32_t* closest_face, cudaStream_t st) {
    mesh_query<false>(verts, V, faces, F, query, Q, dist, closest_face, nullptr, closest, st);
}

}  // namespace p2s
