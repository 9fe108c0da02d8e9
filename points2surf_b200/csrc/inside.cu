// Solid voxelisation: the inside flag of every voxel centre of a res^3 grid, by the parity of the faces that the ray from
// the centre towards +z crosses (rules in include/p2s_b200.h, "solid voxelisation"; restated in oracle/inside_oracle.py).
// The exact-sign volume of make_dataset's 06_mc_gt_exact_sign stage.  One pass over the faces, no per-voxel face loop:
//   1. inside_check_kernel: every face index in [0, V), every vertex finite with |x|, |y| < 16 (read back)
//   2. inside_faces_kernel: one warp per face; the lanes walk the columns of the face's bounding box, test each column
//      centre against the projected face exactly (fixed-point x / y, int64 edge functions), and for a crossing at height
//      z toggle bit k0 - 1 of the column's toggle words, k0 = the number of voxel centres below z.  atomicXor commutes,
//      so the result does not depend on the order of the faces.
//   3. inside_scan_kernel: one warp per column; suffix XOR of the toggles from the top of the column down -> the uint8
//      flag of each voxel, written in 32-byte coalesced runs.
// Work: O(F + sum of the faces' projected areas in columns) for the faces, res^3 / 8 bytes of toggles and res^3 bytes of
// flags for the scan.
#include "common.cuh"

namespace p2s {

namespace {

constexpr double kFixScale = 67108864.0;   // 2^26: fixed-point fraction of the projected coordinates
constexpr float kMaxXY = 16.0f;            // |x|, |y| < 16 keeps |X| < 2^30, so every edge function fits in int64

__device__ __forceinline__ long long fix(float x) { return __double2ll_rn((double)x * kFixScale); }

// voxel centre i of res (the points of p2s_query_points_dev)
__device__ __forceinline__ float centre(int i, int res) { return (float)(((double)i + 0.5) / (double)res * 2.0 - 1.0); }

// the edge function (u - p) x (v - p) of the directed projected edge u -> v at p, exact in int64, and its sign at p moved
// by (eps, eps^2) (simulation of simplicity): the sign of e, else -sign(v.y - u.y), else sign(v.x - u.x); 0 only when u
// and v project to the same point
__device__ __forceinline__ long long edge_fn(long long ux, long long uy, long long vx, long long vy, long long px,
                                             long long py, int& sign) {
    const long long e = (ux - px) * (vy - py) - (uy - py) * (vx - px);
    const long long dx = vx - ux, dy = vy - uy;
    sign = e != 0 ? (e > 0 ? 1 : -1) : (dy != 0 ? (dy < 0 ? 1 : -1) : (dx > 0 ? 1 : (dx < 0 ? -1 : 0)));
    return e;
}

__global__ void __launch_bounds__(256)
inside_check_kernel(const float* __restrict__ verts, int64_t V, const int32_t* __restrict__ faces, int64_t F,
                    unsigned* __restrict__ flags) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool bad_face = false, bad_vert = false;
    if (i < 3 * F) {
        const int32_t x = faces[i];
        bad_face = x < 0 || x >= V;
    }
    if (i < V) {
        const float x = verts[3 * i], y = verts[3 * i + 1], z = verts[3 * i + 2];
        bad_vert = !(fabsf(x) < kMaxXY && fabsf(y) < kMaxXY && isfinite(z));   // NaN fails the comparisons
    }
    const unsigned nf = __popc(__ballot_sync(0xffffffffu, bad_face));
    const unsigned nv = __popc(__ballot_sync(0xffffffffu, bad_vert));
    if ((threadIdx.x & 31) == 0) {
        if (nf) atomicAdd(flags, nf);
        if (nv) atomicAdd(flags + 1, nv);
    }
}

// toggles: [res * res][words] u32, column (ix, iy) at ix * res + iy, bit k of a column = voxels 0..k flip
__global__ void __launch_bounds__(256)
inside_faces_kernel(const float* __restrict__ verts, const int32_t* __restrict__ faces, int64_t F, int res, int words,
                    unsigned* __restrict__ toggles) {
    const int64_t f = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (f >= F) return;
    int32_t id[3];
    long long X[3], Y[3];
    double Z[3];
    float lo_x = INFINITY, hi_x = -INFINITY, lo_y = INFINITY, hi_y = -INFINITY;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        id[k] = faces[3 * f + k];
        const float x = verts[3 * (int64_t)id[k]], y = verts[3 * (int64_t)id[k] + 1];
        X[k] = fix(x);
        Y[k] = fix(y);
        Z[k] = verts[3 * (int64_t)id[k] + 2];
        lo_x = fminf(lo_x, x); hi_x = fmaxf(hi_x, x);
        lo_y = fminf(lo_y, y); hi_y = fmaxf(hi_y, y);
    }
    // twice the projected area, exact: 0 for a face parallel to z or with a repeated vertex, which crosses no column
    if ((X[1] - X[0]) * (Y[2] - Y[0]) - (Y[1] - Y[0]) * (X[2] - X[0]) == 0) return;
    // columns of the bounding box, one column of margin on each side for the rounding of the bounds
    auto first = [res](float lo) { return max(0, (int)floorf(((lo + 1.0f) * 0.5f) * (float)res - 0.5f) - 1); };
    auto last = [res](float hi) { return min(res - 1, (int)ceilf(((hi + 1.0f) * 0.5f) * (float)res - 0.5f) + 1); };
    const int i0 = first(fmaxf(lo_x, -2.0f)), i1 = last(fminf(hi_x, 2.0f));
    const int j0 = first(fmaxf(lo_y, -2.0f)), j1 = last(fminf(hi_y, 2.0f));
    if (i0 > i1 || j0 > j1) return;
    const int nj = j1 - j0 + 1;
    const int64_t n = (int64_t)(i1 - i0 + 1) * nj;
    for (int64_t t = lane; t < n; t += 32) {
        const int i = i0 + (int)(t / nj), j = j0 + (int)(t % nj);
        const long long px = fix(centre(i, res)), py = fix(centre(j, res));
        long long e[3];
        int s[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            // edge k runs from corner k to corner k + 1; evaluated on its canonical order (lower vertex index first)
            const int a = k, b = k == 2 ? 0 : k + 1;
            const bool fwd = id[a] < id[b];
            const int u = fwd ? a : b, v = fwd ? b : a;
            e[k] = edge_fn(X[u], Y[u], X[v], Y[v], px, py, s[k]);
            if (!fwd) { e[k] = -e[k]; s[k] = -s[k]; }
        }
        if (s[0] != s[1] || s[1] != s[2]) continue;
        // barycentric height: corner k is weighted by the edge opposite it (edge k + 1)
        const double w0 = __ll2double_rn(e[1]), w1 = __ll2double_rn(e[2]), w2 = __ll2double_rn(e[0]);
        const double num = __dadd_rn(__dadd_rn(__dmul_rn(w0, Z[0]), __dmul_rn(w1, Z[1])), __dmul_rn(w2, Z[2]));
        const double z = __ddiv_rn(num, __dadd_rn(__dadd_rn(w0, w1), w2));
        // k0 = #{k : centre(k) < z}, from an estimate corrected against the centres themselves
        const double g = fmin(fmax((z + 1.0) * 0.5 * res, -1.0), (double)res + 1.0);
        int k0 = min(max((int)g, 0), res);
        while (k0 > 0 && (double)centre(k0 - 1, res) >= z) --k0;
        while (k0 < res && (double)centre(k0, res) < z) ++k0;
        if (k0 > 0) {
            const int64_t col = (int64_t)i * res + j;
            atomicXor(toggles + col * words + ((k0 - 1) >> 5), 1u << ((k0 - 1) & 31));
        }
    }
}

__global__ void __launch_bounds__(256)
inside_scan_kernel(const unsigned* __restrict__ toggles, int res, int words, uint8_t* __restrict__ inside) {
    const int64_t col = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (col >= (int64_t)res * res) return;   // whole warps: col is the same for all 32 lanes
    const unsigned w = lane < words ? toggles[col * words + lane] : 0u;
    // bit b of s = XOR of bits b..31 of w; bit 0 = the parity of the whole word
    unsigned s = w;
    s ^= s >> 1; s ^= s >> 2; s ^= s >> 4; s ^= s >> 8; s ^= s >> 16;
    const unsigned par = __ballot_sync(0xffffffffu, s & 1u);
    const unsigned above = lane == 31 ? 0u : par >> (lane + 1);   // the words above this lane's
    const unsigned bits = (__popc(above) & 1) ? ~s : s;
    uint8_t* out = inside + col * res;
    for (int wi = 0; wi < words; ++wi) {
        const unsigned b = __shfl_sync(0xffffffffu, bits, wi);
        const int k = wi * 32 + lane;
        if (k < res) out[k] = (uint8_t)((b >> lane) & 1u);
    }
}

}  // namespace

void mesh_inside_grid(const float* verts, int64_t V, const int32_t* faces, int64_t F, int res, uint8_t* inside,
                      cudaStream_t st) {
    P2S_CHECK(res >= 2 && res <= 1024, "grid resolution out of range");
    P2S_CHECK(V >= 0 && F >= 0, "negative vertex or face count");
    P2S_CHECK(V <= INT32_MAX && F <= INT32_MAX / 3, "mesh too large for int32 indices");
    static thread_local std::vector<Workspace> t_ws;
    Workspace& ws = for_device(t_ws).begin(st);
    unsigned* flags = ws.get<unsigned>(2);   // [0] out-of-range face indices, [1] vertices out of range / non-finite
    const int words = (res + 31) / 32;
    const int64_t cols = (int64_t)res * res;
    unsigned* toggles = ws.get<unsigned>(cols * words);
    P2S_CUDA(cudaMemsetAsync(flags, 0, 2 * sizeof(unsigned), st));
    P2S_LAUNCH(inside_check_kernel, grid1d(std::max(3 * F, V), 256), 256, 0, st, verts, V, faces, F, flags);
    const std::vector<unsigned> h = read_back(flags, 2, st);
    P2S_CHECK(h[0] == 0, "face index outside [0, V)");
    P2S_CHECK(h[1] == 0, "vertex with |x| or |y| >= 16 or a non-finite coordinate");
    P2S_CUDA(cudaMemsetAsync(toggles, 0, (size_t)cols * words * sizeof(unsigned), st));
    if (F > 0) P2S_LAUNCH(inside_faces_kernel, grid1d(32 * F, 256), 256, 0, st, verts, faces, F, res, words, toggles);
    P2S_LAUNCH(inside_scan_kernel, grid1d(32 * cols, 256), 256, 0, st, toggles, res, words, inside);
}

}  // namespace p2s
