// Mesh repair before DeepSDF's far samples -- the first four filters of hole_filling_mesh_simp.mlx
// (dataset_for_deepsdf.py: apply_meshlab_filter).  Rules, output order and the deviations from meshlab are stated in
// include/p2s_b200.h; oracle/mesh_repair_oracle.py restates them in NumPy.
//   1. mr_check_kernel: index range and repeated indices per face
//   2. edges of the input faces (half-edges radix-sorted by undirected edge, run-length encoded); mr_nonmanifold_kernel
//      ranks the faces of every run of > 2 by (squared area, descending index) and drops all but the two largest
//   3. fans: union-find over the corners (face, slot), joining the corners of both faces at both ends of every
//      two-face edge (hook the larger root under the smaller with a CAS, so each root is its fan's lowest corner);
//      the lowest fan head of a vertex keeps it (atomicMin), the other heads, selected in corner order, get copies
//   4. holes: boundary edges into per-vertex tables (exactly two entries per boundary vertex after 3), loops by a
//      union-find over vertices (root = lowest vertex); the owner thread of each short loop walks it and cuts ears
//      sequentially, writing into slots from an exclusive scan; a second scan compacts the loops that closed
// Only integer atomics; the float64 geometry uses explicitly rounded operations, so the output is bitwise identical
// across runs and equal to the oracle's.
#include "common.cuh"
#include "model.cuh"
#include <climits>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

namespace p2s {

namespace {

constexpr int kMaxLoop = 128;             // largest max_hole_size (per-thread loop arrays)
constexpr uint32_t kIdx = 0x7fffffffu;    // boundary table: vertex bits; bit 31 = the face runs from this vertex out

enum Counter { C_BAD_INDEX, C_REPEATED, C_OVER2, C_BAD_DEGREE, C_CLOSED, C_OPEN, C_COUNT };

__device__ __forceinline__ void count(unsigned long long* c, int which) { atomicAdd(c + which, 1ull); }

__global__ void __launch_bounds__(256)
mr_check_kernel(const int32_t* __restrict__ faces, int F, int V, unsigned long long* cnt) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const int a = faces[3 * (int64_t)f], b = faces[3 * (int64_t)f + 1], c = faces[3 * (int64_t)f + 2];
    if (a < 0 || a >= V || b < 0 || b >= V || c < 0 || c >= V) count(cnt, C_BAD_INDEX);
    else if (a == b || b == c || a == c) count(cnt, C_REPEATED);
}

__device__ __forceinline__ int next_he(int h) { return h % 3 == 2 ? h - 2 : h + 1; }

__global__ void __launch_bounds__(256)
mr_halfedge_kernel(const int32_t* __restrict__ W, int n3, unsigned long long* key, int32_t* val) {
    const int h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n3) return;
    const uint32_t u = W[h], v = W[next_he(h)];
    key[h] = u < v ? ((unsigned long long)u << 32) | v : ((unsigned long long)v << 32) | u;
    val[h] = h;
}

__device__ __forceinline__ double vc(const float* v, int i, int k) { return (double)v[3 * (int64_t)i + k]; }

// |(b - a) x (c - a)|^2 in the oracle's order
__device__ double area2(const float* v, int a, int b, int c) {
    const double ux = __dsub_rn(vc(v, b, 0), vc(v, a, 0)), uy = __dsub_rn(vc(v, b, 1), vc(v, a, 1)),
                 uz = __dsub_rn(vc(v, b, 2), vc(v, a, 2));
    const double wx = __dsub_rn(vc(v, c, 0), vc(v, a, 0)), wy = __dsub_rn(vc(v, c, 1), vc(v, a, 1)),
                 wz = __dsub_rn(vc(v, c, 2), vc(v, a, 2));
    const double nx = __dsub_rn(__dmul_rn(uy, wz), __dmul_rn(uz, wy));
    const double ny = __dsub_rn(__dmul_rn(uz, wx), __dmul_rn(ux, wz));
    const double nz = __dsub_rn(__dmul_rn(ux, wy), __dmul_rn(uy, wx));
    return __dadd_rn(__dadd_rn(__dmul_rn(nx, nx), __dmul_rn(ny, ny)), __dmul_rn(nz, nz));
}

// rule 1: in every run of c > 2 faces, drop the c - 2 first in (area ascending, face index descending) order
__global__ void __launch_bounds__(256)
mr_nonmanifold_kernel(const float* __restrict__ verts, const int32_t* __restrict__ faces, const int32_t* __restrict__ he,
                      const int32_t* __restrict__ rcnt, const int32_t* __restrict__ roff, int R, uint8_t* keep) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R || rcnt[r] <= 2) return;
    const int c = rcnt[r], o = roff[r];
    for (int i = 0; i < c; ++i) {
        const int f = he[o + i] / 3;
        const double ai = area2(verts, faces[3 * f], faces[3 * f + 1], faces[3 * f + 2]);
        int rank = 0;
        for (int j = 0; j < c; ++j) {
            const int g = he[o + j] / 3;
            const double aj = area2(verts, faces[3 * g], faces[3 * g + 1], faces[3 * g + 2]);
            rank += aj < ai || (aj == ai && g > f);
        }
        if (rank < c - 2) keep[f] = 0;
    }
}

__global__ void __launch_bounds__(256)
mr_gather_faces_kernel(const int32_t* __restrict__ faces, const int32_t* __restrict__ ids, int n, int32_t* W) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
#pragma unroll
    for (int k = 0; k < 3; ++k) W[3 * (int64_t)i + k] = faces[3 * (int64_t)ids[i] + k];
}

__global__ void __launch_bounds__(256)
mr_over2_kernel(const int32_t* __restrict__ rcnt, int R, unsigned long long* cnt) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < R && rcnt[r] > 2) count(cnt, C_OVER2);
}

// ---- union-find over int32 ids, root = the lowest id of the set
__device__ __forceinline__ int uf_load(const int32_t* par, int x) { return *reinterpret_cast<const volatile int32_t*>(par + x); }

__device__ int uf_find(int32_t* par, int x) {
    while (true) {
        const int p = uf_load(par, x);
        if (p == x) return x;
        const int g = uf_load(par, p);
        if (g != p) atomicCAS(par + x, p, g);   // path halving
        x = p;
    }
}

__device__ void uf_union(int32_t* par, int a, int b) {
    while (true) {
        const int ra = uf_find(par, a), rb = uf_find(par, b);
        if (ra == rb) return;
        const int hi = max(ra, rb), lo = min(ra, rb);
        if (atomicCAS(par + hi, hi, lo) == hi) return;
    }
}

__global__ void __launch_bounds__(256) mr_iota_kernel(int32_t* a, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i] = i;
}

// rule 3: the corners of both faces at both ends of a two-face edge belong to the same fan
__global__ void __launch_bounds__(256)
mr_fan_union_kernel(const int32_t* __restrict__ W, const int32_t* __restrict__ he, const int32_t* __restrict__ rcnt,
                    const int32_t* __restrict__ roff, int R, int32_t* par) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R || rcnt[r] != 2) return;
    const int h0 = he[roff[r]], h1 = he[roff[r] + 1];
    const bool same = W[h0] == W[h1];   // h1 starts at the same vertex as h0
    uf_union(par, h0, same ? h1 : next_he(h1));
    uf_union(par, next_he(h0), same ? next_he(h1) : h1);
}

__global__ void __launch_bounds__(256)
mr_flatten_kernel(int32_t* par, int n, int32_t* root) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) root[i] = uf_find(par, i);
}

__global__ void __launch_bounds__(256)
mr_fan_head_kernel(const int32_t* __restrict__ W, const int32_t* __restrict__ root, int n3, int32_t* minhead) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < n3 && root[c] == c) atomicMin(minhead + W[c], c);
}

__global__ void __launch_bounds__(256)
mr_extra_head_kernel(const int32_t* __restrict__ W, const int32_t* __restrict__ root, const int32_t* __restrict__ minhead,
                     int n3, uint8_t* extra) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < n3) extra[c] = root[c] == c && minhead[W[c]] != c;
}

// copy p of the vertex of fan head E[p] is vertex V + p
__global__ void __launch_bounds__(256)
mr_copy_ids_kernel(const int32_t* __restrict__ W, const int32_t* __restrict__ E, int S, int V, int32_t* copyid,
                   const float* __restrict__ verts, float* verts_out) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= S) return;
    copyid[E[p]] = V + p;
    const int v = W[E[p]];
#pragma unroll
    for (int k = 0; k < 3; ++k) verts_out[3 * ((int64_t)V + p) + k] = verts[3 * (int64_t)v + k];
}

__global__ void __launch_bounds__(256)
mr_renumber_kernel(const int32_t* __restrict__ W, const int32_t* __restrict__ root, const int32_t* __restrict__ minhead,
                   const int32_t* __restrict__ copyid, int n3, int32_t* Wn) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n3) return;
    const int r = root[c];
    Wn[c] = minhead[W[c]] == r ? W[c] : copyid[r];
}

__device__ __forceinline__ void bnd_insert(int32_t* deg, uint32_t* nb, int at, uint32_t entry) {
    const int slot = atomicAdd(deg + at, 1);
    if (slot < 2) nb[2 * (int64_t)at + slot] = entry;
}

__global__ void __launch_bounds__(256)
mr_boundary_kernel(const int32_t* __restrict__ W, const int32_t* __restrict__ he, const int32_t* __restrict__ rcnt,
                   const int32_t* __restrict__ roff, int R, int32_t* deg, uint32_t* nb, int32_t* vpar) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R || rcnt[r] != 1) return;
    const int h = he[roff[r]];
    const int u = W[h], v = W[next_he(h)];
    bnd_insert(deg, nb, u, (uint32_t)v | 0x80000000u);
    bnd_insert(deg, nb, v, (uint32_t)u);
    uf_union(vpar, u, v);
}

__global__ void __launch_bounds__(256)
mr_loop_len_kernel(const int32_t* __restrict__ deg, int32_t* vpar, int V, int32_t* len, unsigned long long* cnt) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V || deg[v] == 0) return;
    if (deg[v] != 2) count(cnt, C_BAD_DEGREE);
    atomicAdd(len + uf_find(vpar, v), 1);
}

// slots reserved per loop owner: L - 2 for a loop short enough to fill, else 0 (the long ones are counted open)
__global__ void __launch_bounds__(256)
mr_reserve_kernel(const int32_t* __restrict__ deg, const int32_t* __restrict__ vpar, const int32_t* __restrict__ len, int V,
                  int max_hole, int32_t* nfill, unsigned long long* cnt) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    int n = 0;
    if (deg[v] == 2 && vpar[v] == v) {
        if (len[v] <= max_hole) n = len[v] - 2;
        else count(cnt, C_OPEN);
    }
    nfill[v] = n;
}

__global__ void __launch_bounds__(256)
mr_corner_count_kernel(const int32_t* __restrict__ Wn, int n3, int32_t* vcnt) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < n3) atomicAdd(vcnt + Wn[c], 1);
}

__global__ void __launch_bounds__(256)
mr_u32_kernel(const int32_t* __restrict__ a, int n, uint32_t* b) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) b[i] = (uint32_t)a[i];
}

// ---- float64 geometry in the oracle's order
struct D3 { double x, y, z; };

__device__ __forceinline__ D3 pos(const float* v, int i) { return {vc(v, i, 0), vc(v, i, 1), vc(v, i, 2)}; }
__device__ __forceinline__ bool same_pt(const D3& a, const D3& b) { return a.x == b.x && a.y == b.y && a.z == b.z; }
__device__ __forceinline__ D3 sub(const D3& a, const D3& b) {
    return {__dsub_rn(a.x, b.x), __dsub_rn(a.y, b.y), __dsub_rn(a.z, b.z)};
}
__device__ __forceinline__ double dot(const D3& a, const D3& b) {
    return __dadd_rn(__dadd_rn(__dmul_rn(a.x, b.x), __dmul_rn(a.y, b.y)), __dmul_rn(a.z, b.z));
}
__device__ __forceinline__ D3 cross(const D3& u, const D3& w) {
    return {__dsub_rn(__dmul_rn(u.y, w.z), __dmul_rn(u.z, w.y)), __dsub_rn(__dmul_rn(u.z, w.x), __dmul_rn(u.x, w.z)),
            __dsub_rn(__dmul_rn(u.x, w.y), __dmul_rn(u.y, w.x))};
}

// ((b - a) x (c - a)) . (d - a), exactly 0 when two of the four points coincide
__device__ double orient3(const D3& a, const D3& b, const D3& c, const D3& d) {
    if (same_pt(a, b) || same_pt(a, c) || same_pt(a, d) || same_pt(b, c) || same_pt(b, d) || same_pt(c, d)) return 0.0;
    return dot(cross(sub(b, a), sub(c, a)), sub(d, a));
}

// segment pq crosses the interior of triangle abc strictly
__device__ bool seg_cross(const D3& p, const D3& q, const D3& a, const D3& b, const D3& c) {
    const double o1 = orient3(a, b, c, p), o2 = orient3(a, b, c, q);
    if (!((o1 > 0.0 && o2 < 0.0) || (o1 < 0.0 && o2 > 0.0))) return false;
    const double s1 = orient3(p, q, a, b), s2 = orient3(p, q, b, c), s3 = orient3(p, q, c, a);
    return (s1 > 0.0 && s2 > 0.0 && s3 > 0.0) || (s1 < 0.0 && s2 < 0.0 && s3 < 0.0);
}

__device__ bool tri_cross(const D3& a, const D3& b, const D3& c, const D3& d, const D3& e, const D3& f) {
    return seg_cross(a, b, d, e, f) || seg_cross(b, c, d, e, f) || seg_cross(c, a, d, e, f) ||
           seg_cross(d, e, a, b, c) || seg_cross(e, f, a, b, c) || seg_cross(f, d, a, b, c);
}

__device__ __forceinline__ double orient2(double ax, double ay, double bx, double by, double qx, double qy) {
    return __dsub_rn(__dmul_rn(__dsub_rn(bx, ax), __dsub_rn(qy, ay)), __dmul_rn(__dsub_rn(by, ay), __dsub_rn(qx, ax)));
}

// the boundary neighbour of p other than prev
__device__ __forceinline__ int bnd_other(const uint32_t* nb, int p, int prev) {
    const int a = nb[2 * (int64_t)p] & kIdx, b = nb[2 * (int64_t)p + 1] & kIdx;
    return a == prev ? b : a;
}

// rule 4 for the loop owned by v: ear cutting into out[0 .. L-3]; -> L - 2 faces, or 0 when no valid ear is left
__device__ int fill_loop(const float* verts, const int32_t* Wn, const int32_t* vstart, const int32_t* vcorner,
                         const uint32_t* nb, int v, int L, bool psi, int32_t* out) {
    int ring[kMaxLoop], idx[kMaxLoop];
    double s[kMaxLoop], t[kMaxLoop];
    bool tried[kMaxLoop];
    // walk: towards the neighbour whose edge runs into v (bit 31 clear), the lower one when both or neither do
    const uint32_t e0 = nb[2 * (int64_t)v], e1 = nb[2 * (int64_t)v + 1];
    const bool in0 = !(e0 >> 31), in1 = !(e1 >> 31);
    const int n0 = e0 & kIdx, n1 = e1 & kIdx;
    int cur = (in0 != in1) ? (in0 ? n0 : n1) : min(n0, n1), prev = v;
    ring[0] = v;
    for (int i = 1; i < L; ++i) {
        ring[i] = cur;
        const int nx = bnd_other(nb, cur, prev);
        prev = cur;
        cur = nx;
    }
    // Newell normal of the walk, then the 2D frame
    double nx = 0.0, ny = 0.0, nz = 0.0;
    for (int i = 0; i < L; ++i) {
        const D3 a = pos(verts, ring[i]), b = pos(verts, ring[(i + 1) % L]);
        nx = __dadd_rn(nx, __dmul_rn(__dsub_rn(a.y, b.y), __dadd_rn(a.z, b.z)));
        ny = __dadd_rn(ny, __dmul_rn(__dsub_rn(a.z, b.z), __dadd_rn(a.x, b.x)));
        nz = __dadd_rn(nz, __dmul_rn(__dsub_rn(a.x, b.x), __dadd_rn(a.y, b.y)));
    }
    const D3 n{nx, ny, nz};
    const double nl = __dsqrt_rn(dot(n, n));
    if (nl == 0.0) return 0;
    const double ax = fabs(nx), ay = fabs(ny), az = fabs(nz);
    D3 u = (ax <= ay && ax <= az) ? D3{0.0, nz, -ny} : (ay <= az ? D3{-nz, 0.0, nx} : D3{ny, -nx, 0.0});
    const double ul = __dsqrt_rn(dot(u, u));
    u = {__ddiv_rn(u.x, ul), __ddiv_rn(u.y, ul), __ddiv_rn(u.z, ul)};
    const D3 w = cross(D3{__ddiv_rn(nx, nl), __ddiv_rn(ny, nl), __ddiv_rn(nz, nl)}, u);
    for (int i = 0; i < L; ++i) {
        const D3 p = pos(verts, ring[i]);
        s[i] = dot(p, u);
        t[i] = dot(p, w);
        idx[i] = i;
    }
    int m = L, added = 0;
    while (m >= 3) {
        for (int j = 0; j < m; ++j) tried[j] = false;
        int cut = -1;
        while (cut < 0) {
            // the untried convex ear with the largest cos (smallest tip angle), ties by the lowest tip vertex id
            int best = -1;
            double best_cos = 0.0;
            for (int j = 0; j < m; ++j) {
                if (tried[j]) continue;
                const int a = idx[(j + m - 1) % m], b = idx[j], c = idx[(j + 1) % m];
                const double px = __dsub_rn(s[a], s[b]), py = __dsub_rn(t[a], t[b]);
                const double qx = __dsub_rn(s[c], s[b]), qy = __dsub_rn(t[c], t[b]);
                if (!(__dsub_rn(__dmul_rn(py, qx), __dmul_rn(px, qy)) > 0.0)) continue;
                const double cs = __ddiv_rn(__dadd_rn(__dmul_rn(px, qx), __dmul_rn(py, qy)),
                                            __dmul_rn(__dsqrt_rn(__dadd_rn(__dmul_rn(px, px), __dmul_rn(py, py))),
                                                      __dsqrt_rn(__dadd_rn(__dmul_rn(qx, qx), __dmul_rn(qy, qy)))));
                if (best < 0 || cs > best_cos || (cs == best_cos && ring[b] < ring[idx[best]])) {
                    best = j;
                    best_cos = cs;
                }
            }
            if (best < 0) return 0;
            tried[best] = true;
            const int a = idx[(best + m - 1) % m], b = idx[best], c = idx[(best + 1) % m];
            bool ok = true;
            for (int j = 0; j < m && ok; ++j) {
                const int q = idx[j];
                if (q == a || q == b || q == c) continue;
                ok = !(orient2(s[a], t[a], s[b], t[b], s[q], t[q]) >= 0.0 &&
                       orient2(s[b], t[b], s[c], t[c], s[q], t[q]) >= 0.0 &&
                       orient2(s[c], t[c], s[a], t[a], s[q], t[q]) >= 0.0);
            }
            // the ear's new edge must not already be an edge of the mesh (it would get a third face)
            for (int k = vstart[ring[a]]; k < vstart[ring[a] + 1] && ok && m > 3; ++k) {
                const int64_t f = vcorner[k] / 3;
                ok = Wn[3 * f] != ring[c] && Wn[3 * f + 1] != ring[c] && Wn[3 * f + 2] != ring[c];
            }
            if (ok && psi) {
                const D3 A = pos(verts, ring[a]), B = pos(verts, ring[b]), C = pos(verts, ring[c]);
                for (int i = 0; i < L && ok; ++i) {
                    for (int k = vstart[ring[i]]; k < vstart[ring[i] + 1] && ok; ++k) {
                        const int64_t f = vcorner[k] / 3;
                        ok = !tri_cross(A, B, C, pos(verts, Wn[3 * f]), pos(verts, Wn[3 * f + 1]), pos(verts, Wn[3 * f + 2]));
                    }
                }
                for (int i = 0; i < added && ok; ++i)
                    ok = !tri_cross(A, B, C, pos(verts, out[3 * i]), pos(verts, out[3 * i + 1]), pos(verts, out[3 * i + 2]));
            }
            if (ok) cut = best;
        }
        const int a = idx[(cut + m - 1) % m], b = idx[cut], c = idx[(cut + 1) % m];
        out[3 * added] = ring[a];
        out[3 * added + 1] = ring[b];
        out[3 * added + 2] = ring[c];
        ++added;
        for (int j = cut; j < m - 1; ++j) idx[j] = idx[j + 1];
        --m;
    }
    return added;
}

__global__ void __launch_bounds__(128)
mr_fill_kernel(const float* __restrict__ verts, const int32_t* __restrict__ Wn, const int32_t* __restrict__ vstart,
               const int32_t* __restrict__ vcorner, const uint32_t* __restrict__ nb, const int32_t* __restrict__ len,
               const int32_t* __restrict__ nfill, const int32_t* __restrict__ foff, int V, bool psi, int32_t* tmp,
               int32_t* done, unsigned long long* cnt) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    done[v] = 0;
    if (nfill[v] == 0) return;
    const int k = fill_loop(verts, Wn, vstart, vcorner, nb, v, len[v], psi, tmp + 3 * (int64_t)foff[v]);
    done[v] = k;
    count(cnt, k ? C_CLOSED : C_OPEN);
}

__global__ void __launch_bounds__(256)
mr_compact_kernel(const int32_t* __restrict__ tmp, const int32_t* __restrict__ foff, const int32_t* __restrict__ done,
                  const int32_t* __restrict__ doff, int V, int32_t* out) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V || done[v] == 0) return;
    for (int i = 0; i < 3 * done[v]; ++i) out[3 * (int64_t)doff[v] + i] = tmp[3 * (int64_t)foff[v] + i];
}

// the undirected edges of faces W [n][3]: half-edges sorted by edge (he), runs (count, offset)
struct Edges {
    int32_t *he, *rcnt, *roff;
    int R;
};

Edges edges(Workspace& ws, const int32_t* W, int n, cudaStream_t st) {
    Edges e{};
    const int n3 = 3 * n;
    auto* key = ws.get<unsigned long long>(n3);
    auto* key_s = ws.get<unsigned long long>(n3);
    int32_t* val = ws.get<int32_t>(n3);
    e.he = ws.get<int32_t>(n3);
    auto* ukey = ws.get<unsigned long long>(n3);
    e.rcnt = ws.get<int32_t>(n3);
    e.roff = ws.get<int32_t>(n3);
    int* d_num = ws.get<int>(1);
    if (n == 0) return e;
    P2S_LAUNCH(mr_halfedge_kernel, grid1d(n3, 256), 256, 0, st, W, n3, key, val);
    cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, key, key_s, val, e.he, n3, 0, 64, st); });
    cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceRunLengthEncode::Encode(t, b, key_s, ukey, e.rcnt, d_num, n3, st); });
    e.R = read_back(d_num, 1, st)[0];
    cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, e.rcnt, e.roff, e.R, st); });
    return e;
}

}  // namespace

void mesh_repair(const float* verts, int64_t V64, const int32_t* faces, int64_t F64, int max_hole_size,
                 bool prevent_self_intersection, float* verts_out, int64_t vcap, int32_t* faces_out, int64_t fcap,
                 p2s_repair_stats* stats, cudaStream_t st) {
    P2S_CHECK(V64 >= 0 && F64 >= 0 && vcap >= 0 && fcap >= 0, "negative size");
    P2S_CHECK(V64 + 3 * F64 < INT32_MAX && 4 * F64 < INT32_MAX / 3, "mesh too large for int32 indices");
    P2S_CHECK(max_hole_size >= 0 && max_hole_size <= kMaxLoop, "max_hole_size outside [0, 128]");
    const int V = (int)V64, F = (int)F64;
    static thread_local std::vector<Workspace> t_ws;
    Workspace& ws = for_device(t_ws).begin(st);
    p2s_repair_stats R{};
    R.vertices_in = V;
    R.faces_in = F;
    unsigned long long* cnt = ws.get<unsigned long long>(C_COUNT);
    P2S_CUDA(cudaMemsetAsync(cnt, 0, C_COUNT * sizeof(unsigned long long), st));
    if (F > 0) P2S_LAUNCH(mr_check_kernel, grid1d(F, 256), 256, 0, st, faces, F, V, cnt);
    std::vector<unsigned long long> h = read_back(cnt, C_COUNT, st);
    P2S_CHECK(h[C_BAD_INDEX] == 0, "face index outside [0, V)");
    P2S_CHECK(h[C_REPEATED] == 0, "face with a repeated vertex index");

    // 1. non-manifold edges: drop the smallest faces of every edge with more than two
    uint8_t* keep = ws.get<uint8_t>(F);
    int32_t* ids = ws.get<int32_t>(F);
    int* d_num = ws.get<int>(1);
    int K = 0;
    if (F > 0) {
        P2S_CUDA(cudaMemsetAsync(keep, 1, F, st));
        const Edges e = edges(ws, faces, F, st);
        P2S_LAUNCH(mr_nonmanifold_kernel, grid1d(e.R, 256), 256, 0, st, verts, faces, e.he, e.rcnt, e.roff, e.R, keep);
        cub::CountingInputIterator<int32_t> counting(0);
        cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, counting, keep, ids, d_num, F, st); });
        K = read_back(d_num, 1, st)[0];
    }
    R.faces_removed = F - K;
    int32_t* W = ws.get<int32_t>(3 * (int64_t)K);
    if (K > 0) P2S_LAUNCH(mr_gather_faces_kernel, grid1d(K, 256), 256, 0, st, faces, ids, K, W);

    // 3. non-manifold vertices: fans over the corners, copies for every fan but a vertex's lowest
    const int n3 = 3 * K;
    int32_t* Wn = ws.get<int32_t>(n3);
    int32_t *root = ws.get<int32_t>(n3), *minhead = ws.get<int32_t>(V), *E = ws.get<int32_t>(n3);
    int32_t* copyid = ws.get<int32_t>(n3);
    int S = 0;
    if (K > 0) {
        const Edges e = edges(ws, W, K, st);
        P2S_LAUNCH(mr_over2_kernel, grid1d(e.R, 256), 256, 0, st, e.rcnt, e.R, cnt);
        int32_t* par = ws.get<int32_t>(n3);
        uint8_t* extra = ws.get<uint8_t>(n3);
        P2S_LAUNCH(mr_iota_kernel, grid1d(n3, 256), 256, 0, st, par, n3);
        P2S_LAUNCH(mr_fan_union_kernel, grid1d(e.R, 256), 256, 0, st, W, e.he, e.rcnt, e.roff, e.R, par);
        P2S_LAUNCH(mr_flatten_kernel, grid1d(n3, 256), 256, 0, st, par, n3, root);
        P2S_CUDA(cudaMemsetAsync(minhead, 0x7f, (size_t)V * sizeof(int32_t), st));
        P2S_LAUNCH(mr_fan_head_kernel, grid1d(n3, 256), 256, 0, st, W, root, n3, minhead);
        P2S_LAUNCH(mr_extra_head_kernel, grid1d(n3, 256), 256, 0, st, W, root, minhead, n3, extra);
        cub::CountingInputIterator<int32_t> counting(0);
        cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, counting, extra, E, d_num, n3, st); });
        S = read_back(d_num, 1, st)[0];
        P2S_CHECK(read_back(cnt + C_OVER2, 1, st)[0] == 0, "internal error: an edge kept more than two faces");
    }
    const int V2 = V + S;
    R.vertices_split = S;
    R.vertices_out = V2;
    P2S_CHECK(V2 <= vcap, "vcap too small for the repaired mesh (vcap >= V + 3 F always suffices)");
    P2S_CHECK(verts_out || V2 == 0, "null output");
    if (S > 0) P2S_LAUNCH(mr_copy_ids_kernel, grid1d(S, 256), 256, 0, st, W, E, S, V, copyid, verts, verts_out);
    if (K > 0) P2S_LAUNCH(mr_renumber_kernel, grid1d(n3, 256), 256, 0, st, W, root, minhead, copyid, n3, Wn);
    if (V > 0) P2S_CUDA(cudaMemcpyAsync(verts_out, verts, (size_t)V * 3 * sizeof(float), cudaMemcpyDeviceToDevice, st));

    // 4. holes: loops of boundary edges, the short ones filled by ear cutting
    int added = 0;
    int32_t* tmp = nullptr;
    int32_t *foff = nullptr, *done = nullptr, *doff = nullptr;
    if (K > 0) {
        const Edges e = edges(ws, Wn, K, st);
        int32_t *deg = ws.get<int32_t>(V2), *vpar = ws.get<int32_t>(V2), *len = ws.get<int32_t>(V2);
        uint32_t* nb = ws.get<uint32_t>(2 * (int64_t)V2);
        int32_t* nfill = ws.get<int32_t>(V2);
        foff = ws.get<int32_t>(V2);
        P2S_CUDA(cudaMemsetAsync(deg, 0, (size_t)V2 * sizeof(int32_t), st));
        P2S_CUDA(cudaMemsetAsync(len, 0, (size_t)V2 * sizeof(int32_t), st));
        P2S_LAUNCH(mr_iota_kernel, grid1d(V2, 256), 256, 0, st, vpar, V2);
        P2S_LAUNCH(mr_boundary_kernel, grid1d(e.R, 256), 256, 0, st, Wn, e.he, e.rcnt, e.roff, e.R, deg, nb, vpar);
        P2S_LAUNCH(mr_loop_len_kernel, grid1d(V2, 256), 256, 0, st, deg, vpar, V2, len, cnt);
        P2S_LAUNCH(mr_flatten_kernel, grid1d(V2, 256), 256, 0, st, vpar, V2, vpar);
        P2S_LAUNCH(mr_reserve_kernel, grid1d(V2, 256), 256, 0, st, deg, vpar, len, V2, max_hole_size, nfill, cnt);
        cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, nfill, foff, V2, st); });
        const int reserved = read_back(foff + (V2 - 1), 1, st)[0] + read_back(nfill + (V2 - 1), 1, st)[0];
        P2S_CHECK(read_back(cnt + C_BAD_DEGREE, 1, st)[0] == 0, "internal error: a boundary vertex without two boundary edges");
        if (reserved > 0) {
            // vertex -> incident corners (ascending), for the intersection tests
            int32_t *vcnt = ws.get<int32_t>(V2 + 1), *vstart = ws.get<int32_t>(V2 + 1);
            uint32_t *ckey = ws.get<uint32_t>(n3), *ckey_s = ws.get<uint32_t>(n3);
            int32_t *cval = ws.get<int32_t>(n3), *vcorner = ws.get<int32_t>(n3);
            P2S_CUDA(cudaMemsetAsync(vcnt, 0, (size_t)(V2 + 1) * sizeof(int32_t), st));
            P2S_LAUNCH(mr_corner_count_kernel, grid1d(n3, 256), 256, 0, st, Wn, n3, vcnt);
            cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, vcnt, vstart, V2 + 1, st); });
            P2S_LAUNCH(mr_u32_kernel, grid1d(n3, 256), 256, 0, st, Wn, n3, ckey);
            P2S_LAUNCH(mr_iota_kernel, grid1d(n3, 256), 256, 0, st, cval, n3);
            cub_run(ws, 1, [&](void* t, size_t& b) {
                return cub::DeviceRadixSort::SortPairs(t, b, ckey, ckey_s, cval, vcorner, n3, 0, 32, st);
            });
            tmp = ws.get<int32_t>(3 * (int64_t)reserved);
            done = ws.get<int32_t>(V2);
            doff = ws.get<int32_t>(V2);
            P2S_LAUNCH(mr_fill_kernel, grid1d(V2, 128), 128, 0, st, verts_out, Wn, vstart, vcorner, nb, len, nfill, foff, V2,
                       prevent_self_intersection, tmp, done, cnt);
            cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, done, doff, V2, st); });
            added = read_back(doff + (V2 - 1), 1, st)[0] + read_back(done + (V2 - 1), 1, st)[0];
        }
    }
    h = read_back(cnt, C_COUNT, st);
    R.holes_closed = (int64_t)h[C_CLOSED];
    R.holes_left_open = (int64_t)h[C_OPEN];
    R.faces_added = added;
    R.faces_out = (int64_t)K + added;
    P2S_CHECK(R.faces_out <= fcap, "fcap too small for the repaired mesh (fcap >= 4 F always suffices)");
    P2S_CHECK(faces_out || R.faces_out == 0, "null output");
    if (K > 0) P2S_CUDA(cudaMemcpyAsync(faces_out, Wn, (size_t)n3 * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    if (added > 0)
        P2S_LAUNCH(mr_compact_kernel, grid1d(V2, 256), 256, 0, st, tmp, foff, done, doff, V2, faces_out + 3 * (int64_t)K);
    P2S_CUDA(cudaStreamSynchronize(st));
    *stats = R;
}

}  // namespace p2s
