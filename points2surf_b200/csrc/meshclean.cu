// K12: mesh repair -- the _clean_mesh stage of make_dataset.py:383-413 (trimesh's process, remove_degenerate_faces,
// remove_duplicate_faces, fill_holes and fix_inversion / fix_normals / fix_winding) without the file I/O and the accept /
// reject decision.  Rules, output order and the deviations from trimesh are stated in include/p2s_b200.h.
//   1. mc_vertex_key_kernel / mc_index_check_kernel: weld keys llround(1e8 x) per coordinate, finite flags, input errors
//   2. weld: three stable radix sorts (z, y, x key) of the vertex indices; a max-scan of the run heads gives every vertex
//      the lowest input index with its key
//   3. mc_face_kernel: non-finite, repeated-index and low-altitude faces; duplicates by two stable radix sorts of the
//      sorted index triple, the first face of each run kept
//   4. classify: the half-edges sorted by undirected edge, run-length encoded; runs of 1 / 2 / >2 faces are boundary,
//      two-face (consistent iff their start vertices differ) and non-manifold edges
//   5. holes: boundary edges inserted into per-vertex tables (two slots); every loop of 3 or 4 edges through vertices of
//      boundary degree 2 is filled by the thread of its lowest vertex, at a place given by an exclusive scan over vertices
//   6. orientation: union-find over two-face edges whose parent word carries the parity to the parent (hook the larger
//      root under the smaller with a 64-bit CAS, path halving on find), so every root is its component's lowest face and
//      the parities of an orientable component do not depend on scheduling; signed volume per component in the fixed
//      order of mc_segment_sum_kernel (oracle/mesh_clean_oracle.py restates it)
//   7. unreferenced vertices dropped by an exclusive scan of the used flags
// Only integer atomics; the output is bitwise identical across runs.
#include "common.cuh"
#include <climits>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

namespace p2s {

namespace {

constexpr int kSumThreads = 256;          // fixed-order sum: lanes per segment (oracle/mesh_clean_oracle.py:fixed_sum)
constexpr double kWeldScale = 1e8;        // trimesh tol.merge = 1e-8
constexpr double kKeyLimit = 9e10;        // |x| * 1e8 must stay below 2^63
constexpr double kMinAltitude = 1e-8;     // remove_degenerate_faces height
constexpr uint32_t kIdx = 0x7fffffffu;    // boundary table: vertex bits; bit 31 = the face runs from this vertex out

enum Counter {
    C_BAD_INDEX, C_OVERFLOW, C_HEADS, C_NONFINITE, C_DEGENERATE, C_DUPLICATE, C_BOUNDARY, C_NONMANIFOLD,
    C_INCONSISTENT, C_HOLES, C_REVERSED, C_NONORIENT, C_COUNT
};

__device__ __forceinline__ void count(unsigned long long* c, int which) { atomicAdd(c + which, 1ull); }

__global__ void __launch_bounds__(256)
mc_index_check_kernel(const int32_t* __restrict__ faces, int64_t n3, int64_t V, unsigned long long* cnt) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n3 && (faces[i] < 0 || faces[i] >= V)) count(cnt, C_BAD_INDEX);
}

__global__ void __launch_bounds__(256)
mc_vertex_key_kernel(const float* __restrict__ verts, int V, long long* kx, long long* ky, long long* kz,
                     uint8_t* finite, int32_t* iota, unsigned long long* cnt) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V) return;
    const double x = verts[3 * (int64_t)i], y = verts[3 * (int64_t)i + 1], z = verts[3 * (int64_t)i + 2];
    const bool fin = isfinite(x) && isfinite(y) && isfinite(z);
    const bool big = fin && (fabs(x) >= kKeyLimit || fabs(y) >= kKeyLimit || fabs(z) >= kKeyLimit);
    if (big) count(cnt, C_OVERFLOW);
    // non-finite vertices sort last (no finite key reaches LLONG_MAX) and never merge
    kx[i] = fin && !big ? llround(x * kWeldScale) : LLONG_MAX;
    ky[i] = fin && !big ? llround(y * kWeldScale) : 0;
    kz[i] = fin && !big ? llround(z * kWeldScale) : 0;
    finite[i] = fin;
    iota[i] = i;
}

template <class T>
__global__ void __launch_bounds__(256) mc_gather_kernel(const T* __restrict__ src, const int32_t* __restrict__ idx, int n,
                                                        T* __restrict__ dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[idx[i]];
}

__global__ void __launch_bounds__(256)
mc_weld_head_kernel(const int32_t* __restrict__ order, int n, const long long* __restrict__ kx,
                    const long long* __restrict__ ky, const long long* __restrict__ kz, const uint8_t* __restrict__ finite,
                    int32_t* headpos, unsigned long long* cnt) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const int v = order[p];
    bool head = p == 0 || !finite[v];
    if (!head) {
        const int u = order[p - 1];
        head = kx[v] != kx[u] || ky[v] != ky[u] || kz[v] != kz[u];
    }
    if (head) count(cnt, C_HEADS);
    headpos[p] = head ? p : 0;
}

__global__ void __launch_bounds__(256)
mc_weld_rep_kernel(const int32_t* __restrict__ order, const int32_t* __restrict__ runstart, int n, int32_t* rep) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < n) rep[order[p]] = order[runstart[p]];
}

__device__ __forceinline__ double vc(const float* v, int i, int k) { return (double)v[3 * (int64_t)i + k]; }

// |(x, y, z)| with the rounding of the oracle
__device__ __forceinline__ double norm3(double x, double y, double z) {
    return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
}

// float64 altitude over the longest edge, 2 area / longest edge <= 1e-8 (zero-length edges count as degenerate)
__device__ bool low_altitude(const float* v, int a, int b, int c) {
    const double ux = __dsub_rn(vc(v, b, 0), vc(v, a, 0)), uy = __dsub_rn(vc(v, b, 1), vc(v, a, 1)),
                 uz = __dsub_rn(vc(v, b, 2), vc(v, a, 2));
    const double wx = __dsub_rn(vc(v, c, 0), vc(v, a, 0)), wy = __dsub_rn(vc(v, c, 1), vc(v, a, 1)),
                 wz = __dsub_rn(vc(v, c, 2), vc(v, a, 2));
    const double ex = __dsub_rn(vc(v, c, 0), vc(v, b, 0)), ey = __dsub_rn(vc(v, c, 1), vc(v, b, 1)),
                 ez = __dsub_rn(vc(v, c, 2), vc(v, b, 2));
    const double nx = __dsub_rn(__dmul_rn(uy, wz), __dmul_rn(uz, wy));
    const double ny = __dsub_rn(__dmul_rn(uz, wx), __dmul_rn(ux, wz));
    const double nz = __dsub_rn(__dmul_rn(ux, wy), __dmul_rn(uy, wx));
    const double longest = fmax(fmax(norm3(ux, uy, uz), norm3(ex, ey, ez)), norm3(wx, wy, wz));
    return longest == 0.0 || __ddiv_rn(norm3(nx, ny, nz), longest) <= kMinAltitude;
}

__global__ void __launch_bounds__(256)
mc_face_kernel(const float* __restrict__ verts, const int32_t* __restrict__ faces, int F, const int32_t* __restrict__ rep,
               const uint8_t* __restrict__ finite, uint8_t* cand, unsigned long long* cnt) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const int i0 = faces[3 * (int64_t)f], i1 = faces[3 * (int64_t)f + 1], i2 = faces[3 * (int64_t)f + 2];
    uint8_t ok = 0;
    if (!finite[i0] || !finite[i1] || !finite[i2]) {
        count(cnt, C_NONFINITE);
    } else {
        const int a = rep[i0], b = rep[i1], c = rep[i2];
        if (a == b || b == c || a == c || low_altitude(verts, a, b, c)) count(cnt, C_DEGENERATE);
        else ok = 1;
    }
    cand[f] = ok;
}

__device__ __forceinline__ void sorted_triple(const int32_t* faces, const int32_t* rep, int f, uint32_t& a, uint32_t& b,
                                              uint32_t& c) {
    uint32_t x = rep[faces[3 * (int64_t)f]], y = rep[faces[3 * (int64_t)f + 1]], z = rep[faces[3 * (int64_t)f + 2]];
    if (x > y) { const uint32_t t = x; x = y; y = t; }
    if (y > z) { const uint32_t t = y; y = z; z = t; }
    if (x > y) { const uint32_t t = x; x = y; y = t; }
    a = x; b = y; c = z;
}

__global__ void __launch_bounds__(256)
mc_dup_key_kernel(const int32_t* __restrict__ faces, const int32_t* __restrict__ rep, const int32_t* __restrict__ ids,
                  int n, bool high, unsigned long long* key) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t a, b, c;
    sorted_triple(faces, rep, ids[i], a, b, c);
    key[i] = high ? (unsigned long long)a : ((unsigned long long)b << 32) | c;
}

__global__ void __launch_bounds__(256)
mc_dup_mark_kernel(const int32_t* __restrict__ faces, const int32_t* __restrict__ rep, const int32_t* __restrict__ ids,
                   int n, uint8_t* alive, unsigned long long* cnt) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p == 0 || p >= n) return;
    uint32_t a, b, c, x, y, z;
    sorted_triple(faces, rep, ids[p], a, b, c);
    sorted_triple(faces, rep, ids[p - 1], x, y, z);
    if (a == x && b == y && c == z) {
        alive[ids[p]] = 0;
        count(cnt, C_DUPLICATE);
    }
}

// working faces W [n][3] in the welded (lowest input index) numbering
__global__ void __launch_bounds__(256)
mc_build_work_kernel(const int32_t* __restrict__ faces, const int32_t* __restrict__ rep, const int32_t* __restrict__ ids,
                     int n, int32_t* W) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t f = ids[i];
#pragma unroll
    for (int k = 0; k < 3; ++k) W[3 * (int64_t)i + k] = rep[faces[3 * f + k]];
}

__device__ __forceinline__ int next_he(int h) { return h % 3 == 2 ? h - 2 : h + 1; }

__global__ void __launch_bounds__(256)
mc_halfedge_kernel(const int32_t* __restrict__ W, int n3, unsigned long long* key, int32_t* val) {
    const int h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= n3) return;
    const uint32_t u = W[h], v = W[next_he(h)];
    key[h] = u < v ? ((unsigned long long)u << 32) | v : ((unsigned long long)v << 32) | u;
    val[h] = h;
}

// per undirected edge (run): boundary / two-face / non-manifold counts and the consistency of two-face edges
__global__ void __launch_bounds__(256)
mc_classify_kernel(const int32_t* __restrict__ W, const int32_t* __restrict__ he, const int32_t* __restrict__ rcnt,
                   const int32_t* __restrict__ roff, int R, unsigned long long* cnt) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    const int c = rcnt[r];
    if (c == 1) count(cnt, C_BOUNDARY);
    else if (c > 2) count(cnt, C_NONMANIFOLD);
    else if (W[he[roff[r]]] == W[he[roff[r] + 1]]) count(cnt, C_INCONSISTENT);   // same start vertex: same direction
}

__device__ __forceinline__ void bnd_insert(int32_t* deg, uint32_t* nb, int at, uint32_t entry) {
    const int slot = atomicAdd(deg + at, 1);
    if (slot < 2) nb[2 * (int64_t)at + slot] = entry;
}

__global__ void __launch_bounds__(256)
mc_boundary_kernel(const int32_t* __restrict__ W, const int32_t* __restrict__ he, const int32_t* __restrict__ rcnt,
                   const int32_t* __restrict__ roff, int R, int32_t* deg, uint32_t* nb) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R || rcnt[r] != 1) return;
    const int h = he[roff[r]];
    const int u = W[h], v = W[next_he(h)];
    bnd_insert(deg, nb, u, (uint32_t)v | 0x80000000u);
    bnd_insert(deg, nb, v, (uint32_t)u);
}

// the boundary neighbour of p other than prev, or -1 when p's boundary degree is not 2
__device__ __forceinline__ int bnd_other(const int32_t* deg, const uint32_t* nb, int p, int prev) {
    if (deg[p] != 2) return -1;
    const int a = nb[2 * (int64_t)p] & kIdx, b = nb[2 * (int64_t)p + 1] & kIdx;
    return a == prev ? b : a;
}

// the loop owned by v (v its lowest vertex): length 3 or 4 (else 0), its vertices in walk order v, p[0], p[1], (p[2])
// starting towards v's lower boundary neighbour, and whether the existing face runs v -> p[0]
__device__ int bnd_loop(const int32_t* deg, const uint32_t* nb, int v, int p[3], bool& out) {
    if (deg[v] != 2) return 0;
    const uint32_t e0 = nb[2 * (int64_t)v], e1 = nb[2 * (int64_t)v + 1];
    const uint32_t e = (e0 & kIdx) < (e1 & kIdx) ? e0 : e1;
    out = (e >> 31) != 0;
    p[0] = e & kIdx;
    p[1] = bnd_other(deg, nb, p[0], v);
    if (p[1] < 0) return 0;
    p[2] = bnd_other(deg, nb, p[1], p[0]);
    if (p[2] < 0) return 0;
    if (p[2] == v) return (v < p[0] && v < p[1]) ? 3 : 0;
    const int q = bnd_other(deg, nb, p[2], p[1]);
    return (q == v && v < p[0] && v < p[1] && v < p[2]) ? 4 : 0;
}

__global__ void __launch_bounds__(256)
mc_loop_count_kernel(const int32_t* __restrict__ deg, const uint32_t* __restrict__ nb, int V, int32_t* nfill) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    int p[3];
    bool out;
    const int L = bnd_loop(deg, nb, v, p, out);
    nfill[v] = L == 3 ? 1 : (L == 4 ? 2 : 0);
}

__device__ __forceinline__ void put_face(int32_t* W, int64_t i, int a, int b, int c) {
    W[3 * i] = a; W[3 * i + 1] = b; W[3 * i + 2] = c;
}

// fill faces run opposite to the loop's edges; a quad is split along the diagonal through its lowest vertex v
__global__ void __launch_bounds__(256)
mc_fill_kernel(const int32_t* __restrict__ deg, const uint32_t* __restrict__ nb, int V, const int32_t* __restrict__ foff,
               int base, int32_t* W, unsigned long long* cnt) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    int p[3];
    bool out;
    const int L = bnd_loop(deg, nb, v, p, out);
    if (!L) return;
    count(cnt, C_HOLES);
    const int64_t i = (int64_t)base + foff[v];
    if (out) put_face(W, i, v, p[1], p[0]);
    else put_face(W, i, v, p[0], p[1]);
    if (L == 4) {
        if (out) put_face(W, i + 1, v, p[2], p[1]);
        else put_face(W, i + 1, v, p[1], p[2]);
    }
}

// ---- union-find with parity: word = parent << 1 | parity of this face relative to the parent
__device__ __forceinline__ unsigned long long uf_load(const unsigned long long* par, int x) {
    return *reinterpret_cast<const volatile unsigned long long*>(par + x);
}

// every face its own root, parity 0
__global__ void __launch_bounds__(256) mc_init_parent_kernel(unsigned long long* par, int n) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < n) par[f] = (unsigned long long)f << 1;
}

__device__ int uf_find(unsigned long long* par, int x, int& parity) {
    int acc = 0;
    while (true) {
        const unsigned long long w = uf_load(par, x);
        const int q = (int)(w >> 1);
        if (q == x) { parity = acc; return x; }
        const unsigned long long wq = uf_load(par, q);
        const int g = (int)(wq >> 1);
        // path halving: x points at its grandparent, with the parity of the two steps
        if (g != q) atomicCAS(par + x, w, ((unsigned long long)g << 1) | ((w ^ wq) & 1ull));
        acc ^= (int)(w & 1ull);
        x = q;
    }
}

// rel = 1 when the two faces traverse their shared edge in the same direction (one of them must be reversed)
__device__ __forceinline__ void two_face_edge(const int32_t* W, const int32_t* he, int o, int& f, int& g, int& rel) {
    const int h0 = he[o], h1 = he[o + 1];
    f = h0 / 3; g = h1 / 3;
    rel = W[h0] == W[h1];
}

__global__ void __launch_bounds__(256)
mc_union_kernel(const int32_t* __restrict__ W, const int32_t* __restrict__ he, const int32_t* __restrict__ rcnt,
                const int32_t* __restrict__ roff, int R, unsigned long long* par, uint8_t* has2) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R || rcnt[r] != 2) return;
    int f, g, rel;
    two_face_edge(W, he, roff[r], f, g, rel);
    has2[f] = 1;
    has2[g] = 1;
    while (true) {
        int pf, pg;
        const int rf = uf_find(par, f, pf), rg = uf_find(par, g, pg);
        if (rf == rg) return;
        const int hi = max(rf, rg), lo = min(rf, rg);
        const unsigned long long self = (unsigned long long)hi << 1;
        if (atomicCAS(par + hi, self, ((unsigned long long)lo << 1) | (unsigned long long)(pf ^ pg ^ rel)) == self) return;
    }
}

__global__ void __launch_bounds__(256)
mc_flatten_kernel(unsigned long long* par, int n, int32_t* root, uint8_t* parity) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    int p;
    root[f] = uf_find(par, f, p);
    parity[f] = (uint8_t)p;
}

__global__ void __launch_bounds__(256)
mc_orientable_kernel(const int32_t* __restrict__ W, const int32_t* __restrict__ he, const int32_t* __restrict__ rcnt,
                     const int32_t* __restrict__ roff, int R, const int32_t* __restrict__ root,
                     const uint8_t* __restrict__ parity, uint8_t* nonorient) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R || rcnt[r] != 2) return;
    int f, g, rel;
    two_face_edge(W, he, roff[r], f, g, rel);
    if ((parity[f] ^ parity[g]) != rel) nonorient[root[f]] = 1;
}

// det(v0, v1, v2) = v0 . (v1 x v2), rounded in the oracle's order
__device__ double det3(const float* v, int a, int b, int c) {
    const double cx = __dsub_rn(__dmul_rn(vc(v, b, 1), vc(v, c, 2)), __dmul_rn(vc(v, b, 2), vc(v, c, 1)));
    const double cy = __dsub_rn(__dmul_rn(vc(v, b, 2), vc(v, c, 0)), __dmul_rn(vc(v, b, 0), vc(v, c, 2)));
    const double cz = __dsub_rn(__dmul_rn(vc(v, b, 0), vc(v, c, 1)), __dmul_rn(vc(v, b, 1), vc(v, c, 0)));
    return __dadd_rn(__dadd_rn(__dmul_rn(vc(v, a, 0), cx), __dmul_rn(vc(v, a, 1), cy)), __dmul_rn(vc(v, a, 2), cz));
}

// det of face ids[i] (all faces when ids is null), after the parity flip when parity is given
__global__ void __launch_bounds__(256)
mc_det_kernel(const float* __restrict__ verts, const int32_t* __restrict__ W, const int32_t* __restrict__ ids, int n,
              const uint8_t* __restrict__ parity, double* d) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t f = ids ? ids[i] : i;
    const int a = W[3 * f], b = W[3 * f + 1], c = W[3 * f + 2];
    d[i] = parity && parity[f] ? det3(verts, c, b, a) : det3(verts, a, b, c);
}

// one CTA per segment: lane t adds elements t, t + 256, ... in order, then a halving tree over the lanes
__global__ void __launch_bounds__(kSumThreads)
mc_segment_sum_kernel(const double* __restrict__ d, const int32_t* __restrict__ off, const int32_t* __restrict__ cnt,
                      int n_single, double* out) {
    __shared__ double s[kSumThreads];
    const int seg = blockIdx.x;
    const int o = off ? off[seg] : 0, n = cnt ? cnt[seg] : n_single;
    double acc = 0.0;
    for (int i = threadIdx.x; i < n; i += kSumThreads) acc = __dadd_rn(acc, d[o + i]);
    s[threadIdx.x] = acc;
    __syncthreads();
    for (int h = kSumThreads / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) s[threadIdx.x] = __dadd_rn(s[threadIdx.x], s[threadIdx.x + h]);
        __syncthreads();
    }
    if (threadIdx.x == 0) out[seg] = s[0];
}

__global__ void __launch_bounds__(256)
mc_component_kernel(const int32_t* __restrict__ seg_root, const double* __restrict__ seg_sum, int nseg,
                    const uint8_t* __restrict__ nonorient, uint8_t* flip, unsigned long long* cnt) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= nseg) return;
    const int r = seg_root[s];
    if (nonorient[r]) count(cnt, C_NONORIENT);
    else flip[r] = seg_sum[s] < 0.0;
}

__global__ void __launch_bounds__(256)
mc_reverse_kernel(int32_t* W, int n, const uint8_t* __restrict__ has2, const int32_t* __restrict__ root,
                  const uint8_t* __restrict__ parity, const uint8_t* __restrict__ nonorient,
                  const uint8_t* __restrict__ flip, unsigned long long* cnt) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n || !has2[f]) return;
    const int r = root[f];
    if (nonorient[r] || !(parity[f] ^ flip[r])) return;
    const int32_t t = W[3 * (int64_t)f];
    W[3 * (int64_t)f] = W[3 * (int64_t)f + 2];
    W[3 * (int64_t)f + 2] = t;
    count(cnt, C_REVERSED);
}

__global__ void __launch_bounds__(256) mc_mark_used_kernel(const int32_t* __restrict__ W, int n3, int32_t* used) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n3) used[W[i]] = 1;
}

__global__ void __launch_bounds__(256)
mc_emit_kernel(const float* __restrict__ verts, int V, const int32_t* __restrict__ used, const int32_t* __restrict__ newidx,
               const int32_t* __restrict__ W, int n3, float* verts_out, int32_t* faces_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < V && used[i]) {
#pragma unroll
        for (int k = 0; k < 3; ++k) verts_out[3 * (int64_t)newidx[i] + k] = verts[3 * (int64_t)i + k];
    }
    if (i < n3) faces_out[i] = newidx[W[i]];
}

struct MaxOp {
    __device__ __forceinline__ int32_t operator()(int32_t a, int32_t b) const { return a > b ? a : b; }
};

// the undirected edges of the working faces W [n][3]: sorted half-edges he, runs (count, offset)
struct Edges {
    int32_t *he, *rcnt, *roff;
    int R;
    long long boundary, nonmanifold, inconsistent;
};

// its buffers are the workspace slots from `at` on, so that every call reuses the same ones
Edges classify(Workspace& ws, size_t at, const int32_t* W, int n, cudaStream_t st) {
    const size_t resume = ws.mark();
    ws.rewind(at);
    Edges e{};
    const int n3 = 3 * n;
    unsigned long long* c = ws.get<unsigned long long>(C_COUNT);
    auto* key = ws.get<unsigned long long>(n3);
    auto* key_s = ws.get<unsigned long long>(n3);
    int32_t* val = ws.get<int32_t>(n3);
    e.he = ws.get<int32_t>(n3);
    auto* ukey = ws.get<unsigned long long>(n3);
    e.rcnt = ws.get<int32_t>(n3);
    e.roff = ws.get<int32_t>(n3);
    int* d_num = ws.get<int>(1);
    ws.rewind(std::max(resume, ws.mark()));
    P2S_CUDA(cudaMemsetAsync(c, 0, C_COUNT * sizeof(unsigned long long), st));
    if (n == 0) return e;
    P2S_LAUNCH(mc_halfedge_kernel, grid1d(n3, 256), 256, 0, st, W, n3, key, val);
    cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, key, key_s, val, e.he, n3, 0, 64, st); });
    cub_run(ws, 1, [&](void* t, size_t& b) {
        return cub::DeviceRunLengthEncode::Encode(t, b, key_s, ukey, e.rcnt, d_num, n3, st);
    });
    e.R = read_back(d_num, 1, st)[0];
    cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, e.rcnt, e.roff, e.R, st); });
    P2S_LAUNCH(mc_classify_kernel, grid1d(e.R, 256), 256, 0, st, W, e.he, e.rcnt, e.roff, e.R, c);
    const auto h = read_back(c, C_COUNT, st);
    e.boundary = (long long)h[C_BOUNDARY];
    e.nonmanifold = (long long)h[C_NONMANIFOLD];
    e.inconsistent = (long long)h[C_INCONSISTENT];
    return e;
}

// the fixed-order sum of mc_segment_sum_kernel over d [n]
double fixed_sum(Workspace& ws, const double* d, int n, cudaStream_t st) {
    double* out = ws.get<double>(1);
    P2S_LAUNCH(mc_segment_sum_kernel, 1, kSumThreads, 0, st, d, nullptr, nullptr, n, out);
    return read_back(out, 1, st)[0];
}

}  // namespace

void mesh_clean(const float* verts, int64_t V64, const int32_t* faces, int64_t F64, float* verts_out, int64_t vcap,
                int32_t* faces_out, int64_t fcap, p2s_clean_report* rep_out, cudaStream_t st) {
    P2S_CHECK(V64 >= 0 && F64 >= 0 && vcap >= 0 && fcap >= 0, "negative size");
    P2S_CHECK(V64 < INT32_MAX && 2 * F64 < INT32_MAX / 3, "mesh too large for int32 indices");
    const int V = (int)V64, F = (int)F64;
    static thread_local std::vector<Workspace> t_ws;
    Workspace& ws = for_device(t_ws).begin(st);
    p2s_clean_report R{};
    R.vertices_in = V;
    R.faces_in = F;
    unsigned long long* cnt = ws.get<unsigned long long>(C_COUNT);
    P2S_CUDA(cudaMemsetAsync(cnt, 0, C_COUNT * sizeof(unsigned long long), st));

    // 1. input checks and weld keys
    long long *kx = ws.get<long long>(V), *ky = ws.get<long long>(V), *kz = ws.get<long long>(V);
    long long* kt = ws.get<long long>(V);
    uint8_t* finite = ws.get<uint8_t>(V);
    int32_t *ord0 = ws.get<int32_t>(V), *ord1 = ws.get<int32_t>(V);
    if (F > 0) P2S_LAUNCH(mc_index_check_kernel, grid1d(3 * (int64_t)F, 256), 256, 0, st, faces, 3 * (int64_t)F, V64, cnt);
    if (V > 0) P2S_LAUNCH(mc_vertex_key_kernel, grid1d(V, 256), 256, 0, st, verts, V, kx, ky, kz, finite, ord0, cnt);
    std::vector<unsigned long long> h = read_back(cnt, C_COUNT, st);
    P2S_CHECK(h[C_BAD_INDEX] == 0, "face index outside [0, V)");
    P2S_CHECK(h[C_OVERFLOW] == 0, "finite vertex coordinate with |x| >= 9e10 (weld key overflows int64)");

    // 2. weld: stable sorts by z, y, x key leave equal keys adjacent in ascending index order
    int32_t* rep = ws.get<int32_t>(V);
    if (V > 0) {
        long long* kg = ws.get<long long>(V);   // keys gathered into the current order
        cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, kz, kt, ord0, ord1, V, 0, 64, st); });
        P2S_LAUNCH(mc_gather_kernel<long long>, grid1d(V, 256), 256, 0, st, ky, ord1, V, kg);
        cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, kg, kt, ord1, ord0, V, 0, 64, st); });
        P2S_LAUNCH(mc_gather_kernel<long long>, grid1d(V, 256), 256, 0, st, kx, ord0, V, kg);
        cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, kg, kt, ord0, ord1, V, 0, 64, st); });
        int32_t *headpos = ws.get<int32_t>(V), *runstart = ws.get<int32_t>(V);
        P2S_LAUNCH(mc_weld_head_kernel, grid1d(V, 256), 256, 0, st, ord1, V, kx, ky, kz, finite, headpos, cnt);
        cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceScan::InclusiveScan(t, b, headpos, runstart, MaxOp(), V, st); });
        P2S_LAUNCH(mc_weld_rep_kernel, grid1d(V, 256), 256, 0, st, ord1, runstart, V, rep);
    }

    // 3. non-finite, degenerate and duplicate faces
    uint8_t* alive = ws.get<uint8_t>(F);
    int32_t *ids0 = ws.get<int32_t>(F), *ids1 = ws.get<int32_t>(F);
    int* d_num = ws.get<int>(1);
    cub::CountingInputIterator<int32_t> counting(0);
    int A = 0;
    if (F > 0) {
        P2S_LAUNCH(mc_face_kernel, grid1d(F, 256), 256, 0, st, verts, faces, F, rep, finite, alive, cnt);
        cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, counting, alive, ids0, d_num, F, st); });
        const int C = read_back(d_num, 1, st)[0];
        if (C > 1) {
            auto *k0 = ws.get<unsigned long long>(C), *k1 = ws.get<unsigned long long>(C);
            P2S_LAUNCH(mc_dup_key_kernel, grid1d(C, 256), 256, 0, st, faces, rep, ids0, C, false, k0);
            cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, k0, k1, ids0, ids1, C, 0, 64, st); });
            P2S_LAUNCH(mc_dup_key_kernel, grid1d(C, 256), 256, 0, st, faces, rep, ids1, C, true, k0);
            cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, k0, k1, ids1, ids0, C, 0, 32, st); });
            P2S_LAUNCH(mc_dup_mark_kernel, grid1d(C, 256), 256, 0, st, faces, rep, ids0, C, alive, cnt);
            cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, counting, alive, ids0, d_num, F, st); });
            A = read_back(d_num, 1, st)[0];
        } else {
            A = C;
        }
    }
    h = read_back(cnt, C_COUNT, st);
    R.merged_vertices = V - (int64_t)h[C_HEADS];
    R.nonfinite_faces = (int64_t)h[C_NONFINITE];
    R.degenerate_faces = (int64_t)h[C_DEGENERATE];
    R.duplicate_faces = (int64_t)h[C_DUPLICATE];

    // working faces: the A survivors in input order, then at most A fill faces (a face borders at most one fillable
    // loop, and a loop gets at most one fill face per bordering face)
    int32_t* W = ws.get<int32_t>(6 * (size_t)std::max(A, 1));
    if (A > 0) P2S_LAUNCH(mc_build_work_kernel, grid1d(A, 256), 256, 0, st, faces, rep, ids0, A, W);

    // 4.-5. classify, fill holes, classify again
    const size_t classify_slots = ws.mark();
    Edges e = classify(ws, classify_slots, W, A, st);
    int n = A;
    if (e.boundary > 0) {
        int32_t* deg = ws.get<int32_t>(V);
        uint32_t* nb = ws.get<uint32_t>(2 * (size_t)V);
        int32_t *nfill = ws.get<int32_t>(V), *foff = ws.get<int32_t>(V);
        P2S_CUDA(cudaMemsetAsync(deg, 0, (size_t)V * sizeof(int32_t), st));
        P2S_LAUNCH(mc_boundary_kernel, grid1d(e.R, 256), 256, 0, st, W, e.he, e.rcnt, e.roff, e.R, deg, nb);
        P2S_LAUNCH(mc_loop_count_kernel, grid1d(V, 256), 256, 0, st, deg, nb, V, nfill);
        cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, nfill, foff, V, st); });
        const int added = read_back(foff + (V - 1), 1, st)[0] + read_back(nfill + (V - 1), 1, st)[0];
        P2S_CHECK(added <= A, "internal error: more fill faces than faces");
        if (added > 0) {
            P2S_LAUNCH(mc_fill_kernel, grid1d(V, 256), 256, 0, st, deg, nb, V, foff, A, W, cnt);
            n = A + added;
            e = classify(ws, classify_slots, W, n, st);
        }
    }
    h = read_back(cnt, C_COUNT, st);
    R.holes_filled = (int64_t)h[C_HOLES];
    R.faces_added = n - A;
    R.boundary_edges = e.boundary;
    R.nonmanifold_edges = e.nonmanifold;
    R.watertight_before = e.boundary == 0 && e.nonmanifold == 0;
    R.winding_consistent_before = e.inconsistent == 0;

    // 6. orientation of every component over two-face edges, only when the winding is inconsistent
    if (e.inconsistent > 0) {
        auto* par = ws.get<unsigned long long>(n);
        uint8_t *has2 = ws.get<uint8_t>(n), *parity = ws.get<uint8_t>(n);
        uint8_t *nonorient = ws.get<uint8_t>(n), *flip = ws.get<uint8_t>(n);
        int32_t* root = ws.get<int32_t>(n);
        P2S_CUDA(cudaMemsetAsync(has2, 0, n, st));
        P2S_CUDA(cudaMemsetAsync(nonorient, 0, n, st));
        P2S_CUDA(cudaMemsetAsync(flip, 0, n, st));
        P2S_LAUNCH(mc_init_parent_kernel, grid1d(n, 256), 256, 0, st, par, n);
        P2S_LAUNCH(mc_union_kernel, grid1d(e.R, 256), 256, 0, st, W, e.he, e.rcnt, e.roff, e.R, par, has2);
        P2S_LAUNCH(mc_flatten_kernel, grid1d(n, 256), 256, 0, st, par, n, root, parity);
        P2S_LAUNCH(mc_orientable_kernel, grid1d(e.R, 256), 256, 0, st, W, e.he, e.rcnt, e.roff, e.R, root, parity, nonorient);
        // faces with a two-face edge, grouped by component (stable: ascending face index inside)
        int32_t *sel = ws.get<int32_t>(n), *sel_s = ws.get<int32_t>(n);
        cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, counting, has2, sel, d_num, n, st); });
        const int m = read_back(d_num, 1, st)[0];
        int32_t *sroot = ws.get<int32_t>(m), *sroot_s = ws.get<int32_t>(m);
        P2S_LAUNCH(mc_gather_kernel<int32_t>, grid1d(m, 256), 256, 0, st, root, sel, m, sroot);
        cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceRadixSort::SortPairs(t, b, sroot, sroot_s, sel, sel_s, m, 0, 32, st); });
        int32_t *segroot = ws.get<int32_t>(m), *segcnt = ws.get<int32_t>(m), *segoff = ws.get<int32_t>(m);
        cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceRunLengthEncode::Encode(t, b, sroot_s, segroot, segcnt, d_num, m, st); });
        const int nseg = read_back(d_num, 1, st)[0];
        cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, segcnt, segoff, nseg, st); });
        double* det = ws.get<double>(m);
        double* segsum = ws.get<double>(nseg);
        P2S_LAUNCH(mc_det_kernel, grid1d(m, 256), 256, 0, st, verts, W, sel_s, m, parity, det);
        P2S_CHECK(nseg > 0, "internal error: inconsistent winding without a two-face edge");
        P2S_LAUNCH(mc_segment_sum_kernel, nseg, kSumThreads, 0, st, det, segoff, segcnt, 0, segsum);
        P2S_LAUNCH(mc_component_kernel, grid1d(nseg, 256), 256, 0, st, segroot, segsum, nseg, nonorient, flip, cnt);
        P2S_LAUNCH(mc_reverse_kernel, grid1d(n, 256), 256, 0, st, W, n, has2, root, parity, nonorient, flip, cnt);
        h = read_back(cnt, C_COUNT, st);
        R.components = nseg;
        R.nonorientable_components = (int64_t)h[C_NONORIENT];
        R.faces_reversed = (int64_t)h[C_REVERSED];
        e = classify(ws, classify_slots, W, n, st);
    }
    R.watertight = e.boundary == 0 && e.nonmanifold == 0;
    R.winding_consistent = e.inconsistent == 0;

    // 7. drop unreferenced vertices; signed volume of the output
    int32_t *used = ws.get<int32_t>(V), *newidx = ws.get<int32_t>(V);
    int vout = 0;
    if (V > 0) {
        P2S_CUDA(cudaMemsetAsync(used, 0, (size_t)V * sizeof(int32_t), st));
        if (n > 0) P2S_LAUNCH(mc_mark_used_kernel, grid1d(3 * (int64_t)n, 256), 256, 0, st, W, 3 * n, used);
        cub_run(ws, 1, [&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, used, newidx, V, st); });
        vout = read_back(newidx + (V - 1), 1, st)[0] + read_back(used + (V - 1), 1, st)[0];
    }
    R.vertices_out = vout;
    R.faces_out = n;
    R.unreferenced_vertices = V - R.merged_vertices - vout;
    P2S_CHECK(vout <= vcap, "vcap too small for the cleaned mesh (vcap >= V always suffices)");
    P2S_CHECK(n <= fcap, "fcap too small for the cleaned mesh (fcap >= 2 F always suffices)");
    P2S_CHECK((verts_out || vout == 0) && (faces_out || n == 0), "null output");
    if (n > 0) {
        double* det = ws.get<double>(n);
        P2S_LAUNCH(mc_det_kernel, grid1d(n, 256), 256, 0, st, verts, W, nullptr, n, nullptr, det);
        R.volume = fixed_sum(ws, det, n, st) / 6.0;
        P2S_LAUNCH(mc_emit_kernel, grid1d(std::max(V, 3 * n), 256), 256, 0, st, verts, V, used, newidx, W, 3 * n, verts_out,
                   faces_out);
        P2S_CUDA(cudaStreamSynchronize(st));
    }
    *rep_out = R;
}

}  // namespace p2s
