// Shared helpers for libp2s_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <stdexcept>
#include <algorithm>
#include <atomic>
#include <set>
#include <vector>

#include "../../include/p2s_b200.h"

namespace p2s {

extern thread_local std::string g_last_error;
extern std::atomic<uint64_t> g_launches;

struct Error : std::runtime_error {
    using std::runtime_error::runtime_error;
};

#define P2S_CUDA(call)                                                                             \
    do {                                                                                           \
        cudaError_t _e = (call);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            char _buf[512];                                                                        \
            snprintf(_buf, sizeof(_buf), "%s:%d: %s failed: %s", __FILE__, __LINE__, #call,       \
                     cudaGetErrorString(_e));                                                      \
            throw ::p2s::Error(_buf);                                                              \
        }                                                                                          \
    } while (0)

#define P2S_CHECK(cond, msg)                                                                       \
    do {                                                                                           \
        if (!(cond)) {                                                                             \
            char _buf[512];                                                                        \
            snprintf(_buf, sizeof(_buf), "%s:%d: check failed (%s): %s", __FILE__, __LINE__,      \
                     #cond, msg);                                                                  \
            throw ::p2s::Error(_buf);                                                              \
        }                                                                                          \
    } while (0)

// every kernel launch goes through this so that p2s_launch_count() is honest
#define P2S_LAUNCH(kernel, grid, block, smem, stream, ...)                                         \
    do {                                                                                           \
        kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);                                \
        ::p2s::g_launches.fetch_add(1, std::memory_order_relaxed);                                 \
        P2S_CUDA(cudaGetLastError());                                                              \
    } while (0)

template <class F>
static inline int guarded(F&& f) {
    try {
        f();
        return 0;
    } catch (const std::exception& e) {
        g_last_error = e.what();
        return 1;
    }
}

static inline int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Optional coarse stage timing (env P2S_STAGE_TIMING=1): synchronises the stream around every stage and
// accumulates host wall-clock per label; printed by p2s_model_destroy.  Diagnostics only.
struct StageTimer {
    static bool enabled();
    static void add(const char* label, double ms);
    static void report();
};
struct StageScope {
    const char* label; cudaStream_t st; double t0 = 0.0; bool on;
    StageScope(const char* l, cudaStream_t s);
    ~StageScope();
};

// grow-only device scratch buffer.  `capturing`: the caller's stream is capturing a CUDA graph, which then holds p, so p
// may not move now and is never freed later (it stays allocated for the rest of the process).
struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
    bool captured = false;
    void* get(size_t need, bool capturing = false) {
        if (need > bytes) {
            P2S_CHECK(!capturing, "library scratch would have to grow while the stream is capturing a CUDA graph: make an "
                                  "eager call of the same size first");
            if (p && !captured) P2S_CUDA(cudaFree(p));
            p = nullptr;
            captured = false;
            size_t want = need + need / 8;
            P2S_CUDA(cudaMalloc(&p, want));
            bytes = want;
        }
        captured = captured || capturing;
        return p;
    }
    template <class T>
    T* as(size_t count) { return reinterpret_cast<T*>(get(count * sizeof(T))); }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        bytes = 0;
    }
};

// v[current device]; v is sized to the device count on first use
template <class T>
T& for_device(std::vector<T>& v) {
    if (v.empty()) {
        int n = 0;
        P2S_CUDA(cudaGetDeviceCount(&n));
        v.resize(n);
    }
    int d = 0;
    P2S_CUDA(cudaGetDevice(&d));
    return v.at(d);
}

// Library scratch (the rules are in include/p2s_b200.h, "Scratch memory").  Every entry point keeps one
// `static thread_local std::vector<Workspace>` and starts each call with `for_device(ws).begin(st)`.  Buffers are handed
// out in request order, so the same sequence of requests reuses the same buffers; mark()/rewind() let a helper called
// more than once reuse its own slots.  CUB's temporary storage is one more grow-only buffer (cub_run).
struct Workspace {
    std::vector<DevBuf> bufs;
    DevBuf cub;
    size_t next = 0;
    cudaStream_t st = nullptr;

    Workspace& begin(cudaStream_t s) {
        next = 0;
        st = s;
        return *this;
    }
    void* grow(DevBuf& b, size_t bytes) {
        cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
        P2S_CUDA(cudaStreamIsCapturing(st, &cs));
        return b.get(bytes, cs != cudaStreamCaptureStatusNone);
    }
    template <class T>
    T* get(int64_t count) {
        if (next == bufs.size()) bufs.emplace_back();
        return reinterpret_cast<T*>(grow(bufs[next++], (size_t)std::max<int64_t>(count, 1) * sizeof(T)));
    }
    size_t mark() const { return next; }
    void rewind(size_t m) { next = m; }
};

// runs a CUB device algorithm: size query, grow the workspace's CUB storage, call.  `counted`: what the call adds to
// p2s_launch_count(), whatever CUB launches.
template <class Fn>
void cub_run(Workspace& ws, int counted, Fn fn) {
    size_t bytes = 0;
    P2S_CUDA(fn(nullptr, bytes));
    P2S_CUDA(fn(ws.grow(ws.cub, std::max<size_t>(bytes, 16)), bytes));
    g_launches.fetch_add(counted, std::memory_order_relaxed);
}

// copies n values to the host and waits for the stream
template <class T>
std::vector<T> read_back(const T* dev, size_t n, cudaStream_t st) {
    std::vector<T> h(n);
    P2S_CUDA(cudaMemcpyAsync(h.data(), dev, n * sizeof(T), cudaMemcpyDeviceToHost, st));
    P2S_CUDA(cudaStreamSynchronize(st));
    return h;
}

static inline unsigned grid1d(int64_t n, int threads) { return (unsigned)cdiv(std::max<int64_t>(n, 1), threads); }

static inline int sm_count() {   // of the current device
    int d = 0, n = 0;
    P2S_CUDA(cudaGetDevice(&d));
    P2S_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d));
    return n;
}

// raises the kernel's dynamic shared-memory limit to `bytes` on the current device, once per device and thread
template <class K>
void set_smem_attr_once(K* kernel, size_t bytes) {
    static thread_local std::set<std::pair<const void*, int>> done;   // (kernel, device)
    int d = 0;
    P2S_CUDA(cudaGetDevice(&d));
    if (done.count({(const void*)kernel, d})) return;
    P2S_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    done.insert({(const void*)kernel, d});
}

// true when the environment variable starts with '1'; call sites that read it once keep it in a static
static inline bool env_flag(const char* name) {
    const char* e = getenv(name);
    return e && e[0] == '1';
}

// per-cloud cell index (device pointers): the cloud binned into kCloudGrid^3 cells of its bounding box.  Built by
// cloud_index_build (assemble.cu) for the weighted sub-sampler; the neighbour search of normals.cu walks it too.
constexpr int kCloudGrid = 12;
struct CloudIndex {
    const float* meta;      // [6] bounding-box low corner, cells per unit length
    const float* spts;      // [N,3] points in cell order
    const int32_t* perm;    // [N]   original id of sorted point i
    const int32_t* start;   // [C+1] first sorted point of each cell
    const float* cbox;      // [C,6] tight bounding box of each cell's points
};
const CloudIndex* cloud_index_build(const float* pts, int64_t N, cudaStream_t st);

// ---- Philox4x32-10 (Salmon et al. 2011), counter-based: (key, counter) -> 4 x u32 ----
__host__ __device__ inline void philox4x32_10(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1,
                                              uint32_t c2, uint32_t c3, uint32_t out[4]) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        uint64_t p0 = (uint64_t)M0 * c0, p1 = (uint64_t)M1 * c2;
        uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
        uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
        uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += W0; k1 += W1;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

}  // namespace p2s
