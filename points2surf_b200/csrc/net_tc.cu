// Tensor-core implementation of PointsToSurfModel.forward (source/points_to_surf_model.py:296-352) for sm_90a.
//
// The per-point Conv1d(k=1) stacks (98 % of the FLOPs, SURVEY.md section 2a) run as wgmma tiles with fp16
// operands / fp32 accumulation in registers; the three dependent max-reductions of the vanilla network become three
// launches of ONE kernel (`pointnet_pass_kernel`):
//   pass A  QSTN        : x(1300 pts) -> 64 (fp32 FMA) -> 128 -> 1024, max          (model.py:100-107)
//   pass B  STN64       : x -> 64 -> 64 | 64 -> 128 -> 1024, max                     (model.py:190-191,41-48)
//   pass C  final       : x -> 64 -> 64 | (W1*T) 64 -> 128 -> 1024 (no ReLU), max    (model.py:190-212)
// The quaternion rotation is folded into the first layer's weights per query (W0*R), the 64x64 feature
// transform into conv1's weights per query (W1*T), both exactly as in the fp32 path up to operation order.
//
// Tile = 64 points of one query (segments are padded with a duplicate of their first point: max-invariant).
// Every layer after the first: M = 64 points, A operand = activations in registers (the accumulator fragment of one
// layer, packed to fp16 pairs, is the A fragment of the next), B operand = weights in smem.  The big layer 128 -> 1024
// runs as m64n128 per 128-channel chunk with B = the resident W3 chunk, so the activations never go through shared
// memory; D[point][channel], and the max over points is a max over accumulator rows (in-thread, then a shuffle
// reduce-scatter across the warp, then across the 4 warps once per query).  Each CTA owns 512 of the 1024 channels
// (its half of W3, 128 KB fp16, stays resident in shared memory); CTA 2j and 2j+1 stream the same queries.
//
// Each warpgroup of the CTA streams its own queries (qi = wg, wg + 2, ...) through all layers; the two warpgroups
// interleave on the SM, so one's FMA / epilogue work overlaps the other's tensor-core work.
//
// The small per-query FC tails between the passes run on the split-precision FC kernel (fc_tc.cu).
#include "model.cuh"
#include "tc_ptx.cuh"

namespace p2s {

using namespace ptx;

namespace {

constexpr int kTile = 64;                       // points per tile (M of every tensor-core layer)
constexpr int kWG = 2;                          // warpgroups per CTA
constexpr int kThreads = 128 * kWG;
// shared memory map (bytes).  PRECISE = split-precision variant used for the guard-band recompute: every fp16
// operand x is carried as x_hi + x_lo and every product is evaluated as a_hi*b_hi + a_lo*b_hi + a_hi*b_lo (three MMAs
// per k-step, ~2^-22 relative), so the images are twice as large and a CTA owns two 128-channel chunks instead of four.
template <bool PRECISE>
struct Cfg {
    static constexpr int kChunks = PRECISE ? 2 : 4;                  // 128-channel chunks of the big layer per CTA
    static constexpr int kSplit = 8 / kChunks;                       // CTAs that share one query stream
    static constexpr uint32_t kChunkBytes = PRECISE ? 65536u : 32768u;   // W3 chunk image (hi [+ lo])
    static constexpr uint32_t kW3Bytes = kChunks * kChunkBytes;
    static constexpr uint32_t kMidScale = PRECISE ? 2u : 1u;
    static constexpr uint32_t kMidBytes = (8192u + 8192u + 16384u) * kMidScale;
    static constexpr uint32_t kPerqBytes = PRECISE ? 16384u : 8192u; // per-query conv1*(T+I) image
    static constexpr uint32_t kRedBytes = 4u * kChunks * 128u * 4u;  // end of query: [warp][channel] maxima, aliases perq
    static constexpr uint32_t kOffMid = kW3Bytes;
    // per warpgroup: the per-query conv1 image, (W0*R)^T [3][64] fp32
    static constexpr uint32_t kWgWq = kPerqBytes;
    static constexpr uint32_t kWgBytes = kWgWq + 192 * 4;
    static constexpr uint32_t kOffWg = kOffMid + kMidBytes;
    static constexpr uint32_t kOffBias = kOffWg + kWG * kWgBytes;     // [256] mid biases back to back, [64] first-layer bias
    static constexpr uint32_t kSmemBytes = kOffBias + 320 * 4;
};
static_assert(Cfg<false>::kSmemBytes <= 232448 && Cfg<true>::kSmemBytes <= 232448, "shared memory budget");
static_assert(Cfg<false>::kRedBytes <= Cfg<false>::kPerqBytes && Cfg<true>::kRedBytes <= Cfg<true>::kPerqBytes, "reduction scratch");

struct Seg {
    const float* ptr;   // [B, n, 3]
    int n;              // real points per query
    int tiles;          // ceil(n / kTile)
    int center;         // subtract the query point (model.py:303)
};

struct PassParams {
    Seg seg[2];
    const float* query;        // [B,3]
    const float* R;            // [B,9] rotation folded into W0, or null
    int tiles_per_query;
    int B;
    const float* W0;           // [64,3]
    const float* b0;           // [64]
    int num_mid;               // 1 or 3: 64 -> 128, or 64 -> 64 -> 64 -> 128
    int mid_N[3];              // output channels of each mid layer
    const uint8_t* mid_img[3]; // packed fp16 operand images (K-major, LBO 128, SBO 1024)
    const float* mid_bias[3];
    int perq_layer;            // index of the mid layer with per-query weights, or -1
    const uint8_t* perq_img;   // [B] x 8192 B (precise: hi | lo, 16384 B)
    const uint8_t* w3_img;     // [8 chunks][32768 B] (precise: [8][hi | lo])  (K-major, LBO 128, SBO 2048)
    float* out;                // [B,1024] raw max (bias / ReLU applied by the consumer: the FC kernel's producers add it on load)
};

// relu(a), relu(b) -> packed fp16x2 (low half = a), saturating
__device__ __forceinline__ uint32_t pack_relu(float a, float b) {
    uint32_t r;
    asm("cvt.rn.relu.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    return r;
}
// split-precision variant: hi = fp16(relu(x)), lo = fp16(relu(x) - hi)
__device__ __forceinline__ void pack_relu_split(float a, float b, uint32_t& hi, uint32_t& lo) {
    hi = pack_relu(a, b);
    const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi));
    lo = pack_half2(fmaxf(a, 0.f) - hf.x, fmaxf(b, 0.f) - hf.y);
}
template <bool PRECISE>
__device__ __forceinline__ void pack_act(float a, float b, uint32_t& hi, uint32_t& lo) {
    if (PRECISE) pack_relu_split(a, b, hi, lo);
    else hi = pack_relu(a, b);
}

// one k16 step of a mid layer: D (+)= A (registers) * W^T; precise: a_lo*w_hi + a_hi*w_lo + a_hi*w_hi (small terms first)
template <bool PRECISE, int R>
__device__ __forceinline__ void mid_mma(float (&d)[R], const uint32_t (&a)[4], const uint32_t (&al)[4], uint64_t w, uint64_t w_lo, uint32_t acc) {
    if (R == 32) {
        auto& d32 = reinterpret_cast<float (&)[32]>(d);
        if (PRECISE) { wgmma_rs_n64(d32, al, w, acc); wgmma_rs_n64(d32, a, w_lo, 1); wgmma_rs_n64(d32, a, w, 1); }
        else wgmma_rs_n64(d32, a, w, acc);
    } else {
        auto& d64 = reinterpret_cast<float (&)[64]>(d);
        if (PRECISE) { wgmma_rs_n128(d64, al, w, acc); wgmma_rs_n128(d64, a, w_lo, 1); wgmma_rs_n128(d64, a, w, 1); }
        else wgmma_rs_n128(d64, a, w, acc);
    }
}

// epilogue of a mid layer: m64nN accumulator + bias, ReLU, fp16 pairs -> the A fragments of the next layer's N/16 k-steps
template <bool PRECISE, int R, int KL>
__device__ __forceinline__ void pack_acc(const float (&d)[R], const float* bias, int q4, uint32_t (&a)[R / 8][4], uint32_t (&al)[R / 8][KL]) {
#pragma unroll
    for (int j = 0; j < R / 4; ++j) {
        const float2 bb = *reinterpret_cast<const float2*>(bias + 8 * j + 2 * q4);
        pack_act<PRECISE>(d[4 * j] + bb.x, d[4 * j + 1] + bb.y, a[j >> 1][(j & 1) * 2], al[j >> 1][PRECISE ? (j & 1) * 2 : 0]);
        pack_act<PRECISE>(d[4 * j + 2] + bb.x, d[4 * j + 3] + bb.y, a[j >> 1][(j & 1) * 2 + 1], al[j >> 1][PRECISE ? (j & 1) * 2 + 1 : 0]);
    }
}

// one step of a butterfly max reduce-scatter between lanes l and l ^ S: each keeps m[0 .. S) for the half of m[0 .. 2S)
// selected by its lane bit S, folded with the partner's values of that half
template <int S>
__device__ __forceinline__ void max_halve(float (&m)[32], int lane) {
    const bool up = (lane & S) != 0;
#pragma unroll
    for (int i = 0; i < S; ++i) {
        const float send = up ? m[i] : m[i + S], keep = up ? m[i + S] : m[i];
        m[i] = fmaxf(keep, __shfl_xor_sync(0xffffffffu, send, S));
    }
}

template <bool PRECISE>
__global__ void __launch_bounds__(kThreads, 1) pointnet_pass_kernel(const PassParams p) {
    using C = Cfg<PRECISE>;
    constexpr int kL = PRECISE ? 4 : 1;
    extern __shared__ __align__(1024) uint8_t smem[];
    float* s_bias = reinterpret_cast<float*>(smem + C::kOffBias);
    const int tid = threadIdx.x, wg = tid >> 7, t = tid & 127, lane = tid & 31, q4 = lane & 3;
    const int r0 = (t >> 5) * 16 + (lane >> 2);                          // fragment rows r0, r0 + 8
    const int part = blockIdx.x % C::kSplit;                             // which 128-channel chunks this CTA owns
    const int stream = blockIdx.x / C::kSplit, nstreams = gridDim.x / C::kSplit;
    const int nq = (p.B > stream) ? (p.B - stream + nstreams - 1) / nstreams : 0;   // queries of this CTA
    const int tpq = p.tiles_per_query;
    uint32_t mid_off[3] = {0, 0, 0};
    {
        uint32_t o = 0;
        for (int l = 0; l < p.num_mid; ++l) { mid_off[l] = o; o += (uint32_t)p.mid_N[l] * 128u * C::kMidScale; }
    }

    // ---- resident weights: this CTA's W3 chunks, the mid layers shared by every query, the biases
    if (nq > 0) {
        const uint4* src = reinterpret_cast<const uint4*>(p.w3_img + (size_t)part * C::kW3Bytes);
        uint4* dst = reinterpret_cast<uint4*>(smem);
        for (uint32_t i = tid; i < C::kW3Bytes / 16; i += kThreads) dst[i] = src[i];
        for (int l = 0; l < p.num_mid; ++l) {
            if (l == p.perq_layer) continue;
            const uint4* s = reinterpret_cast<const uint4*>(p.mid_img[l]);
            uint4* d = reinterpret_cast<uint4*>(smem + C::kOffMid + mid_off[l]);
            for (uint32_t i = tid; i < (uint32_t)p.mid_N[l] * 8u * C::kMidScale; i += kThreads) d[i] = s[i];
        }
    }
    {
        int off = 0;
        for (int l = 0; l < p.num_mid; ++l) {
            for (int i = tid; i < p.mid_N[l]; i += kThreads) s_bias[off + i] = p.mid_bias[l][i];
            off += p.mid_N[l];
        }
        for (int i = tid; i < 64; i += kThreads) s_bias[256 + i] = p.b0[i];
    }
    fence_proxy_async_smem();
    __syncthreads();

    uint8_t* wsm = smem + C::kOffWg + wg * C::kWgBytes;
    uint8_t* perq = wsm;
    float* red = reinterpret_cast<float*>(perq);                          // [4 warps][kChunks * 128 channels]
    float* wq = reinterpret_cast<float*>(wsm + C::kWgWq);                 // [3][64]: rows of (W0*R)^T
    const float* s_b0 = s_bias + 256;
    const uint32_t bar_id = 1 + (uint32_t)wg;
    auto wg_sync = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory"); };
    const uint64_t dsc_w3 = make_smem_desc(smem_u32(smem), 128, 2048);   // N = 128 channels of a chunk, K-major
    uint64_t dsc_mid[3], dsc_mid_lo[3];
    for (int l = 0; l < 3; ++l) {
        const bool pq = l == p.perq_layer;
        dsc_mid[l] = make_smem_desc(pq ? smem_u32(perq) : smem_u32(smem + C::kOffMid) + mid_off[l], 128, 1024);
        dsc_mid_lo[l] = dsc_mid[l] + (uint64_t)((pq ? 8192u : (uint32_t)p.mid_N[l] * 128u) >> 4);   // lo image follows hi
    }

    for (int qi = wg; qi < nq; qi += kWG) {
        const size_t q = (size_t)stream + (size_t)qi * nstreams;
        wg_sync();                                    // the previous query's readers of wq / perq are done
        if (t < 64) {
            // (W0 * R)^T for this query
            const float w0 = p.W0[t * 3 + 0], w1 = p.W0[t * 3 + 1], w2 = p.W0[t * 3 + 2];
            float r[9] = {1.f, 0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 1.f};
            if (p.R) {
#pragma unroll
                for (int i = 0; i < 9; ++i) r[i] = p.R[q * 9 + i];
            }
            wq[0 * 64 + t] = w0 * r[0] + w1 * r[3] + w2 * r[6];
            wq[1 * 64 + t] = w0 * r[1] + w1 * r[4] + w2 * r[7];
            wq[2 * 64 + t] = w0 * r[2] + w1 * r[5] + w2 * r[8];
        }
        if (p.perq_layer >= 0) {
            const uint4* s = reinterpret_cast<const uint4*>(p.perq_img + q * C::kPerqBytes);
            uint4* d = reinterpret_cast<uint4*>(perq);
            for (uint32_t i = t; i < C::kPerqBytes / 16; i += 128) d[i] = s[i];
            fence_proxy_async_smem();
        }
        wg_sync();
        // [chunk][i]: max over the warp's 16 points so far of chunk channel 16 (lane / 4) + 8 (i / 2) + 2 q4 + i % 2
        float vmax[4 * C::kChunks];
#pragma unroll
        for (int i = 0; i < 4 * C::kChunks; ++i) vmax[i] = -INFINITY;
        for (int tq = 0; tq < tpq; ++tq) {
            // ---- first layer (fp32 FMA): points r0, r0 + 8 of the tile, channels 16 kk + 8 hc + 2 q4 + {0, 1}
            const int sgi = tq < p.seg[0].tiles ? 0 : 1;
            const Seg& sg = p.seg[sgi];
            float cx = 0.f, cy = 0.f, cz = 0.f;
            if (sg.center) { cx = p.query[q * 3 + 0]; cy = p.query[q * 3 + 1]; cz = p.query[q * 3 + 2]; }
            float px[2], py[2], pz[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                int local = (tq - (sgi ? p.seg[0].tiles : 0)) * kTile + r0 + 8 * h;
                if (local >= sg.n) local = 0;                              // duplicate padding
                const float* src = sg.ptr + (q * sg.n + local) * 3;
                px[h] = src[0] - cx; py[h] = src[1] - cy; pz[h] = src[2] - cz;   // model.py:303
            }
            uint32_t a[4][4], al[4][kL];
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
                for (int hc = 0; hc < 2; ++hc) {
                    const int ch = kk * 16 + hc * 8 + 2 * q4;
                    const float2 wx = *reinterpret_cast<const float2*>(wq + 0 * 64 + ch);
                    const float2 wy = *reinterpret_cast<const float2*>(wq + 1 * 64 + ch);
                    const float2 wz = *reinterpret_cast<const float2*>(wq + 2 * 64 + ch);
                    const float2 bb = *reinterpret_cast<const float2*>(s_b0 + ch);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        // same association as the fp32 path: fma(wx, x, fma(wy, y, fma(wz, z, b)))
                        const float v0 = fmaf(wx.x, px[h], fmaf(wy.x, py[h], fmaf(wz.x, pz[h], bb.x)));
                        const float v1 = fmaf(wx.y, px[h], fmaf(wy.y, py[h], fmaf(wz.y, pz[h], bb.y)));
                        pack_act<PRECISE>(v0, v1, a[kk][hc * 2 + h], al[kk][PRECISE ? hc * 2 + h : 0]);
                    }
                }
            }
            // ---- mid layers: 64 -> 64 ..., then 64 -> 128 into the big layer's A fragments; A stays in registers
            const float* bl = s_bias;
#pragma unroll
            for (int l = 0; l < 2; ++l) {
                if (l >= p.num_mid - 1) break;
                float d[32];
#pragma unroll
                for (int i = 0; i < 32; ++i) d[i] = 0.f;
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < 4; ++ks)
                    mid_mma<PRECISE>(d, a[ks], reinterpret_cast<const uint32_t (&)[4]>(al[PRECISE ? ks : 0]), dsc_mid[l] + (uint64_t)(ks * 16), dsc_mid_lo[l] + (uint64_t)(ks * 16), ks > 0);
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(d);
                pack_acc<PRECISE>(d, bl, q4, a, al);
                bl += 64;
            }
            uint32_t a2[8][4], a2l[8][kL];                // the tile's 128 activations: A fragments of the big layer's 8 k-steps
            {
                const uint64_t w = p.num_mid == 3 ? dsc_mid[2] : dsc_mid[0], w_lo = p.num_mid == 3 ? dsc_mid_lo[2] : dsc_mid_lo[0];
                float d[64];
#pragma unroll
                for (int i = 0; i < 64; ++i) d[i] = 0.f;
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < 4; ++ks)
                    mid_mma<PRECISE>(d, a[ks], reinterpret_cast<const uint32_t (&)[4]>(al[PRECISE ? ks : 0]), w + (uint64_t)(ks * 16), w_lo + (uint64_t)(ks * 16), ks > 0);
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(d);
                pack_acc<PRECISE>(d, bl, q4, a2, a2l);
            }
            // ---- big layer 128 -> this CTA's channels: D[64 points][128 channels] per chunk, max over the points.  Unrolled,
            // ptxas overlaps one chunk's reduction with the next chunk's MMAs (two accumulators); the precise variant's
            // twice-as-large A fragments leave no registers for that, so its loop stays rolled.  vmax[0 .. 4) is always the
            // current chunk's: the running maxima rotate by one chunk per iteration, back in order after the last one.
#pragma unroll(PRECISE ? 1 : C::kChunks)
            for (int c = 0; c < C::kChunks; ++c) {
                float d[64];
#pragma unroll
                for (int i = 0; i < 64; ++i) d[i] = 0.f;
                const uint64_t w = dsc_w3 + (uint64_t)((uint32_t)c * (C::kChunkBytes >> 4));
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < 8; ++ks) {
                    const uint64_t o = w + (uint64_t)(ks * 16);
                    if (PRECISE) {                        // small terms first: a_hi*w_lo, a_lo*w_hi, then a_hi*w_hi
                        wgmma_rs_n128(d, a2[ks], o + (uint64_t)(32768u >> 4), ks > 0);
                        wgmma_rs_n128(d, reinterpret_cast<const uint32_t (&)[4]>(a2l[PRECISE ? ks : 0]), o, 1);
                        wgmma_rs_n128(d, a2[ks], o, 1);
                    } else {
                        wgmma_rs_n128(d, a2[ks], o, ks > 0);
                    }
                }
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(d);
                // rows r0, r0 + 8 in-thread, then a reduce-scatter over the 8 lanes of a column group (lane bits 2-4): at
                // each step a lane keeps half of its values and receives its partner's maxima of that half; what is left,
                // m[i] for i < 4, is element 4 (lane / 4) + i of the original 32
                float m[32];
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    m[2 * j] = fmaxf(d[4 * j], d[4 * j + 2]);
                    m[2 * j + 1] = fmaxf(d[4 * j + 1], d[4 * j + 3]);
                }
                max_halve<16>(m, lane);
                max_halve<8>(m, lane);
                max_halve<4>(m, lane);
                float v[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) v[i] = fmaxf(vmax[i], m[i]);
#pragma unroll
                for (int i = 0; i < 4 * (C::kChunks - 1); ++i) vmax[i] = vmax[i + 4];
#pragma unroll
                for (int i = 0; i < 4; ++i) vmax[4 * (C::kChunks - 1) + i] = v[i];
            }
        }
        // ---- combine the 4 warps through shared memory (perq is dead: every MMA of this query has completed), then one
        // thread per 4 consecutive channels writes them
        constexpr int kC = C::kChunks * 128;
        const int warp = t >> 5;
        wg_sync();
#pragma unroll
        for (int c = 0; c < C::kChunks; ++c)
#pragma unroll
            for (int h = 0; h < 2; ++h)
                *reinterpret_cast<float2*>(red + warp * kC + c * 128 + 16 * (lane >> 2) + 8 * h + 2 * q4) = make_float2(vmax[4 * c + 2 * h], vmax[4 * c + 2 * h + 1]);
        wg_sync();
        for (int i = t; i < kC / 4; i += 128) {
            const float4* r4 = reinterpret_cast<const float4*>(red);
            float4 v = r4[i];
#pragma unroll
            for (int w = 1; w < 4; ++w) {
                const float4 u = r4[w * (kC / 4) + i];
                v = make_float4(fmaxf(v.x, u.x), fmaxf(v.y, u.y), fmaxf(v.z, u.z), fmaxf(v.w, u.w));
            }
            *reinterpret_cast<float4*>(p.out + q * 1024 + (size_t)(part * kC + 4 * i)) = v;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// weight packing (device side, once per model)
// ------------------------------------------------------------------------------------------------
// fp32 W[rows][K] -> fp16 K-major no-swizzle operand image: (r/8)*sbo + (k/8)*128 + (r%8)*16 + (k%8)*2
// lo = 1 writes the residual fp16(w - fp16(w)) instead (split-precision images)
__global__ void pack_kmajor_kernel(const float* __restrict__ W, int rows, int K, int row0, uint32_t sbo, uint8_t* __restrict__ img, int lo) {
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= rows * K) return;
    int r = e / K, k = e % K;
    uint32_t off = (uint32_t)(r >> 3) * sbo + (uint32_t)(k >> 3) * 128u + (uint32_t)(r & 7) * 16u + (uint32_t)(k & 7) * 2u;
    const float w = W[(size_t)(row0 + r) * K + k];
    const __half h = __float2half_rn(w);
    *reinterpret_cast<__half*>(img + off) = lo ? __float2half_rn(w - __half2float(h)) : h;
}

// per-query W1*T (fp32 [B][64][64], row = output channel) -> fp16 images of 8192 B
__global__ void pack_perq_kernel(const float* __restrict__ W, int64_t B, uint8_t* __restrict__ img) {
    int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= B * 4096) return;
    int64_t b = e >> 12;
    int r = (int)((e >> 6) & 63), k = (int)(e & 63);
    uint32_t off = (uint32_t)(r >> 3) * 1024u + (uint32_t)(k >> 3) * 128u + (uint32_t)(r & 7) * 16u + (uint32_t)(k & 7) * 2u;
    *reinterpret_cast<__half*>(img + b * 8192 + off) = __float2half_rn(W[e]);
}

// Fused per-query fold: img[b] = fp16 operand image of W1 * (T[b] + I), T[b] = the STN's raw fc3 output
// viewed as [64][64] (model.py:66-68,196,201).  One CTA per query, 256 threads, W1 and T staged in shared memory.
__global__ void __launch_bounds__(256) fold_w1_kernel(const float* __restrict__ W1, const float* __restrict__ T, int64_t B, uint8_t* __restrict__ img) {
    __shared__ float sW[64][65];
    __shared__ __align__(16) float sT[64][68];
    const int64_t b = blockIdx.x;
    const int tid = threadIdx.x;
    for (int e = tid; e < 4096; e += 256) {
        const int r = e >> 6, c = e & 63;
        sW[r][c] = W1[e];
        sT[r][c] = T[b * 4096 + e] + (r == c ? 1.0f : 0.0f);
    }
    __syncthreads();
    // thread -> output row o = tid / 4, 16 consecutive input columns i0 = (tid % 4) * 16
    const int o = tid >> 2, i0 = (tid & 3) * 16;
    float acc[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = 0.f;
    for (int j = 0; j < 64; ++j) {
        const float w = sW[o][j];
#pragma unroll
        for (int i4 = 0; i4 < 4; ++i4) {
            const float4 t4 = *reinterpret_cast<const float4*>(&sT[j][i0 + 4 * i4]);
            acc[4 * i4 + 0] = fmaf(w, t4.x, acc[4 * i4 + 0]);
            acc[4 * i4 + 1] = fmaf(w, t4.y, acc[4 * i4 + 1]);
            acc[4 * i4 + 2] = fmaf(w, t4.z, acc[4 * i4 + 2]);
            acc[4 * i4 + 3] = fmaf(w, t4.w, acc[4 * i4 + 3]);
        }
    }
    uint8_t* dst = img + b * 8192 + (uint32_t)(o >> 3) * 1024u + (uint32_t)(o & 7) * 16u;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        uint32_t v[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) v[e] = pack_half2(acc[h * 8 + 2 * e], acc[h * 8 + 2 * e + 1]);
        *reinterpret_cast<uint4*>(dst + (uint32_t)(i0 / 8 + h) * 128u) = make_uint4(v[0], v[1], v[2], v[3]);
    }
}

// conv1 folded into the STN's last layer: W1*(T+I) with T = view(fc3(f) + b, 64, 64) is linear in f, so
//   (W1*(T+I))[o][i] = sum_k f[k] * G[o*64+i][k] + g0[o*64+i],
//   G[o*64+i][k] = sum_j W1[o][j] * Wfc3[j*64+i][k],   g0[o*64+i] = sum_j W1[o][j] * bfc3[j*64+i] + W1[o][i].
// One FC layer then yields the per-query operand directly (model.py:62-68,196,201).
__global__ void fold_fc3_kernel(const float* __restrict__ W1, const float* __restrict__ Wfc3, const float* __restrict__ bfc3,
                                float* __restrict__ G, float* __restrict__ g0) {
    const int oi = blockIdx.x;                 // o*64 + i
    const int o = oi >> 6, i = oi & 63;
    const int k = threadIdx.x;                 // 0..255 (fc3 input width)
    float acc = 0.f;
    for (int j = 0; j < 64; ++j) acc = fmaf(W1[o * 64 + j], Wfc3[(size_t)(j * 64 + i) * 256 + k], acc);
    G[(size_t)oi * 256 + k] = acc;
    if (k == 0) {
        float b = W1[o * 64 + i];
        for (int j = 0; j < 64; ++j) b = fmaf(W1[o * 64 + j], bfc3[j * 64 + i], b);
        g0[oi] = b;
    }
}

// out[b][i][j] = in[b][j][i] for 64x64 blocks (the STN's transform, transposed for the W1*T product)
__global__ void transpose64_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t B) {
    int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= B * 4096) return;
    int64_t b = e >> 12;
    int i = (int)((e >> 6) & 63), j = (int)(e & 63);
    out[e] = in[b * 4096 + j * 64 + i];
}

// logits [B][od]; the sign-deciding logit is the last column (od 2: the sign logit, od 1: the signed-distance logit)
__global__ void guard_flag_kernel(const float* __restrict__ logits, int od, int64_t B, float band, int32_t* __restrict__ list, int* __restrict__ count, int64_t base, int64_t cap) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    if (fabsf(logits[i * od + od - 1]) < band) {
        int slot = atomicAdd(count, 1);
        if (slot < cap) list[slot] = (int32_t)(base + i);
    }
}
__global__ void guard_gather_kernel(const float* __restrict__ src, const int32_t* __restrict__ list, int n, int row_floats, float* __restrict__ dst) {
    int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)n * row_floats) return;
    int i = (int)(e / row_floats), j = (int)(e % row_floats);
    dst[e] = src[(int64_t)list[i] * row_floats + j];
}
__global__ void guard_scatter_kernel(const float* __restrict__ src, const int32_t* __restrict__ list, int n, int od, float* __restrict__ logits) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    for (int j = 0; j < od; ++j) logits[(int64_t)list[i] * od + j] = src[i * od + j];
}
__global__ void guard_scatter_rows_kernel(const float* __restrict__ src, const int32_t* __restrict__ list, int n, int row_floats, float* __restrict__ dst) {
    int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)n * row_floats) return;
    int i = (int)(e / row_floats), j = (int)(e % row_floats);
    dst[(int64_t)list[i] * row_floats + j] = src[e];
}

}  // namespace

// ------------------------------------------------------------------------------------------------
struct TcStack {           // one conv stack ending in the 128 -> 1024 layer
    uint8_t* w3_img = nullptr;     // 8 x 32768
    uint8_t* mid_img[3] = {nullptr, nullptr, nullptr};
    uint8_t* w3_img_p = nullptr;   // split precision: 8 x (hi 32768 | lo 32768)
    uint8_t* mid_img_p[3] = {nullptr, nullptr, nullptr};   // split precision: hi | lo
    const float* mid_bias[3] = {nullptr, nullptr, nullptr};
    int mid_N[3] = {0, 0, 0};
    int num_mid = 0;
    const float* W0 = nullptr;
    const float* b0 = nullptr;
    const float* b3 = nullptr;
};

struct TcFc {                 // one Linear layer: fp32 weights + (optional) tensor-core operand images
    const Layer* L = nullptr;
    const uint8_t* img = nullptr;
};
struct TcStnFc { TcFc fc1, fc2, fc3; };

struct TcWeights {
    TcStack qstn;                // pass A (point_stn, feat_global.stn1 or feat_local_global.stn1)
    TcStack stn[2], fin[2];      // [0] local, [1] global: pass B, pass C
    TcStnFc qstn_fc, stn_fc[2];
    TcFc head_fc1[2], head_fc2, head_fc3;
    // conv1 folded into stn2.fc3 per branch: images of G [4096 x 256] and bias g0 [4096]
    const uint8_t* fold_img[2] = {nullptr, nullptr};
    const float* fold_bias[2] = {nullptr, nullptr};
    // shared encoder (feat_local_global): passes B and C, the STN64 tail and its fold, fc1_local_global
    TcStack stn_enc, fin_enc;
    TcStnFc stn_fc_enc;
    TcFc head_fc1_enc;
    const uint8_t* fold_img_enc = nullptr;
    const float* fold_bias_enc = nullptr;
    bool fc_on_tc = true;
    std::vector<void*> allocs;
    int sm_count = 132;
    // profile of the dominant kernel (bench.py roofline)
    bool prof_on = false;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof_events;
    double prof_flops = 0.0;
    ~TcWeights() {
        for (void* a : allocs) cudaFree(a);
        for (auto& e : prof_events) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
    }
};

namespace {

uint8_t* tc_alloc(TcWeights& t, size_t bytes) {
    void* p = nullptr;
    P2S_CUDA(cudaMalloc(&p, bytes));
    P2S_CUDA(cudaMemset(p, 0, bytes));
    t.allocs.push_back(p);
    return (uint8_t*)p;
}

uint8_t* pack_layer(TcWeights& t, const Layer& L, uint32_t sbo, bool split = false) {   // whole layer as one image (hi [| lo])
    const size_t one = (size_t)L.cout * L.cin * 2;
    uint8_t* img = tc_alloc(t, one * (split ? 2 : 1));
    P2S_LAUNCH(pack_kmajor_kernel, (unsigned)cdiv((int64_t)L.cout * L.cin, 256), 256, 0, 0, L.W, L.cout, L.cin, 0, sbo, img, 0);
    if (split) P2S_LAUNCH(pack_kmajor_kernel, (unsigned)cdiv((int64_t)L.cout * L.cin, 256), 256, 0, 0, L.W, L.cout, L.cin, 0, sbo, img + one, 1);
    return img;
}

uint8_t* pack_w3(TcWeights& t, const Layer& L, bool split = false) {   // 8 chunks of 128 rows, each its own image (hi [| lo])
    P2S_CHECK(L.cout == 1024 && L.cin == 128, "big layer must be 128 -> 1024");
    const size_t chunk = split ? 65536 : 32768;
    uint8_t* img = tc_alloc(t, 8 * chunk);
    for (int c = 0; c < 8; ++c) {
        P2S_LAUNCH(pack_kmajor_kernel, (unsigned)cdiv(128 * 128, 256), 256, 0, 0, L.W, 128, 128, c * 128, 2048u, img + (size_t)c * chunk, 0);
        if (split) P2S_LAUNCH(pack_kmajor_kernel, (unsigned)cdiv(128 * 128, 256), 256, 0, 0, L.W, 128, 128, c * 128, 2048u, img + (size_t)c * chunk + 32768, 1);
    }
    return img;
}

void launch_pass(Model& m, const TcStack& s, const Seg& s0, const Seg& s1, const float* query, const float* R,
                 int64_t B, int perq_layer, const uint8_t* perq_img, float* out, cudaStream_t st, bool precise) {
    PassParams p{};
    p.seg[0] = s0; p.seg[1] = s1;
    p.query = query; p.R = R;
    p.tiles_per_query = s0.tiles + s1.tiles;
    p.B = (int)B;
    p.W0 = s.W0; p.b0 = s.b0;
    p.num_mid = s.num_mid;
    for (int l = 0; l < 3; ++l) { p.mid_N[l] = s.mid_N[l]; p.mid_img[l] = precise ? s.mid_img_p[l] : s.mid_img[l]; p.mid_bias[l] = s.mid_bias[l]; }
    p.perq_layer = perq_layer;
    p.perq_img = perq_img;
    p.w3_img = precise ? s.w3_img_p : s.w3_img;
    p.out = out;
    for (int l = 0; l < s.num_mid; ++l)
        P2S_CHECK(s.mid_N[l] == (l == s.num_mid - 1 ? 128 : 64), "pass kernel: mid layers must be 64 -> 64 ... -> 128");
    TcWeights& t = *m.tc;
    const int split = precise ? Cfg<true>::kSplit : Cfg<false>::kSplit;
    int streams = t.sm_count / split;
    if ((int64_t)streams > B) streams = (int)B;
    const int grid = streams * split;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    const bool prof = t.prof_on && !precise;
    if (prof) {
        P2S_CUDA(cudaEventCreate(&e0)); P2S_CUDA(cudaEventCreate(&e1));
        P2S_CUDA(cudaEventRecord(e0, st));
    }
    if (precise) P2S_LAUNCH(pointnet_pass_kernel<true>, grid, kThreads, Cfg<true>::kSmemBytes, st, p);
    else P2S_LAUNCH(pointnet_pass_kernel<false>, grid, kThreads, Cfg<false>::kSmemBytes, st, p);
    if (prof) {
        P2S_CUDA(cudaEventRecord(e1, st));
        t.prof_events.emplace_back(e0, e1);
        // algorithmic FLOPs of this launch: real (un-padded) points, un-duplicated layers (SURVEY.md section 8d)
        double mac_pt = 3.0 * 64 + 128.0 * 1024;
        int prev = 64;
        for (int l = 0; l < s.num_mid; ++l) { mac_pt += (double)prev * s.mid_N[l]; prev = s.mid_N[l]; }
        t.prof_flops += 2.0 * mac_pt * (double)(s0.n + s1.n) * (double)B;
    }
}

Seg make_seg(const float* ptr, int n, int center) { return Seg{ptr, n, n > 0 ? (n + kTile - 1) / kTile : 0, center}; }

// in_bias (optional, tensor-core kernel only): the layer reads act(in + in_bias) -- the raw max features of a pass get their
// conv3 bias (and the STN's ReLU) on the way into the first FC layer instead of in separate copy / bias kernels
void run_fc(const TcFc& f, const float* in, int lda, float* out, int ldc, int64_t Bc, bool relu, bool on_tc, cudaStream_t st,
            const float* in_bias = nullptr, bool in_relu = false) {
    const Layer& L = *f.L;
    if (on_tc && f.img) launch_fc_tc(in, lda, f.img, L.b, out, ldc, Bc, L.cout, L.cin, relu, st, 0, in_bias, in_relu);
    else {
        P2S_CHECK(!in_bias, "input bias needs the tensor-core FC kernel");
        launch_gemm_nt(in, 0, lda, L.W, 0, L.b, out, 0, ldc, (int)Bc, L.cout, L.cin, 1, relu, st);
    }
}

void fc_tail(const Layer& b3src, const TcStnFc& s, bool on_tc, const float* gmax_raw, int64_t Bc, float* g, float* f1, float* f2, float* out, cudaStream_t st) {
    // g = relu(max + b3) ; fc1 ; fc2 ; fc3     (model.py:44-64 / 103-122)
    if (on_tc && s.fc1.img) run_fc(s.fc1, gmax_raw, 1024, f1, 512, Bc, true, true, st, b3src.b, true);
    else {
        P2S_CUDA(cudaMemcpyAsync(g, gmax_raw, (size_t)Bc * 1024 * 4, cudaMemcpyDeviceToDevice, st));
        launch_bias_act(g, b3src.b, Bc, 1024, true, st);
        run_fc(s.fc1, g, 1024, f1, 512, Bc, true, on_tc, st);
    }
    run_fc(s.fc2, f1, 512, f2, 256, Bc, true, on_tc, st);
    run_fc(s.fc3, f2, 256, out, s.fc3.L->cout, Bc, false, on_tc, st);
}

}  // namespace

void tc_build(Model& m) {
    P2S_CHECK(m.cfg.net_size == 1024, "tensor-core path needs net_size 1024");
    TcWeights* t = new TcWeights();
    m.tc = t;
    cudaDeviceProp prop;
    P2S_CUDA(cudaGetDeviceProperties(&prop, m.device));
    t->sm_count = prop.multiProcessorCount;
    P2S_CUDA(cudaFuncSetAttribute(pointnet_pass_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg<false>::kSmemBytes));
    P2S_CUDA(cudaFuncSetAttribute(pointnet_pass_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg<true>::kSmemBytes));
    auto build_stn = [&](TcStack& s, const Stn& stn, const Layer* c0a, const Layer* c0b) {
        // QSTN: x -> conv1(3->64) [layer 0] -> conv2 (64->128) -> conv3 ; STN64 on feat: conv0a [layer 0] -> conv0b -> conv1 -> conv2 -> conv3
        if (!c0a) {
            s.W0 = stn.c1.W; s.b0 = stn.c1.b;
            s.num_mid = 1;
            s.mid_img[0] = pack_layer(*t, stn.c2, 1024); s.mid_bias[0] = stn.c2.b; s.mid_N[0] = 128;
            s.mid_img_p[0] = pack_layer(*t, stn.c2, 1024, true);
        } else {
            s.W0 = c0a->W; s.b0 = c0a->b;
            s.num_mid = 3;
            s.mid_img[0] = pack_layer(*t, *c0b, 1024); s.mid_bias[0] = c0b->b; s.mid_N[0] = 64;
            s.mid_img[1] = pack_layer(*t, stn.c1, 1024); s.mid_bias[1] = stn.c1.b; s.mid_N[1] = 64;
            s.mid_img[2] = pack_layer(*t, stn.c2, 1024); s.mid_bias[2] = stn.c2.b; s.mid_N[2] = 128;
            s.mid_img_p[0] = pack_layer(*t, *c0b, 1024, true);
            s.mid_img_p[1] = pack_layer(*t, stn.c1, 1024, true);
            s.mid_img_p[2] = pack_layer(*t, stn.c2, 1024, true);
        }
        s.w3_img_p = pack_w3(*t, stn.c3, true);
        s.w3_img = pack_w3(*t, stn.c3);
        s.b3 = stn.c3.b;
    };
    auto build_fin = [&](TcStack& s, const Feat& f) {
        s.W0 = f.conv0a.W; s.b0 = f.conv0a.b;
        s.num_mid = 3;
        s.mid_img[0] = pack_layer(*t, f.conv0b, 1024); s.mid_bias[0] = f.conv0b.b; s.mid_N[0] = 64;
        s.mid_img[1] = nullptr; s.mid_bias[1] = f.conv1.b; s.mid_N[1] = 64;       // per query: conv1 * T
        s.mid_img[2] = pack_layer(*t, f.conv2, 1024); s.mid_bias[2] = f.conv2.b; s.mid_N[2] = 128;
        s.mid_img_p[0] = pack_layer(*t, f.conv0b, 1024, true);
        s.mid_img_p[2] = pack_layer(*t, f.conv2, 1024, true);
        s.w3_img_p = pack_w3(*t, f.conv3, true);
        s.w3_img = pack_w3(*t, f.conv3);
        s.b3 = f.conv3.b;
    };
    fc_tc_init();
    t->fc_on_tc = !env_flag("P2S_FC_FP32");
    auto mk_fc = [&](const Layer& L) {
        TcFc f;
        f.L = &L;
        f.img = fc_tc_supported(L.cout, L.cin) ? fc_tc_pack(L, t->allocs) : nullptr;
        return f;
    };
    auto mk_stn_fc = [&](const Stn& s) { TcStnFc r; r.fc1 = mk_fc(s.fc1); r.fc2 = mk_fc(s.fc2); r.fc3 = mk_fc(s.fc3); return r; };
    auto fold = [&](const Feat& f, const uint8_t*& img, const float*& bias) {
        P2S_CHECK(f.stn2.fc3.cout == 4096 && f.stn2.fc3.cin == 256 && f.conv1.cout == 64 && f.conv1.cin == 64, "unexpected STN shape");
        float* G = reinterpret_cast<float*>(tc_alloc(*t, (size_t)4096 * 256 * 4));
        float* g0 = reinterpret_cast<float*>(tc_alloc(*t, 4096 * 4));
        P2S_LAUNCH(fold_fc3_kernel, 4096, 256, 0, 0, f.conv1.W, f.stn2.fc3.W, f.stn2.fc3.b, G, g0);
        img = fc_tc_pack_raw(G, 4096, 256, t->allocs);
        bias = g0;
    };
    if (m.single_transformer) {
        // one encoder over patch + sub-sample: only its stacks exist (local / global / point_stn are empty)
        t->qstn_fc = mk_stn_fc(m.enc.stn1);
        t->stn_fc_enc = mk_stn_fc(m.enc.stn2);
        fold(m.enc, t->fold_img_enc, t->fold_bias_enc);
        t->head_fc1_enc = mk_fc(m.fc1_enc);
        t->head_fc2 = mk_fc(m.fc2);
        t->head_fc3 = mk_fc(m.fc3);
        build_stn(t->qstn, m.enc.stn1, nullptr, nullptr);
        build_stn(t->stn_enc, m.enc.stn2, &m.enc.conv0a, &m.enc.conv0b);
        build_fin(t->fin_enc, m.enc);
        P2S_CUDA(cudaDeviceSynchronize());
        return;
    }
    if (m.shared_qstn) t->qstn_fc = mk_stn_fc(m.point_stn);
    else if (m.global.has_qstn) t->qstn_fc = mk_stn_fc(m.global.stn1);
    t->stn_fc[0] = mk_stn_fc(m.local.stn2);
    t->stn_fc[1] = mk_stn_fc(m.global.stn2);
    for (int br = 0; br < 2; ++br) fold(br ? m.global : m.local, t->fold_img[br], t->fold_bias[br]);
    t->head_fc1[0] = mk_fc(m.fc1_local);
    t->head_fc1[1] = mk_fc(m.fc1_global);
    t->head_fc2 = mk_fc(m.fc2);
    t->head_fc3 = mk_fc(m.fc3);
    if (m.shared_qstn) build_stn(t->qstn, m.point_stn, nullptr, nullptr);
    else if (m.global.has_qstn) build_stn(t->qstn, m.global.stn1, nullptr, nullptr);
    build_stn(t->stn[0], m.local.stn2, &m.local.conv0a, &m.local.conv0b);
    build_stn(t->stn[1], m.global.stn2, &m.global.conv0a, &m.global.conv0b);
    build_fin(t->fin[0], m.local);
    build_fin(t->fin[1], m.global);
    P2S_CUDA(cudaDeviceSynchronize());
}

void tc_destroy(Model& m) {
    delete m.tc;
    m.tc = nullptr;
}

void tc_profile_reset(Model& m, bool on) {
    TcWeights& t = *m.tc;
    for (auto& e : t.prof_events) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
    t.prof_events.clear();
    t.prof_flops = 0.0;
    t.prof_on = on;
}

void tc_profile_get(Model& m, double* ms, int64_t* launches, double* flops) {
    TcWeights& t = *m.tc;
    double total = 0.0;
    for (auto& e : t.prof_events) {
        P2S_CUDA(cudaEventSynchronize(e.second));
        float x = 0.f;
        P2S_CUDA(cudaEventElapsedTime(&x, e.first, e.second));
        total += x;
    }
    *ms = total;
    *launches = (int64_t)t.prof_events.size();
    *flops = t.prof_flops;
}

// One pass of the network over B queries on tensor cores.  precise = split-precision operands everywhere
// (the accurate path used for the guard band); fp16 operands otherwise.
static void forward_tc_core(Model& m, const float* patch, const float* sub, const float* query, int64_t B,
                            float* logits, cudaStream_t st, bool precise) {
    TcWeights& t = *m.tc;
    const int P = m.cfg.points_per_patch, S = m.cfg.sub_sample_size;
    const int64_t Bc_max = 8192;
    // workspace (floats per query)
    const size_t per_q = 1024 * 4 + 512 + 256 + 4 + 9 + 4096 * 2 + 1024 + 256 + 128 + 4096 /* 16 KB perq image (hi | lo) */ + 16 +
                         1024 + 512 + 256 /* A operand images of the FC tails (4 B per element: hi + lo fp16) */;
    float* base = m.ws_net.as<float>(per_q * (size_t)Bc_max + 1024);
    float* pcur = base;
    auto take = [&](size_t n) { float* r = pcur; pcur += (n * (size_t)Bc_max + 63) / 64 * 64; return r; };
    float* gmax = take(1024); float* g = take(1024); float* f1 = take(512); float* f2 = take(256);
    float* q4 = take(4); float* R = take(9); float* T = take(4096); float* Tt = take(4096);
    float* fmax_l = take(1024); float* fmax_g = take(1024); float* cat = take(1024); float* h3 = take(256); float* h4 = take(128);
    uint8_t* perq = reinterpret_cast<uint8_t*>(take(4096));
    // A operand images (hi | lo fp16, 4 B per element; Bc_max is a multiple of 128): K = 1024, 512, 256
    uint8_t* imgA = reinterpret_cast<uint8_t*>(take(1024)); uint8_t* imgB = reinterpret_cast<uint8_t*>(take(512)); uint8_t* imgC = reinterpret_cast<uint8_t*>(take(256));
    const bool fc_tc = t.fc_on_tc || precise;   // the precise path needs the split-precision FC kernel's image output
    // FC tails as a chain of operand images: the raw max features are packed once (bias + ReLU on the way), every layer reads
    // its A operand by bulk copy and writes its output as the next layer's image -- no per-N-tile re-conversion of A
    auto img_ok = [](const TcStnFc& f) { return f.fc1.img && f.fc2.img; };
    // gmax_raw [Bc,1024] -> relu(+b3) -> fc1 -> fc2; f2 as fp32 rows (out_f2) or as an image in imgC
    auto stn_tail_img = [&](const Layer& c3, const TcStnFc& f, const float* gmax_raw, int64_t Bc, float* out_f2) {
        launch_pack_a(gmax_raw, 1024, Bc, 1024, c3.b, true, imgA, st);
        launch_fc_tc_img(imgA, f.fc1.img, f.fc1.L->b, imgB, 0, Bc, 512, 1024, true, st, 3, 16, 0);
        if (out_f2) launch_fc_tc_img(imgB, f.fc2.img, f.fc2.L->b, out_f2, 256, Bc, 256, 512, true, st, 0);
        else launch_fc_tc_img(imgB, f.fc2.img, f.fc2.L->b, imgC, 0, Bc, 256, 512, true, st, 3, 8, 0);
    };
    // tail of a pass A (QSTN): raw max gmax -> fc1, fc2, fc3 -> quaternion q4 -> rotation R
    auto qstn_rot = [&](const Layer& c3, int64_t Bc) {
        { StageScope ts("net: fc tails", st);
          if (fc_tc && img_ok(t.qstn_fc)) {
              stn_tail_img(c3, t.qstn_fc, gmax, Bc, f2);
              run_fc(t.qstn_fc.fc3, f2, 256, q4, 4, Bc, false, false, st);
          } else fc_tail(c3, t.qstn_fc, fc_tc, gmax, Bc, g, f1, f2, q4, st); }
        launch_quat_to_rot(q4, R, Bc, st);
    };
    // tail of a pass B (STN64 of feature stack f): raw max gmax -> the per-query operand image of conv1 * (T + I) in perq
    auto stn64_perq = [&](const Feat& f, const TcStnFc& fc, const uint8_t* fold_img, const float* fold_bias, int64_t Bc) {
        if (fc_tc) {
            // fc1, fc2, then the folded last layer writes the per-query fp16 operand images of conv1*(T+I) directly
            StageScope ts("net: fc tails", st);
            if (img_ok(fc)) {
                stn_tail_img(f.stn2.c3, fc, gmax, Bc, nullptr);
                launch_fc_tc_img(imgC, fold_img, fold_bias, perq, 0, Bc, 4096, 256, false, st, precise ? 2 : 1);
            } else {
                run_fc(fc.fc1, gmax, 1024, f1, 512, Bc, true, true, st, f.stn2.c3.b, true);
                run_fc(fc.fc2, f1, 512, f2, 256, Bc, true, true, st);
                launch_fc_tc(f2, 256, fold_img, fold_bias, reinterpret_cast<float*>(perq), 0, Bc, 4096, 256, false, st, precise ? 2 : 1);
            }
        } else {
            { StageScope ts("net: fc tails", st); fc_tail(f.stn2.c3, fc, false, gmax, Bc, g, f1, f2, T, st); }
            // W1' = conv1.W * (T + I) -> per-query fp16 operand images (one fused kernel)
            { StageScope ts("net: fold W1*T", st); P2S_LAUNCH(fold_w1_kernel, (unsigned)Bc, 256, 0, st, f.conv1.W, T, Bc, perq); }
        }
    };

    for (int64_t b0 = 0; b0 < B; b0 += Bc_max) {
        const int64_t Bc = (B - b0 < Bc_max) ? (B - b0) : Bc_max;
        const float* pa = patch + b0 * P * 3;
        const float* su = sub + b0 * S * 3;
        const float* qu = query + b0 * 3;
        const float* Rq = nullptr;
        if (m.single_transformer) {
            // shared encoder (model.py:320-323): every pass runs over both segments, cat(patch, sub - q), so each pass still
            // sees P + S points per query, but there are three passes instead of five and one STN64 tail instead of two
            const Seg sp = make_seg(pa, P, 0), ss = make_seg(su, S, 1);
            // pass A: feat_local_global.stn1 -> R, which rotates all P + S points (model.py:180-184)
            { StageScope ts("net: pass kernels", st); launch_pass(m, t.qstn, sp, ss, qu, nullptr, Bc, -1, nullptr, gmax, st, precise); }
            qstn_rot(m.enc.stn1.c3, Bc);
            // pass B: STN64 over both segments with R folded into W0 -> the per-query conv1 * (T + I) image
            { StageScope ts("net: pass kernels", st); launch_pass(m, t.stn_enc, sp, ss, qu, R, Bc, -1, nullptr, gmax, st, precise); }
            stn64_perq(m.enc, t.stn_fc_enc, t.fold_img_enc, t.fold_bias_enc, Bc);
            // pass C: both segments with R and the per-query image -> the encoder's raw max feature
            { StageScope ts("net: pass kernels", st); launch_pass(m, t.fin_enc, sp, ss, qu, R, Bc, 1, perq, fmax_l, st, precise); }
            const bool fuse_b3 = fc_tc && !m.debug_aux && t.head_fc1_enc.img;
            if (!fuse_b3) launch_bias_act(fmax_l, m.enc.conv3.b, Bc, 1024, false, st);
            debug_aux_copy(m, b0, Bc, R, fmax_l, nullptr, st);
            StageScope ts_head("net: fc tails", st);
            if (fuse_b3 && t.head_fc2.img && t.head_fc3.img) {
                // fc1_local_global (N = 1024) writes fc2's K = 1024 operand image directly
                uint8_t* imgCat = reinterpret_cast<uint8_t*>(cat);
                launch_pack_a(fmax_l, 1024, Bc, 1024, m.enc.conv3.b, false, imgA, st);
                launch_fc_tc_img(imgA, t.head_fc1_enc.img, m.fc1_enc.b, imgCat, 0, Bc, 1024, 1024, true, st, 3, 32, 0);
                launch_fc_tc_img(imgCat, t.head_fc2.img, m.fc2.b, imgC, 0, Bc, 256, 1024, true, st, 3, 8, 0);
                launch_fc_tc_img(imgC, t.head_fc3.img, m.fc3.b, h4, 128, Bc, 128, 256, true, st, 0);
            } else {
                run_fc(t.head_fc1_enc, fmax_l, 1024, cat, 1024, Bc, true, fc_tc, st, fuse_b3 ? m.enc.conv3.b : nullptr, false);
                run_fc(t.head_fc2, cat, 1024, h3, 256, Bc, true, fc_tc, st);
                run_fc(t.head_fc3, h3, 256, h4, 128, Bc, true, fc_tc, st);
            }
            const int od = m.fc4.cout;
            launch_gemm_nt(h4, 0, 128, m.fc4.W, 0, m.fc4.b, logits + b0 * od, 0, od, (int)Bc, od, 128, 1, false, st);
            continue;
        }
        if (m.shared_qstn) {
            // pass A over cat(patch, sub - q)   (model.py:303,325-327)
            { StageScope ts("net: pass kernels", st); launch_pass(m, t.qstn, make_seg(pa, P, 0), make_seg(su, S, 1), qu, nullptr, Bc, -1, nullptr, gmax, st, precise); }
            qstn_rot(m.point_stn.c3, Bc);
            Rq = R;
        } else if (m.global.has_qstn) {
            launch_pass(m, t.qstn, make_seg(su, S, 1), make_seg(nullptr, 0, 0), qu, nullptr, Bc, -1, nullptr, gmax, st, precise);
            qstn_rot(m.global.stn1.c3, Bc);
            Rq = R;
        }
        for (int br = 1; br >= 0; --br) {    // global first like the reference, then local
            const Feat& f = br ? m.global : m.local;
            const Seg sg = br ? make_seg(su, S, 1) : make_seg(pa, P, 0);
            float* fmax = br ? fmax_g : fmax_l;
            // pass B: STN64 -> T
            { StageScope ts("net: pass kernels", st); launch_pass(m, t.stn[br], sg, make_seg(nullptr, 0, 0), qu, Rq, Bc, -1, nullptr, gmax, st, precise); }
            stn64_perq(f, t.stn_fc[br], t.fold_img[br], t.fold_bias[br], Bc);
            (void)Tt;
            // pass C: final stack -> max feature (bias, no ReLU: model.py:203,210-212)
            { StageScope ts("net: pass kernels", st); launch_pass(m, t.fin[br], sg, make_seg(nullptr, 0, 0), qu, Rq, Bc, 1, perq, fmax, st, precise); }
        }
        // max features = raw max + conv3 bias, no ReLU (model.py:203,210-212): added by the first head FC on load, or by a
        // separate kernel when the features are exported (debug_aux) or the FCs run on the fp32 kernels
        const bool fuse_b3 = fc_tc && !m.debug_aux && t.head_fc1[0].img && t.head_fc1[1].img;
        if (!fuse_b3) {
            launch_bias_act(fmax_l, m.local.conv3.b, Bc, 1024, false, st);
            launch_bias_act(fmax_g, m.global.conv3.b, Bc, 1024, false, st);
        }
        debug_aux_copy(m, b0, Bc, Rq, fmax_l, fmax_g, st);
        StageScope ts_head("net: fc tails", st);
        if (fuse_b3 && t.head_fc2.img && t.head_fc3.img) {
            // cat(local, global) (model.py:335,343,346) is the K = 1024 operand image of fc2: k-steps 0-15 local, 16-31 global
            uint8_t* imgCat = reinterpret_cast<uint8_t*>(cat);            // [Bc,1024] x 4 B: same footprint as the fp32 rows
            launch_pack_a(fmax_l, 1024, Bc, 1024, m.local.conv3.b, false, imgA, st);
            launch_fc_tc_img(imgA, t.head_fc1[0].img, m.fc1_local.b, imgCat, 0, Bc, 512, 1024, true, st, 3, 32, 0);
            launch_pack_a(fmax_g, 1024, Bc, 1024, m.global.conv3.b, false, imgA, st);
            launch_fc_tc_img(imgA, t.head_fc1[1].img, m.fc1_global.b, imgCat, 0, Bc, 512, 1024, true, st, 3, 32, 16);
            launch_fc_tc_img(imgCat, t.head_fc2.img, m.fc2.b, imgC, 0, Bc, 256, 1024, true, st, 3, 8, 0);
            launch_fc_tc_img(imgC, t.head_fc3.img, m.fc3.b, h4, 128, Bc, 128, 256, true, st, 0);
        } else {
            run_fc(t.head_fc1[0], fmax_l, 1024, cat, 1024, Bc, true, fc_tc, st, fuse_b3 ? m.local.conv3.b : nullptr, false);
            run_fc(t.head_fc1[1], fmax_g, 1024, cat + 512, 1024, Bc, true, fc_tc, st, fuse_b3 ? m.global.conv3.b : nullptr, false);
            run_fc(t.head_fc2, cat, 1024, h3, 256, Bc, true, fc_tc, st);
            run_fc(t.head_fc3, h3, 256, h4, 128, Bc, true, fc_tc, st);
        }
        const int od = m.fc4.cout;
        launch_gemm_nt(h4, 0, 128, m.fc4.W, 0, m.fc4.b, logits + b0 * od, 0, od, (int)Bc, od, 128, 1, false, st);
    }
}

// accurate recompute used for the guard band: split-precision tensor-core path (default) or the fp32 FMA path
// (environment P2S_GUARD_FP32=1)
void forward_guard(Model& m, const float* patch, const float* sub, const float* query, int64_t B, float* logits, cudaStream_t st) {
    static const bool use_fp32 = env_flag("P2S_GUARD_FP32");
    if (use_fp32) forward_fp32(m, patch, sub, query, B, logits, st);
    else forward_tc_core(m, patch, sub, query, B, logits, st, true);
}

void forward_tc(Model& m, const float* patch, const float* sub, const float* query, int64_t B,
                float* logits, cudaStream_t st) {
    const int P = m.cfg.points_per_patch, S = m.cfg.sub_sample_size, od = m.fc4.cout;
    forward_tc_core(m, patch, sub, query, B, logits, st, false);

    // guard band: queries whose sign-deciding logit is too close to 0 for fp16-operand arithmetic are recomputed in fp32
    if (m.guard_band > 0.f && m.guard_list) {
        // deferred: only record which queries fall into the band (the fused pipeline recomputes them in one batch)
        P2S_LAUNCH(guard_flag_kernel, (unsigned)cdiv(B, 256), 256, 0, st, logits, od, B, m.guard_band, m.guard_list, m.guard_list_count, m.guard_base, m.guard_list_cap);
    } else if (m.guard_band > 0.f) {
        StageScope ts_guard("net: guard-band fp32 recompute", st);
        int32_t* list = m.ws_guard.as<int32_t>((size_t)B + 64);
        int* count = reinterpret_cast<int*>(list + B);
        P2S_CUDA(cudaMemsetAsync(count, 0, sizeof(int), st));
        P2S_LAUNCH(guard_flag_kernel, (unsigned)cdiv(B, 256), 256, 0, st, logits, od, B, m.guard_band, list, count, (int64_t)0, B);
        int n = 0;
        P2S_CUDA(cudaMemcpyAsync(&n, count, sizeof(int), cudaMemcpyDeviceToHost, st));
        P2S_CUDA(cudaStreamSynchronize(st));
        m.last_guard_count += n;
        if (n > 0) {
            const size_t rowp = (size_t)P * 3, rows = (size_t)S * 3;
            float* const aux = m.debug_aux;
            const size_t aux_floats = aux ? (size_t)n * kAuxStride : 0;
            float* gbuf = m.ws_misc.as<float>((size_t)n * (rowp + rows + 3 + od) + 64 + aux_floats);
            float* gp = gbuf; float* gs = gp + (size_t)n * rowp; float* gq = gs + (size_t)n * rows; float* gl = gq + ((size_t)n * 3 + 3) / 4 * 4;
            float* gaux = gl + ((size_t)n * od + 3) / 4 * 4;
            P2S_LAUNCH(guard_gather_kernel, (unsigned)cdiv((int64_t)n * rowp, 256), 256, 0, st, patch, list, n, (int)rowp, gp);
            P2S_LAUNCH(guard_gather_kernel, (unsigned)cdiv((int64_t)n * rows, 256), 256, 0, st, sub, list, n, (int)rows, gs);
            P2S_LAUNCH(guard_gather_kernel, (unsigned)cdiv((int64_t)n * 3, 256), 256, 0, st, query, list, n, 3, gq);
            // the recompute sees the flagged queries in list order: its diagnostics go to scratch rows and are scattered
            // back to the queries' own rows, like the logits
            if (aux) m.debug_aux = gaux;
            try {
                forward_guard(m, gp, gs, gq, n, gl, st);
            } catch (...) {
                m.debug_aux = aux;
                throw;
            }
            m.debug_aux = aux;
            P2S_LAUNCH(guard_scatter_kernel, (unsigned)cdiv(n, 256), 256, 0, st, gl, list, n, od, logits);
            if (aux) P2S_LAUNCH(guard_scatter_rows_kernel, (unsigned)cdiv((int64_t)n * kAuxStride, 256), 256, 0, st, gaux, list, n, (int)kAuxStride, aux);
        }
    }
}

}  // namespace p2s
