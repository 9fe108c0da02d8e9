// Tensor-core GEMM for the per-query FC tails of the TC path (QSTN/STN heads 1024->512->256->{4,4096} and the
// decoder 1024->512 (x2), 1024->256, 256->128; source/points_to_surf_model.py:62-64,120-122,335,343,348-350):
//     C[M][N] = act( A[M][K] * W[N][K]^T + b ),  A fp32 row-major, W pre-packed operand images, fp32 accumulation
//     in registers (wgmma), C fp32 row-major.
// These layers produce the point rotation, the 64x64 feature transform and the logits, so they keep ~22-bit operands:
// every fp32 operand x is split into two fp16 numbers x_hi + x_lo (x_hi = fp16(x), x_lo = fp16(x - x_hi))
// and the product is evaluated as A_hi*W_hi + A_lo*W_hi + A_hi*W_lo (the dropped lo*lo term is ~2^-22 relative).
// That holds while x_hi and x_lo are fp16 normal numbers (2^-3 <~ |x| <= 65504).  The training GEMMs (launch_gemm_nt_tc)
// scale every row of A and W by a power of two first (split_exp, model.cuh); the inference chain's activations are O(1).
// Three tensor-core passes cost nothing here: the FC tails are 1 % of the network's FLOPs.
// One CTA per 128 x 128 output tile; K streamed in 32-wide stages (3-deep ring):
//   warps 0-3   producers (fp32 A only): thread = output row; load 32 fp32 of that row, split, store the two K-major
//               A operands
//   warps 4-7   consumer warpgroup 0: wgmma for output rows 0-63 of the tile, then its epilogue (+bias, ReLU -> global)
//   warps 8-11  consumer warpgroup 1: rows 64-127
//   warp 12     bulk-copies the W stage images (hi + lo, 16 KB) and, for an A operand image, the A stage too
#include "model.cuh"
#include "tc_ptx.cuh"

namespace p2s {

using namespace ptx;

namespace {

constexpr int kStages = 3;
constexpr int kBK = 32;
constexpr int kFcThreads = 416;
constexpr uint32_t kHalf = 128 * kBK * 2;     // one 128 x 32 fp16 operand image: 8 KB (K-major, LBO 128, SBO 512)
constexpr uint32_t kStageA = 2 * kHalf;       // hi + lo
constexpr uint32_t kStageB = 2 * kHalf;       // hi + lo
constexpr uint32_t kFcSmem = kStages * (kStageA + kStageB) + 256;

struct FcBars {
    uint64_t full[kStages], empty[kStages];
};

__device__ __forceinline__ void split_half2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
    const __half2 h = __floats2half2_rn(x0, x1);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}

// A operand: fp32 rows (converted by the producer warps, `A`) or a pre-packed operand image `Aimg`
// ([M/128][K/32][hi | lo][128 x 32 fp16], the W layout): then the producers have nothing to do and both operands of a k-step
// arrive by bulk copy (every A element is loaded and split once instead of once per N tile).
// pack_img == 3 writes C as the NEXT layer's operand image (k-steps out_kt_off.. of out_kt_total).
// kScaled (training GEMMs only): rows of A and W scaled by 2^a_exp[m] / 2^w_exp[n] (model.cuh, split_exp); a template
// parameter so that the inference instantiation carries none of it.
template <bool kScaled>
__global__ void __launch_bounds__(kFcThreads, 1) fc_tc_kernel(const float* __restrict__ A, int lda, const uint8_t* __restrict__ Wimg,
                                                              const float* __restrict__ bias, float* __restrict__ C, int ldc,
                                                              int M, int N, int K, int relu, int pack_img,
                                                              const float* __restrict__ in_bias, int in_relu,
                                                              const uint8_t* __restrict__ Aimg, int out_kt_total, int out_kt_off,
                                                              const int* __restrict__ a_exp, const int* __restrict__ w_exp) {
    extern __shared__ __align__(1024) uint8_t smem[];
    FcBars* bars = reinterpret_cast<FcBars*>(smem + kStages * (kStageA + kStageB));
    const int tid = threadIdx.x, warp = tid >> 5;
    const int m0 = blockIdx.y * 128, nt = blockIdx.x;   // N tiles of one row block are adjacent: A is re-read from L2
    const int nk = K / kBK;
    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) { mbar_init(&bars->full[s], Aimg ? 1 : 129); mbar_init(&bars->empty[s], 2); }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ---- producers: A[m0 + tid][k0 .. k0+31] -> fp16 hi / lo, K-major (LBO 128, SBO 512)
        if (Aimg) return;
        const int row = m0 + tid;
        const float* src = A + (int64_t)(row < M ? row : 0) * lda;
        // register double buffer: the loads of k-step kt + 1 are in flight while k-step kt is converted and stored
        float4 v[8], nv[8];
        const bool row_ok = row < M;
        // training GEMMs (a_exp set, no in_bias): the row is scaled by 2^s before the split (model.cuh, split_exp)
        const int sa_row = kScaled && row_ok ? a_exp[row] : 0;
        const bool fa_one = sa_row >= -126 && sa_row <= 127;            // 2^s is a normal float: one multiplication
        const float2 fa = fa_one ? make_float2(__int_as_float((127 + sa_row) << 23), 1.f) : split_factors(sa_row);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = row_ok ? *reinterpret_cast<const float4*>(src + j * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
        for (int kt = 0; kt < nk; ++kt) {
            const int s = kt % kStages;
            const uint32_t use = (uint32_t)(kt / kStages);
            const bool more = row_ok && (kt + 1 < nk);
#pragma unroll
            for (int j = 0; j < 8; ++j) nv[j] = more ? *reinterpret_cast<const float4*>(src + (kt + 1) * kBK + j * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
            mbar_wait_bounded(&bars->empty[s], (use & 1) ^ 1);
            uint8_t* dst = smem + s * kStageA + (uint32_t)(tid >> 3) * 512u + (uint32_t)(tid & 7) * 16u;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                float x[8] = {v[2 * c].x, v[2 * c].y, v[2 * c].z, v[2 * c].w, v[2 * c + 1].x, v[2 * c + 1].y, v[2 * c + 1].z, v[2 * c + 1].w};
                if (in_bias) {          // A = act(A_raw + in_bias[k]): same fp32 operations as a separate bias / ReLU kernel
                    const float4 b0 = __ldg(reinterpret_cast<const float4*>(in_bias + kt * kBK + c * 8)), b1 = __ldg(reinterpret_cast<const float4*>(in_bias + kt * kBK + c * 8 + 4));
                    x[0] += b0.x; x[1] += b0.y; x[2] += b0.z; x[3] += b0.w; x[4] += b1.x; x[5] += b1.y; x[6] += b1.z; x[7] += b1.w;
                    if (in_relu) {
#pragma unroll
                        for (int e = 0; e < 8; ++e) x[e] = fmaxf(x[e], 0.f);
                    }
                }
                if (kScaled) {
                    if (fa_one) {
#pragma unroll
                        for (int e = 0; e < 8; ++e) x[e] *= fa.x;
                    } else {
#pragma unroll
                        for (int e = 0; e < 8; ++e) x[e] = x[e] * fa.x * fa.y;
                    }
                }
                uint32_t hi[4], lo[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) split_half2(x[2 * e], x[2 * e + 1], hi[e], lo[e]);
                *reinterpret_cast<uint4*>(dst + c * 128) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
                *reinterpret_cast<uint4*>(dst + kHalf + c * 128) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
            }
            fence_proxy_async_smem();
            mbar_arrive(&bars->full[s]);
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = nv[j];
        }
    } else if (warp == 12) {
        // ---- W (and A image) stage copies, one elected lane
        const uint8_t* wsrc = Wimg + (size_t)nt * nk * kStageB;
        const uint8_t* asrc = Aimg ? Aimg + (size_t)blockIdx.y * nk * kStageA : nullptr;
        for (int kt = 0; kt < nk; ++kt) {
            const int s = kt % kStages;
            if (kt >= kStages) mbar_wait_bounded(&bars->empty[s], (uint32_t)(kt / kStages - 1) & 1);
            if (elect_one()) {
                mbar_arrive_expect_tx(&bars->full[s], kStageB + (asrc ? kStageA : 0u));
                bulk_g2s(smem + kStages * kStageA + s * kStageB, wsrc + (size_t)kt * kStageB, kStageB, &bars->full[s]);
                if (asrc) bulk_g2s(smem + s * kStageA, asrc + (size_t)kt * kStageA, kStageA, &bars->full[s]);
            }
            __syncwarp();
        }
    } else {
        // ---- consumers: warpgroup wg owns output rows wg*64 .. wg*64+63 of the tile
        const int wg = (warp - 4) >> 2, t = tid & 127;
        const uint64_t dsc_a = make_smem_desc(smem_u32(smem) + (uint32_t)wg * 4096u, 128, 512);
        const uint64_t dsc_b = make_smem_desc(smem_u32(smem + kStages * kStageA), 128, 512);
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        for (int kt = 0; kt < nk; ++kt) {
            const int s = kt % kStages;
            mbar_wait_bounded(&bars->full[s], (uint32_t)(kt / kStages) & 1);
            const uint64_t a_hi = dsc_a + (uint64_t)(s * (kStageA >> 4)), a_lo = a_hi + (uint64_t)(kHalf >> 4);
            const uint64_t b_hi = dsc_b + (uint64_t)(s * (kStageB >> 4)), b_lo = b_hi + (uint64_t)(kHalf >> 4);
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < kBK / 16; ++ks) {
                wgmma_ss_n128(acc, a_lo + (uint64_t)(ks * 16), b_hi + (uint64_t)(ks * 16), (kt | ks) > 0);   // small terms first
                wgmma_ss_n128(acc, a_hi + (uint64_t)(ks * 16), b_lo + (uint64_t)(ks * 16), 1);
                wgmma_ss_n128(acc, a_hi + (uint64_t)(ks * 16), b_hi + (uint64_t)(ks * 16), 1);
            }
            wgmma_commit();
            wgmma_wait<1>();                               // k-step kt - 1 has finished reading its stage
            if (kt >= 1 && t == 0) mbar_arrive(&bars->empty[(kt - 1) % kStages]);
        }
        wgmma_wait<0>();
        fence_regs(acc);
        // ---- epilogue: thread holds rows r, r + 8 and column pairs 8 j + 2 (t % 4) of the tile
        const int q = t & 3;
        const float* b = bias + nt * 128;
        int2 sw[16];                                         // column scales of the training GEMMs, loaded up front
#pragma unroll
        for (int j = 0; j < 16; ++j) sw[j] = kScaled && nt * 128 + 8 * j + 2 * q < N ? __ldg(reinterpret_cast<const int2*>(w_exp + nt * 128 + 8 * j + 2 * q)) : make_int2(0, 0);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2) + h * 8, row = m0 + r;
            const int sa = kScaled && row < M ? a_exp[row] : 0;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int col = 8 * j + 2 * q;
                if (pack_img != 3 && (row >= M || nt * 128 + col >= N)) continue;   // padded rows / N tile (N % 4 == 0)
                float a0 = acc[4 * j + 2 * h], a1 = acc[4 * j + 2 * h + 1];
                if (kScaled) {       // undo the operand scales: exact unless the product leaves fp32's range
                    a0 = split_unscale(a0, -(sa + sw[j].x));
                    a1 = split_unscale(a1, -(sa + sw[j].y));
                }
                float x0 = a0 + b[col], x1 = a1 + b[col + 1];
                if (relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
                if (pack_img == 3) {
                    // C as the next layer's A operand image: 32 columns are exactly one k-step of that layer
                    if (row >= M) { x0 = 0.f; x1 = 0.f; }
                    uint8_t* blk = reinterpret_cast<uint8_t*>(C) + ((size_t)blockIdx.y * out_kt_total + out_kt_off + nt * 4 + (col >> 5)) * (size_t)kStageA;
                    const uint32_t off = (uint32_t)(r >> 3) * 512u + (uint32_t)((col & 31) >> 3) * 128u + (uint32_t)(r & 7) * 16u + (uint32_t)(col & 7) * 2u;
                    uint32_t hi, lo;
                    split_half2(x0, x1, hi, lo);
                    *reinterpret_cast<uint32_t*>(blk + off) = hi;
                    *reinterpret_cast<uint32_t*>(blk + kHalf + off) = lo;
                } else if (pack_img) {
                    // C is a per-row fp16 operand image of a [64][64] matrix (row-major index = column of this GEMM):
                    // K-major, LBO 128, SBO 1024 -- the per-query B operand of the pass kernel
                    // pack_img == 2: split precision, 16384 B per row: hi image | lo image
                    uint8_t* img = reinterpret_cast<uint8_t*>(C) + (size_t)row * (pack_img == 2 ? 16384 : 8192);
                    const int gc = nt * 128 + col, o = gc >> 6, i = gc & 63;
                    const uint32_t off = (uint32_t)(o >> 3) * 1024u + (uint32_t)(i >> 3) * 128u + (uint32_t)(o & 7) * 16u + (uint32_t)(i & 7) * 2u;
                    uint32_t hi, lo;
                    split_half2(x0, x1, hi, lo);
                    *reinterpret_cast<uint32_t*>(img + off) = hi;
                    if (pack_img == 2) *reinterpret_cast<uint32_t*>(img + 8192 + off) = lo;
                } else {
                    *reinterpret_cast<float2*>(C + (int64_t)row * ldc + nt * 128 + col) = make_float2(x0, x1);
                }
            }
        }
    }
}

// fp32 W[N][K] -> images [N/128][K/32][hi | lo][128 x 32 fp16, K-major, LBO 128, SBO 512]
__global__ void pack_fc_kernel(const float* __restrict__ W, int N, int K, uint8_t* __restrict__ img) {
    int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)N * K) return;
    int n = (int)(e / K), k = (int)(e % K);
    int nt = n >> 7, r = n & 127, kt = k / kBK, kk = k % kBK;
    size_t off = ((size_t)nt * (K / kBK) + kt) * kStageB + (size_t)(r >> 3) * 512 + (size_t)(kk >> 3) * 128 + (size_t)(r & 7) * 16 + (size_t)(kk & 7) * 2;
    const float w = W[e];
    const __half h = __float2half_rn(w);
    *reinterpret_cast<__half*>(img + off) = h;
    *reinterpret_cast<__half*>(img + off + kHalf) = __float2half_rn(w - __half2float(h));
}

// fp32 activations A[M][K] (+ optional bias / ReLU) -> A operand images [ceil(M/128)][K/32][hi | lo][128 x 32 fp16, K-major,
// LBO 128, SBO 512]; rows >= M are zero.  One CTA per (row tile, k-step): 8 lanes read one row's 128 bytes (coalesced).
__global__ void __launch_bounds__(256) pack_a_kernel(const float* __restrict__ A, int lda, int M, int K, const float* __restrict__ in_bias,
                                                     int in_relu, uint8_t* __restrict__ img) {
    const int kt = blockIdx.x, mt = blockIdx.y, c = threadIdx.x & 7;
    uint8_t* blk = img + ((size_t)mt * (K / kBK) + kt) * (size_t)kStageA;
    float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (in_bias) b4 = __ldg(reinterpret_cast<const float4*>(in_bias + kt * kBK + c * 4));
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = (threadIdx.x >> 3) + 32 * i, row = mt * 128 + r;
        float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row < M) {
            x = *reinterpret_cast<const float4*>(A + (int64_t)row * lda + kt * kBK + c * 4);
            x.x += b4.x; x.y += b4.y; x.z += b4.z; x.w += b4.w;
            if (in_relu) { x.x = fmaxf(x.x, 0.f); x.y = fmaxf(x.y, 0.f); x.z = fmaxf(x.z, 0.f); x.w = fmaxf(x.w, 0.f); }
        }
        const __half2 h0 = __floats2half2_rn(x.x, x.y), h1 = __floats2half2_rn(x.z, x.w);
        const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
        const __half2 l0 = __floats2half2_rn(x.x - f0.x, x.y - f0.y), l1 = __floats2half2_rn(x.z - f1.x, x.w - f1.y);
        const uint32_t off = (uint32_t)(r >> 3) * 512u + (uint32_t)(c >> 1) * 128u + (uint32_t)(r & 7) * 16u + (uint32_t)(c & 1) * 8u;
        *reinterpret_cast<uint2*>(blk + off) = make_uint2(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1));
        *reinterpret_cast<uint2*>(blk + kHalf + off) = make_uint2(*reinterpret_cast<const uint32_t*>(&l0), *reinterpret_cast<const uint32_t*>(&l1));
    }
}

// same image for N rows padded with zeros to Npad (multiple of 128), row n scaled by 2^w_exp[n] (model.cuh, split_exp)
__global__ void pack_fc_pad_kernel(const float* __restrict__ W, int N, int Npad, int K, const int* __restrict__ w_exp,
                                   uint8_t* __restrict__ img) {
    int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)Npad * K) return;
    int n = (int)(e / K), k = (int)(e % K);
    int nt = n >> 7, r = n & 127, kt = k / kBK, kk = k % kBK;
    size_t off = ((size_t)nt * (K / kBK) + kt) * kStageB + (size_t)(r >> 3) * 512 + (size_t)(kk >> 3) * 128 + (size_t)(r & 7) * 16 + (size_t)(kk & 7) * 2;
    const float2 f = split_factors(n < N ? w_exp[n] : 0);
    const float w = n < N ? W[e] * f.x * f.y : 0.f;
    const __half h = __float2half_rn(w);
    *reinterpret_cast<__half*>(img + off) = h;
    *reinterpret_cast<__half*>(img + off + kHalf) = __float2half_rn(w - __half2float(h));
}

}  // namespace

bool fc_tc_supported(int N, int K) { return (N % 128 == 0) && (K % kBK == 0) && N >= 128 && K >= kBK; }

uint8_t* fc_tc_pack(const Layer& L, std::vector<void*>& allocs) {
    P2S_CHECK(fc_tc_supported(L.cout, L.cin), "layer shape not supported by the tensor-core FC kernel");
    void* p = nullptr;
    P2S_CUDA(cudaMalloc(&p, (size_t)L.cout * L.cin * 4));
    allocs.push_back(p);
    P2S_LAUNCH(pack_fc_kernel, (unsigned)cdiv((int64_t)L.cout * L.cin, 256), 256, 0, 0, L.W, L.cout, L.cin, (uint8_t*)p);
    return (uint8_t*)p;
}

void fc_tc_init() {
    set_smem_attr_once(fc_tc_kernel<false>, kFcSmem);
    set_smem_attr_once(fc_tc_kernel<true>, kFcSmem);
}

void launch_fc_tc(const float* A, int lda, const uint8_t* Wimg, const float* bias, float* C, int ldc,
                  int64_t M, int N, int K, bool relu, cudaStream_t st, int pack_img, const float* in_bias, bool in_relu,
                  const int* a_exp, const int* w_exp) {
    if (M <= 0) return;
    P2S_CHECK(!(a_exp || w_exp) || (a_exp && w_exp && !pack_img && !in_bias), "operand scales need both exponents and a plain fp32 C");
    const bool padded_ok = !pack_img && N % 4 == 0 && N >= 64 && K % kBK == 0;   // partial last N tile (training GEMMs)
    P2S_CHECK((fc_tc_supported(N, K) || padded_ok) && lda % 4 == 0 && (pack_img ? N == 4096 : ldc % 4 == 0), "bad FC shape for the tensor-core kernel");
    P2S_CHECK(cdiv(M, 128) <= 65535, "too many rows for one launch");
    dim3 grid((unsigned)cdiv(N, 128), (unsigned)cdiv(M, 128), 1);
    if (a_exp)
        P2S_LAUNCH(fc_tc_kernel<true>, grid, kFcThreads, kFcSmem, st, A, lda, Wimg, bias, C, ldc, (int)M, N, K, relu ? 1 : 0, pack_img, in_bias,
                   in_relu ? 1 : 0, (const uint8_t*)nullptr, 0, 0, a_exp, w_exp);
    else
        P2S_LAUNCH(fc_tc_kernel<false>, grid, kFcThreads, kFcSmem, st, A, lda, Wimg, bias, C, ldc, (int)M, N, K, relu ? 1 : 0, pack_img, in_bias,
                   in_relu ? 1 : 0, (const uint8_t*)nullptr, 0, 0, (const int*)nullptr, (const int*)nullptr);
}

size_t fc_tc_a_image_bytes(int64_t M, int K) { return (size_t)cdiv(M, 128) * (size_t)(K / kBK) * kStageA; }

void launch_pack_a(const float* A, int lda, int64_t M, int K, const float* in_bias, bool in_relu, uint8_t* img, cudaStream_t st) {
    if (M <= 0) return;
    P2S_CHECK(K % kBK == 0 && lda % 4 == 0 && cdiv(M, 128) <= 65535, "bad shape for the A operand image");
    dim3 grid((unsigned)(K / kBK), (unsigned)cdiv(M, 128), 1);
    P2S_LAUNCH(pack_a_kernel, grid, 256, 0, st, A, lda, (int)M, K, in_bias, in_relu ? 1 : 0, img);
}

// A given as an operand image (launch_pack_a or a previous layer's out_mode 3).  out_mode: 0 fp32 row-major C (ldc), 1 / 2 the
// per-query operand image of the pass kernel (N == 4096), 3 the next layer's A image (k-steps out_kt_off.. of out_kt_total).
void launch_fc_tc_img(const uint8_t* Aimg, const uint8_t* Wimg, const float* bias, void* C, int ldc, int64_t M, int N, int K,
                      bool relu, cudaStream_t st, int out_mode, int out_kt_total, int out_kt_off) {
    if (M <= 0) return;
    P2S_CHECK(fc_tc_supported(N, K) && Aimg && (out_mode == 0 ? ldc % 4 == 0 : (out_mode == 3 ? out_kt_off + N / 32 <= out_kt_total : N == 4096)),
              "bad FC shape for the tensor-core kernel (operand-image mode)");
    P2S_CHECK(cdiv(M, 128) <= 65535, "too many rows for one launch");
    dim3 grid((unsigned)(N / 128), (unsigned)cdiv(M, 128), 1);
    P2S_LAUNCH(fc_tc_kernel<false>, grid, kFcThreads, kFcSmem, st, (const float*)nullptr, 0, Wimg, bias, reinterpret_cast<float*>(C), ldc, (int)M, N, K, relu ? 1 : 0,
               out_mode, (const float*)nullptr, 0, Aimg, out_kt_total, out_kt_off, (const int*)nullptr, (const int*)nullptr);
}

// images of a raw fp32 matrix W[N][K] (device pointer)
uint8_t* fc_tc_pack_raw(const float* W, int N, int K, std::vector<void*>& allocs) {
    P2S_CHECK(fc_tc_supported(N, K), "layer shape not supported by the tensor-core FC kernel");
    void* p = nullptr;
    P2S_CUDA(cudaMalloc(&p, (size_t)N * K * 4));
    allocs.push_back(p);
    P2S_LAUNCH(pack_fc_kernel, (unsigned)cdiv((int64_t)N * K, 256), 256, 0, 0, W, N, K, (uint8_t*)p);
    return (uint8_t*)p;
}

namespace {

// split_exp(max |x|) per row: one warp per row (W may sit at any float offset of the flat parameter buffer: scalar loads)
__global__ void __launch_bounds__(256) split_exp_rows_kernel(const float* __restrict__ X, int ld, int64_t rows, int cols,
                                                             int* __restrict__ out) {
    const int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (r >= rows) return;
    const float* x = X + r * ld;
    float m = 0.f;
    for (int c = threadIdx.x & 31; c < cols; c += 32) m = fmaxf(m, fabsf(x[c]));
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) out[r] = split_exp(m);
}

// max |x| per column: a CTA covers 128 columns (32 lanes x float4) of a slice of rows; per-CTA maxima are merged with
// atomicMax on the float bits (order-preserving for non-negative floats)
__global__ void __launch_bounds__(256) absmax_cols_kernel(const float* __restrict__ X, int ld, int64_t rows, int cols,
                                                          unsigned* __restrict__ out) {
    __shared__ float4 red[8][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int c = blockIdx.x * 128 + lane * 4;
    float4 m = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < cols) {
        for (int64_t r = (int64_t)blockIdx.y * 8 + w; r < rows; r += (int64_t)gridDim.y * 8) {
            const float4 v = *reinterpret_cast<const float4*>(X + r * ld + c);
            m.x = fmaxf(m.x, fabsf(v.x)); m.y = fmaxf(m.y, fabsf(v.y)); m.z = fmaxf(m.z, fabsf(v.z)); m.w = fmaxf(m.w, fabsf(v.w));
        }
    }
    red[w][lane] = m;
    __syncthreads();
    if (w == 0 && c < cols) {
#pragma unroll
        for (int i = 1; i < 8; ++i) {
            const float4 o = red[i][lane];
            m.x = fmaxf(m.x, o.x); m.y = fmaxf(m.y, o.y); m.z = fmaxf(m.z, o.z); m.w = fmaxf(m.w, o.w);
        }
        atomicMax(out + c, __float_as_uint(m.x));
        atomicMax(out + c + 1, __float_as_uint(m.y));
        atomicMax(out + c + 2, __float_as_uint(m.z));
        atomicMax(out + c + 3, __float_as_uint(m.w));
    }
}

}  // namespace

void launch_split_exp_rows(const float* X, int ld, int64_t rows, int cols, int* out, cudaStream_t st) {
    if (rows <= 0) return;
    P2S_LAUNCH(split_exp_rows_kernel, (unsigned)cdiv(rows, 8), 256, 0, st, X, ld, rows, cols, out);
}

void launch_absmax_cols(const float* X, int ld, int64_t rows, int cols, unsigned* out, cudaStream_t st) {
    P2S_CHECK(cols % 4 == 0 && ld % 4 == 0 && (uintptr_t)X % 16 == 0, "absmax_cols: unaligned rows");
    P2S_CUDA(cudaMemsetAsync(out, 0, sizeof(unsigned) * (size_t)cols, st));
    if (rows <= 0) return;
    const int64_t cb = cdiv(cols, 128);
    const int64_t slices = std::min<int64_t>(cdiv(rows, 64), std::max<int64_t>(1, cdiv(8 * (int64_t)sm_count(), cb)));
    P2S_LAUNCH(absmax_cols_kernel, dim3((unsigned)cb, (unsigned)std::min<int64_t>(slices, 65535)), 256, 0, st, X, ld, rows, cols, out);
}

// Split-precision tensor-core GEMM for weights that change between calls (training): takes the row scales of A and W,
// packs the scaled W [N][K] into a reusable scratch image on `st`, then runs fc_tc_kernel with the scaled A rows (see
// split_exp in model.cuh).  Stream order makes the scratch reuse safe.  bias may be null.
// Every output element meets |C - C_exact| <= gamma_K sum_k |a_k b_k| + 2^-40 K max_k |a_k| max_k |b_k| (up to the
// tensor cores' accumulation order) at any operand scale inside fp32's normal range.
bool gemm_nt_tc_ok(const float* A, int lda, const float* C, int ldc, int64_t M, int N, int K) {
    static const bool disabled = env_flag("P2S_TRAIN_GEMM_FP32");
    return !disabled && N % 4 == 0 && N >= 64 && K % kBK == 0 && K >= kBK && N <= 4096 && M >= 128 && M < (int64_t)1 << 31 && lda % 4 == 0 && ldc % 4 == 0 &&
           ((uintptr_t)A % 16 == 0) && ((uintptr_t)C % 16 == 0);
}

void launch_gemm_nt_tc(const float* A, int lda, const float* W, const float* bias, float* C, int ldc, int64_t M, int N,
                       int K, bool relu, cudaStream_t st) {
    static thread_local std::vector<Workspace> t_ws;
    static thread_local std::vector<DevBuf> t_zeros;   // 4096 zeros per device: the bias of calls without one
    Workspace& ws = for_device(t_ws).begin(st);
    const int Npad = (int)(cdiv(N, 128) * 128);
    uint8_t* wimg = ws.get<uint8_t>((int64_t)Npad * K * 4);
    int* a_exp = ws.get<int>(M + N + 2);
    int* w_exp = a_exp + ((M + 1) & ~(int64_t)1);          // 8-byte aligned: the epilogue reads column pairs
    fc_tc_init();
    if (!bias) {
        DevBuf& z = for_device(t_zeros);
        const bool fresh = !z.p;
        bias = reinterpret_cast<float*>(ws.grow(z, 4096 * sizeof(float)));
        if (fresh) P2S_CUDA(cudaMemsetAsync(z.p, 0, 4096 * sizeof(float), st));
    }
    launch_split_exp_rows(A, lda, M, K, a_exp, st);
    launch_split_exp_rows(W, K, N, K, w_exp, st);
    P2S_LAUNCH(pack_fc_pad_kernel, (unsigned)cdiv((int64_t)Npad * K, 256), 256, 0, st, W, N, Npad, K, w_exp, wimg);
    launch_fc_tc(A, lda, wimg, bias, C, ldc, M, N, K, relu, st, 0, nullptr, false, a_exp, w_exp);
}

}  // namespace p2s
