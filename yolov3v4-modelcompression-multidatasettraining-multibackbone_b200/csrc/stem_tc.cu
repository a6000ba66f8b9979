// Fused tensor-core stem (reference models.py:52-110, the first [convolutional] block: Conv2d(3->C, k, s) + BN + act).
//
// The image (NCHW; fp32, fp16 or uint8) has too few channels for a TMA im2col gather: a pixel is 6 bytes.  Here the
// CTA's own threads build the im2col tile in shared memory instead, straight from the image, so nothing but the image
// is read and nothing but the NHWC fp16 output is written (the two-pass variant in conv_tc.cu writes and re-reads a
// 64-byte-per-pixel im2col matrix in HBM).
//
//   A[128 output pixels][32]  : row = one output pixel, columns (kh*K + kw)*Cin + c, zero padded to 32 (64 bytes),
//                               written with st.shared in the canonical K-major SWIZZLE_64B layout
//   B[BLOCK_N out channels][32]: the BN-folded weights, same layout, loaded once per CTA
//   D = A * B^T               : two wgmma.mma_async pairs (M = 2 x 64, K = 2 x 16) per tile, fp32 accumulators in
//                               registers, staged through shared memory for the row-per-thread epilogue
//
// Persistent CTAs (one per SM).  STEM_NG warpgroups of "worker" warps; a group owns every STEM_NG-th tile of the CTA
// and runs a three-stage software pipeline per thread (thread = one pixel row of the tile):
//     issue the image loads of tile j      (27 predicated LDGs for 3x3 RGB)
//     epilogue of tile j-1                 (staged accumulators -> bias/act -> 64-byte fp16 row), overlapping the
//                                          loads in flight
//     convert + store the A row of tile j  -> fence.proxy.async -> group barrier -> wgmma -> accumulators to smem
#include <cmath>

#include "common.cuh"

namespace b2y {

enum { STEM_X_F32 = 0, STEM_X_F16 = 1, STEM_X_U8 = 2 };
constexpr int STEM_NG = 4;      // worker warpgroups per CTA

struct StemParams {
    const void* x;        // NCHW image
    float x_div;          // value = raw / x_div  (256 for uint8 images: reference test.py:95, train.py:348; 1 otherwise)
    float x_mul;          // host: 1/x_div when that multiplication gives the same fp16 as the division, else 0
    int B, H, W, Ho, Wo, stride, pad;
    const __half* w;      // [BLOCK_N][32] fp16, column (kh*K + kw)*Cin + c  (b2y_pack_stem_weights)
    const float* bias;    // [Cout] or null
    __half* out;          // NHWC fp16, or int8 codes when out_i8 (first layer of the INT8 graph)
    int out_i8;
    float q_scale, q_mul, q_lo, q_hi;   // q = clamp(round_half_away(v / q_scale)); q_mul = 1/q_scale when that is exact
    long long out_pitch;
    int Cout;
    int act;
    float slope;
    long long M_total;    // B*Ho*Wo
    int num_tiles;
};

__device__ __noinline__ float stem_mish(float x) { return mish_f(x); }

template <typename T>
__device__ __forceinline__ float stem_ld(const T* p);
template <>
__device__ __forceinline__ float stem_ld<float>(const float* p) { return __ldg(p); }
template <>
__device__ __forceinline__ float stem_ld<__half>(const __half* p) { return __half2float(__ldg(p)); }
template <>
__device__ __forceinline__ float stem_ld<uint8_t>(const uint8_t* p) { return (float)__ldg(p); }

__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

template <typename XT, int CIN, int K, int BLOCK_N>
__global__ void __launch_bounds__(128 * STEM_NG, 1) stem_fused_kernel(const __grid_constant__ StemParams p) {
    constexpr int KK = CIN * K * K;            // <= 32
    constexpr int A_BYTES = 128 * 64;
    constexpr int B_BYTES = BLOCK_N * 64;
    constexpr int ACC_BYTES = 128 * BLOCK_N * 4;

    // smem: [STEM_NG A tiles] [B] [STEM_NG accumulator tiles]
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* smem_b = smem + STEM_NG * A_BYTES;
    uint8_t* smem_acc = smem_b + B_BYTES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    // weights -> smem (SWIZZLE_64B: 16-byte chunk index ^= (row >> 1) & 3)
    for (int i = threadIdx.x; i < BLOCK_N * 4; i += blockDim.x) {
        const int row = i >> 2, ch = i & 3;
        const uint4 v = row < p.Cout ? __ldg(reinterpret_cast<const uint4*>(p.w) + i) : make_uint4(0, 0, 0, 0);
        *reinterpret_cast<uint4*>(smem_b + row * 64 + ((ch ^ ((row >> 1) & 3)) << 4)) = v;
    }
    // The bias rides in the GEMM: A carries 1.0 in two spare K columns and B the bias split in two fp16 terms
    // (hi + lo reproduces the fp32 bias to ~2^-22), so the epilogue has no bias loads or adds.
    constexpr bool FOLD_BIAS = KK + 2 <= 32;
    if (FOLD_BIAS) {
        __syncthreads();
        for (int row = threadIdx.x; row < BLOCK_N; row += blockDim.x) {
            const float bf = (p.bias != nullptr && row < p.Cout) ? __ldg(p.bias + row) : 0.f;
            const __half hi = __float2half_rn(bf);
            const __half lo = __float2half_rn(bf - __half2float(hi));
#pragma unroll
            for (int t = 0; t < 2; ++t) {
                const int col = KK + t;
                *reinterpret_cast<__half*>(smem_b + row * 64 + (((col >> 3) ^ ((row >> 1) & 3)) << 4) + (col & 7) * 2) =
                    t == 0 ? hi : lo;
            }
        }
    }
    fence_proxy_async_smem();
    __syncthreads();
    const int my_tiles = (p.num_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // tiles of this CTA

    {
        // ===================== workers: build A rows, MMA, epilogue =====================
        const int g = warp >> 2;
        const int ew = warp & 3;                 // row quarter of the tile
        const int r_in_tile = ew * 32 + lane;
        const XT* xin = reinterpret_cast<const XT*>(p.x);
        const int plane = p.H * p.W;             // 32-bit image indexing (host checks B*Cin*H*W < 2^31)
        const int W = p.W, H = p.H;
        const bool use_mul = p.x_mul != 0.f && p.x_mul != 1.f;
        const float mul = p.x_mul;
        const bool exact_div = p.x_div != 1.f && p.x_mul == 0.f;
        const int act = p.act;
        const float slope = p.slope;
        const bool leaky_max = act == B2Y_ACT_LEAKY && slope >= 0.f && slope <= 1.f;
        const unsigned HoWo = (unsigned)(p.Ho * p.Wo), Wo = (unsigned)p.Wo;
        const unsigned M_total = (unsigned)p.M_total;
        const int my_group_tiles = (my_tiles - g + STEM_NG - 1) / STEM_NG;
        uint8_t* const arow = smem + g * A_BYTES + r_in_tile * 64;
        uint8_t* const acc_tile = smem_acc + g * ACC_BYTES;
        const int sw = (r_in_tile >> 1) & 3;
        const int tid_wg = (int)threadIdx.x & 127;
        const uint32_t bar_id = 1 + g;           // named barrier of this group
        const uint64_t desc_base = smem_desc_base(16, 8 * 64, swizzle_layout_type(64));
        const uint32_t a_addr = smem_u32(smem + g * A_BYTES);
        const uint64_t adesc0 = smem_desc_at(desc_base, a_addr), adesc1 = smem_desc_at(desc_base, a_addr + 64 * 64);
        const uint64_t bdesc = smem_desc_at(desc_base, smem_u32(smem_b));

        unsigned prev_row = 0;
        for (int j = 0; j <= my_group_tiles; ++j) {
            float raw[KK];
            const bool have = j < my_group_tiles;
            unsigned row = 0;
            if (have) {
                const unsigned tile = blockIdx.x + (unsigned)(g + j * STEM_NG) * gridDim.x;
                row = tile * 128u + (unsigned)r_in_tile;
                // ---- 1. issue the image loads of tile j
                const bool row_ok = row < M_total;
                const unsigned rr = row_ok ? row : 0u;
                const unsigned n = rr / HoWo;
                const unsigned rem = rr - n * HoWo;
                const unsigned yo = rem / Wo, xo = rem - yo * Wo;
                const int y0 = (int)yo * p.stride - p.pad, x0 = (int)xo * p.stride - p.pad;
                const int base = (int)n * CIN * plane + y0 * W + x0;
                bool xok[K];
#pragma unroll
                for (int kw = 0; kw < K; ++kw) xok[kw] = (unsigned)(x0 + kw) < (unsigned)W;
#pragma unroll
                for (int kh = 0; kh < K; ++kh) {
                    const bool yok = row_ok && (unsigned)(y0 + kh) < (unsigned)H;
#pragma unroll
                    for (int c = 0; c < CIN; ++c) {
                        const XT* prow = xin + (base + kh * W + c * plane);
#pragma unroll
                        for (int kw = 0; kw < K; ++kw)
                            raw[(kh * K + kw) * CIN + c] = (yok && xok[kw]) ? stem_ld<XT>(prow + kw) : 0.f;
                    }
                }
            }
            // ---- 2. epilogue of tile j-1 (accumulators staged at the end of the previous iteration)
            if (j > 0) {
                const bool prow_ok = prev_row < M_total;
                __half* orow = p.out + (long long)prev_row * p.out_pitch;
#pragma unroll 1
                for (int c0 = 0; c0 < BLOCK_N; c0 += 32) {
                    uint32_t acc[32];
                    stage_row32<BLOCK_N>(acc_tile, r_in_tile, c0, acc);
                    float v[32];
#pragma unroll
                    for (int q = 0; q < 32; ++q) v[q] = __uint_as_float(acc[q]);
                    if (!FOLD_BIAS && p.bias != nullptr) {
#pragma unroll
                        for (int q = 0; q < 32; ++q)
                            if (c0 + q < p.Cout) v[q] += __ldg(p.bias + c0 + q);
                    }
                    if (leaky_max) {
#pragma unroll
                        for (int q = 0; q < 32; ++q) v[q] = fmaxf(v[q], v[q] * slope);
                    } else {
                        switch (act) {
                            case B2Y_ACT_LEAKY:
#pragma unroll
                                for (int q = 0; q < 32; ++q) v[q] = v[q] > 0.f ? v[q] : v[q] * slope;
                                break;
                            case B2Y_ACT_MISH:
#pragma unroll
                                for (int q = 0; q < 32; ++q) v[q] = mish_f(v[q]);   // inlined: 32 independent chains
                                break;
                            case B2Y_ACT_RELU:
#pragma unroll
                                for (int q = 0; q < 32; ++q) v[q] = fmaxf(v[q], 0.f);
                                break;
                            case B2Y_ACT_RELU6:
#pragma unroll
                                for (int q = 0; q < 32; ++q) v[q] = fminf(fmaxf(v[q], 0.f), 6.f);
                                break;
                            case B2Y_ACT_HSWISH:
#pragma unroll
                                for (int q = 0; q < 32; ++q) v[q] = v[q] * (fminf(fmaxf(v[q] + 3.f, 0.f), 6.f) / 6.f);
                                break;
                            case B2Y_ACT_SWISH:
#pragma unroll
                                for (int q = 0; q < 32; ++q) v[q] = v[q] * sigmoid_f(v[q]);
                                break;
                            default:
                                break;
                        }
                    }
                    if (prow_ok && p.out_i8) {
                        // requantise (ptq_cos.py:14-20 round half away from zero, then clamp) and store 32 codes
                        int8_t* op8 = reinterpret_cast<int8_t*>(p.out) + (long long)prev_row * p.out_pitch + c0;
                        const int nvalid = min(32, p.Cout - c0);
                        uint32_t w[8];
#pragma unroll
                        for (int t = 0; t < 8; ++t) {
                            uint32_t word = 0;
#pragma unroll
                            for (int e = 0; e < 4; ++e) {
                                const float vv = v[t * 4 + e];
                                float q = p.q_mul != 0.f ? vv * p.q_mul : __fdiv_rn(vv, p.q_scale);
                                q = copysignf(floorf(fabsf(q) + 0.5f), q);
                                q = fminf(fmaxf(q, p.q_lo), p.q_hi);
                                word |= ((uint32_t)(uint8_t)(int8_t)(int)q) << (8 * e);
                            }
                            w[t] = word;
                        }
                        if ((nvalid & 15) == 0 && ((reinterpret_cast<uintptr_t>(op8) & 15) == 0)) {
                            reinterpret_cast<uint4*>(op8)[0] = make_uint4(w[0], w[1], w[2], w[3]);
                            if (nvalid == 32) reinterpret_cast<uint4*>(op8)[1] = make_uint4(w[4], w[5], w[6], w[7]);
                        } else {
#pragma unroll
                            for (int q = 0; q < 32; ++q)
                                if (q < nvalid) op8[q] = (int8_t)((w[q >> 2] >> (8 * (q & 3))) & 0xff);
                        }
                    } else if (prow_ok) {
                        __half* op = orow + c0;
                        const int nvalid = min(32, p.Cout - c0);
                        if ((nvalid & 7) == 0 && ((reinterpret_cast<uintptr_t>(op) & 15) == 0)) {
#pragma unroll
                            for (int q = 0; q < 4; ++q) {
                                if (q * 8 >= nvalid) break;
                                uint4 u;
                                __half2* h2 = reinterpret_cast<__half2*>(&u);
#pragma unroll
                                for (int t = 0; t < 4; ++t) h2[t] = __floats2half2_rn(v[q * 8 + t * 2], v[q * 8 + t * 2 + 1]);
                                reinterpret_cast<uint4*>(op)[q] = u;
                            }
                        } else {
#pragma unroll
                            for (int q = 0; q < 32; ++q)
                                if (q < nvalid) op[q] = __float2half_rn(v[q]);
                        }
                    }
                }
            }
            // ---- 3. convert + store the A row of tile j, multiply, stage the accumulators
            if (have) {
                // every thread of the group is done with the staged accumulators and the A tile of tile j-1
                named_bar_sync(bar_id, 128);
                if (exact_div) {
#pragma unroll
                    for (int k0 = 0; k0 < KK; ++k0) raw[k0] = __fdiv_rn(raw[k0], p.x_div);
                } else if (use_mul) {
#pragma unroll
                    for (int k0 = 0; k0 < KK; ++k0) raw[k0] *= mul;
                }
#pragma unroll
                for (int ch = 0; ch < 4; ++ch) {
                    uint4 u;
                    __half2* h2 = reinterpret_cast<__half2*>(&u);
#pragma unroll
                    for (int t = 0; t < 4; ++t) {
                        float ab[2];
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int k0 = ch * 8 + t * 2 + e;
                            float a = 0.f;
                            if (k0 < KK) {
                                a = raw[k0 < KK ? k0 : 0];
                            } else if (FOLD_BIAS && k0 < KK + 2) {
                                a = 1.f;
                            }
                            ab[e] = a;
                        }
                        h2[t] = __floats2half2_rn(ab[0], ab[1]);
                    }
                    *reinterpret_cast<uint4*>(arow + ((ch ^ sw) << 4)) = u;
                }
                fence_proxy_async_smem();     // generic-proxy stores -> visible to the tensor core (async proxy)
                named_bar_sync(bar_id, 128);
                float acc0[BLOCK_N / 2], acc1[BLOCK_N / 2];
                wgmma_fence();
                wgmma_ss<BLOCK_N, 0, 0>(acc0, adesc0, bdesc, 0u);
                wgmma_ss<BLOCK_N, 0, 0>(acc0, adesc0 + 2, bdesc + 2, 1u);
                wgmma_ss<BLOCK_N, 0, 0>(acc1, adesc1, bdesc, 0u);
                wgmma_ss<BLOCK_N, 0, 0>(acc1, adesc1 + 2, bdesc + 2, 1u);
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_acc(acc0);
                wgmma_fence_acc(acc1);
                frag_to_stage<BLOCK_N>(acc0, acc_tile, 0, tid_wg);
                frag_to_stage<BLOCK_N>(acc1, acc_tile, 64, tid_wg);
                named_bar_sync(bar_id, 128);
                prev_row = row;
            }
        }
    }
}

template <typename XT, int CIN, int K, int BLOCK_N>
static int stem_launch(const StemParams& p, cudaStream_t st) {
    constexpr int SMEM = 1024 + STEM_NG * 128 * 64 + BLOCK_N * 64 + STEM_NG * 128 * BLOCK_N * 4;
    auto kern = stem_fused_kernel<XT, CIN, K, BLOCK_N>;
    static unsigned long long attr_set = 0;      // one bit per device: the attribute is per (function, device)
    if (b2y_first_use_on_device(attr_set)) {
        B2Y_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    }
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int grid = p.num_tiles < sms ? p.num_tiles : sms;
    kern<<<grid, 128 * STEM_NG, SMEM, st>>>(p);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

template <typename XT>
static int stem_dispatch(const StemParams& p, int cin, int k, cudaStream_t st) {
#define B2Y_STEM_CASE(CI, KK)                                                                  \
    if (cin == CI && k == KK) {                                                                 \
        if (p.Cout <= 32) return stem_launch<XT, CI, KK, 32>(p, st);                           \
        return stem_launch<XT, CI, KK, 64>(p, st);                                             \
    }
    B2Y_STEM_IM2COL_SHAPES(B2Y_STEM_CASE)
#undef B2Y_STEM_CASE
    return B2Y_ERR_UNSUPPORTED;
}

}  // namespace b2y

using namespace b2y;

// x: NCHW image in x_dtype (B2Y_STEM_X_*), value = raw / x_div.  w_stem: the [out_c][32] rows of
// b2y_pack_stem_weights ((in_c, k) in B2Y_STEM_IM2COL_SHAPES).  y: NHWC fp16.
static int stem_fused_common(const b2y_conv_desc* d, const void* x_nchw, int x_dtype, float x_div, const void* w_stem,
                             const float* bias, void* y, int out_i8, float q_scale, float q_lo, float q_hi, void* stream) {
    if (!d || !x_nchw || !w_stem || !y) return B2Y_ERR_INVALID;
    if (d->in_c * d->ksize * d->ksize > 32 || d->out_c > 64 || x_div == 0.f) return B2Y_ERR_UNSUPPORTED;
    if (reinterpret_cast<uintptr_t>(w_stem) & 15) return B2Y_ERR_INVALID;
    const int Ho = (d->in_h + 2 * d->pad - d->ksize) / d->stride + 1;
    const int Wo = (d->in_w + 2 * d->pad - d->ksize) / d->stride + 1;
    if (Ho != d->out_h || Wo != d->out_w) return B2Y_ERR_INVALID;
    StemParams p{};
    p.x = x_nchw;
    p.x_div = x_div;
    {
        // raw * (1/x_div) == raw / x_div exactly when x_div is a power of two; for uint8 codes / 255 the two round to the
        // same fp16 for all 256 codes (checked exhaustively); anything else takes the IEEE division
        int ex = 0;
        const float mant = frexpf(fabsf(x_div), &ex);
        if (mant == 0.5f || (x_dtype == STEM_X_U8 && x_div == 255.f)) p.x_mul = 1.f / x_div;
    }
    p.B = d->batch;
    p.H = d->in_h;
    p.W = d->in_w;
    p.Ho = Ho;
    p.Wo = Wo;
    p.stride = d->stride;
    p.pad = d->pad;
    p.w = reinterpret_cast<const __half*>(w_stem);
    p.bias = bias;
    p.out = reinterpret_cast<__half*>(y);
    p.out_pitch = d->out_pitch;
    p.out_i8 = out_i8;
    if (out_i8) {
        if (q_scale <= 0.f) return B2Y_ERR_INVALID;
        int ex = 0;
        p.q_scale = q_scale;
        p.q_mul = frexpf(q_scale, &ex) == 0.5f ? 1.f / q_scale : 0.f;
        p.q_lo = q_lo;
        p.q_hi = q_hi;
    }
    p.Cout = d->out_c;
    p.act = d->act;
    p.slope = d->slope;
    p.M_total = (long long)d->batch * Ho * Wo;
    const long long tiles = (p.M_total + 127) / 128;
    if (p.M_total > 0x7fffff00LL || (long long)d->batch * d->in_c * d->in_h * d->in_w > 0x7fffffffLL)
        return B2Y_ERR_UNSUPPORTED;
    p.num_tiles = (int)tiles;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (x_dtype) {
        case STEM_X_F32: return stem_dispatch<float>(p, d->in_c, d->ksize, st);
        case STEM_X_F16: return stem_dispatch<__half>(p, d->in_c, d->ksize, st);
        case STEM_X_U8: return stem_dispatch<uint8_t>(p, d->in_c, d->ksize, st);
        default: return B2Y_ERR_INVALID;
    }
}

// x: NCHW image in x_dtype (B2Y_STEM_X_*), value = raw / x_div.  w_stem: the [out_c][32] rows of
// b2y_pack_stem_weights ((in_c, k) in B2Y_STEM_IM2COL_SHAPES).  y: NHWC fp16.
extern "C" int b2y_stem_conv_fwd_fused(const b2y_conv_desc* d, const void* x_nchw, int x_dtype, float x_div,
                                       const void* w_stem, const float* bias, void* y, void* stream) {
    return stem_fused_common(d, x_nchw, x_dtype, x_div, w_stem, bias, y, 0, 1.f, 0.f, 0.f, stream);
}

// First layer of the INT8 graph (ptq_cos.py:288-296 on the float image): the fake-quantised weights (int8 code x
// power-of-two scale) are exact in fp16 and so are the image values k/256, so every product is exact and only the fp32
// summation order differs from the reference's fp32 convolution; the output is requantised to int8 codes.
extern "C" int b2y_stem_conv_fwd_fused_q(const b2y_conv_desc* d, const void* x_nchw, int x_dtype, float x_div,
                                         const void* w_stem, const float* bias_q, void* y_i8, float out_scale, float lo,
                                         float hi, void* stream) {
    return stem_fused_common(d, x_nchw, x_dtype, x_div, w_stem, bias_q, y_i8, 1, out_scale, lo, hi, stream);
}
