// HBM-bound layers of the Darknet graph on NHWC fp16 activations: stem conv (Cin<=4), weight
// fold/pack, upsample, maxpool, channel copy, add, standalone activations, layout converters.
// All kernels move 16-byte vectors per thread and size the grid from the element count.
#include "b200yolo.h"
#include "common.cuh"

using namespace b2y;

static inline int grid_for(long long n, int block) {
    long long g = (n + block - 1) / block;
    if (g < 1) g = 1;
    if (g > 132LL * 64) g = 132LL * 64;  // grid-stride beyond ~64 CTAs/SM worth of work
    return (int)g;
}

// ------------------------------------------------------------------------------------------------
// Stem: direct conv for Cin <= 4 from the NCHW fp32 image, out NHWC fp16 (models.py:92-113, layer 0)
// ------------------------------------------------------------------------------------------------
template <int CO>
__global__ void __launch_bounds__(128)
stem_conv_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                 __half* __restrict__ y, int B, int Cin, int H, int W, int Cout, int k, int stride, int pad,
                 int Ho, int Wo, long long out_pitch, int act, float slope) {
    extern __shared__ float sw[];  // [Cin*k*k][CO] for the current cout chunk, then bias[CO]
    const int taps = Cin * k * k;
    const long long M = (long long)B * Ho * Wo;
    for (int co0 = 0; co0 < Cout; co0 += CO) {
        __syncthreads();
        for (int i = threadIdx.x; i < taps * CO; i += blockDim.x) {
            int t = i / CO, c = i - t * CO;
            sw[i] = (co0 + c < Cout) ? w[(long long)(co0 + c) * taps + t] : 0.f;
        }
        for (int i = threadIdx.x; i < CO; i += blockDim.x)
            sw[taps * CO + i] = (bias != nullptr && co0 + i < Cout) ? bias[co0 + i] : 0.f;
        __syncthreads();
        for (long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x; m < M;
             m += (long long)gridDim.x * blockDim.x) {
            const int xo = (int)(m % Wo);
            const int yo = (int)((m / Wo) % Ho);
            const int n = (int)(m / ((long long)Wo * Ho));
            float acc[CO];
#pragma unroll
            for (int c = 0; c < CO; ++c) acc[c] = 0.f;
            int t = 0;
            for (int ci = 0; ci < Cin; ++ci) {
                const float* xp = x + ((long long)n * Cin + ci) * H * W;
                for (int kh = 0; kh < k; ++kh) {
                    const int yi = yo * stride - pad + kh;
                    for (int kw = 0; kw < k; ++kw, ++t) {
                        const int xi = xo * stride - pad + kw;
                        float v = 0.f;
                        if (yi >= 0 && yi < H && xi >= 0 && xi < W) v = __ldg(xp + (long long)yi * W + xi);
                        const float4* wp = reinterpret_cast<const float4*>(sw + t * CO);
#pragma unroll
                        for (int c4 = 0; c4 < CO / 4; ++c4) {
                            float4 ww = wp[c4];
                            acc[c4 * 4 + 0] = fmaf(v, ww.x, acc[c4 * 4 + 0]);
                            acc[c4 * 4 + 1] = fmaf(v, ww.y, acc[c4 * 4 + 1]);
                            acc[c4 * 4 + 2] = fmaf(v, ww.z, acc[c4 * 4 + 2]);
                            acc[c4 * 4 + 3] = fmaf(v, ww.w, acc[c4 * 4 + 3]);
                        }
                    }
                }
            }
            __half* op = y + m * out_pitch + co0;
            const int nvalid = min(CO, Cout - co0);
#pragma unroll
            for (int c = 0; c < CO; ++c) acc[c] = apply_act(acc[c] + sw[taps * CO + c], act, slope);
            if (nvalid == CO && ((reinterpret_cast<uintptr_t>(op) & 15) == 0)) {
#pragma unroll
                for (int q = 0; q < CO / 8; ++q) {
                    uint4 u;
                    __half2* h2 = reinterpret_cast<__half2*>(&u);
#pragma unroll
                    for (int j = 0; j < 4; ++j) h2[j] = __floats2half2_rn(acc[q * 8 + j * 2], acc[q * 8 + j * 2 + 1]);
                    reinterpret_cast<uint4*>(op)[q] = u;
                }
            } else {
#pragma unroll
                for (int c = 0; c < CO; ++c)
                    if (c < nvalid) op[c] = __float2half_rn(acc[c]);
            }
        }
    }
}

extern "C" int b2y_stem_conv_fwd(const b2y_conv_desc* d, const float* x_nchw, const float* w, const float* bias,
                                 void* y, void* stream) {
    if (!d || !x_nchw || !w || !y) return B2Y_ERR_INVALID;
    if (d->in_c < 1 || d->in_c > 4 || d->out_dtype != B2Y_OUT_F16) return B2Y_ERR_UNSUPPORTED;
    const int Ho = (d->in_h + 2 * d->pad - d->ksize) / d->stride + 1;
    const int Wo = (d->in_w + 2 * d->pad - d->ksize) / d->stride + 1;
    if (Ho != d->out_h || Wo != d->out_w) return B2Y_ERR_INVALID;
    constexpr int CO = 32;
    const long long M = (long long)d->batch * Ho * Wo;
    const int taps = d->in_c * d->ksize * d->ksize;
    size_t smem = (size_t)(taps * CO + CO) * sizeof(float);
    if (smem > 48 * 1024) return B2Y_ERR_UNSUPPORTED;
    int grid = (int)((M + 127) / 128);
    if (grid > 132 * 16) grid = 132 * 16;
    stem_conv_kernel<CO><<<grid, 128, smem, static_cast<cudaStream_t>(stream)>>>(
        x_nchw, w, bias, reinterpret_cast<__half*>(y), d->batch, d->in_c, d->in_h, d->in_w, d->out_c, d->ksize,
        d->stride, d->pad, Ho, Wo, d->out_pitch, d->act, d->slope);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// ------------------------------------------------------------------------------------------------
// BN fold + OIHW fp32 -> [O][kh][kw][I] fp16 pack (utils/torch_utils.py:65-89)
// ------------------------------------------------------------------------------------------------
__global__ void pack_weights_kernel(const float* __restrict__ w, const float* __restrict__ conv_bias,
                                    const float* __restrict__ gamma, const float* __restrict__ beta,
                                    const float* __restrict__ mean, const float* __restrict__ var, float eps, int O,
                                    int I, int k, __half* __restrict__ wp, float* __restrict__ bias_out,
                                    float* __restrict__ w32) {
    const long long total = (long long)O * I * k * k;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        // idx enumerates the packed layout [o][kh][kw][i]
        const int i = (int)(idx % I);
        long long t = idx / I;
        const int kw = (int)(t % k);
        t /= k;
        const int kh = (int)(t % k);
        const int o = (int)(t / k);
        const long long src = (((long long)o * I + i) * k + kh) * k + kw;
        float s = 1.f;
        if (gamma != nullptr) s = gamma[o] / sqrtf(eps + var[o]);
        const float v = w[src] * s;
        if (wp != nullptr) wp[idx] = __float2half_rn(v);
        if (w32 != nullptr) w32[src] = v;
    }
    if (bias_out != nullptr) {
        for (long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x; o < O;
             o += (long long)gridDim.x * blockDim.x) {
            float b = conv_bias != nullptr ? conv_bias[o] : 0.f;
            if (gamma != nullptr) {
                const float sd = sqrtf(var[o] + eps);
                b = (gamma[o] / sqrtf(eps + var[o])) * b + (beta[o] - gamma[o] * mean[o] / sd);
            }
            bias_out[o] = b;
        }
    }
}

extern "C" int b2y_pack_conv_weights(const float* w_oihw, const float* conv_bias, const float* gamma,
                                     const float* beta, const float* mean, const float* var, float eps, int out_c,
                                     int in_c, int ksize, void* w_packed_f16, float* bias_out, float* w_fp32_out,
                                     void* stream) {
    if (!w_oihw || out_c <= 0 || in_c <= 0 || ksize <= 0) return B2Y_ERR_INVALID;
    if (gamma != nullptr && (!beta || !mean || !var)) return B2Y_ERR_INVALID;
    const long long total = (long long)out_c * in_c * ksize * ksize;
    pack_weights_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        w_oihw, conv_bias, gamma, beta, mean, var, eps, out_c, in_c, ksize, reinterpret_cast<__half*>(w_packed_f16),
        bias_out, w_fp32_out);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// ------------------------------------------------------------------------------------------------
// Upsample nearest (models.py:224-225)
// ------------------------------------------------------------------------------------------------
__global__ void upsample_kernel(const __half* __restrict__ x, long long xp, __half* __restrict__ y, long long yp,
                                int B, int H, int W, int C, int s) {
    const int CV = C / 8;
    const int Ho = H * s, Wo = W * s;
    const long long total = (long long)B * Ho * Wo * CV;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(idx % CV);
        long long pix = idx / CV;
        const int xo = (int)(pix % Wo);
        const int yo = (int)((pix / Wo) % Ho);
        const int n = (int)(pix / ((long long)Wo * Ho));
        const long long ipix = ((long long)n * H + yo / s) * W + xo / s;
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + ipix * xp) + cv);
        reinterpret_cast<uint4*>(y + pix * yp)[cv] = v;
    }
}

extern "C" int b2y_upsample_nearest(const void* x, long long x_pitch, void* y, long long y_pitch, int batch, int in_h,
                                    int in_w, int c, int scale, void* stream) {
    if (!x || !y || c % 8 != 0 || x_pitch % 8 != 0 || y_pitch % 8 != 0 || scale < 1) return B2Y_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15)) return B2Y_ERR_INVALID;
    const long long total = (long long)batch * in_h * scale * in_w * scale * (c / 8);
    upsample_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const __half*>(x), x_pitch, reinterpret_cast<__half*>(y), y_pitch, batch, in_h, in_w, c,
        scale);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// ------------------------------------------------------------------------------------------------
// MaxPool (models.py:207-215)
// ------------------------------------------------------------------------------------------------
__global__ void maxpool_kernel(const __half* __restrict__ x, long long xp, __half* __restrict__ y, long long yp,
                               int B, int H, int W, int C, int k, int stride, int pad, int Ho, int Wo, int zero_pad) {
    const int CV = C / 8;
    const long long total = (long long)B * Ho * Wo * CV;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(idx % CV);
        long long pix = idx / CV;
        const int xo = (int)(pix % Wo);
        const int yo = (int)((pix / Wo) % Ho);
        const int n = (int)(pix / ((long long)Wo * Ho));
        __half2 m[4];
        const __half2 ninf = __half2half2(__ushort_as_half((unsigned short)0xFC00));
#pragma unroll
        for (int j = 0; j < 4; ++j) m[j] = ninf;
        bool touched_pad = false;
        for (int kh = 0; kh < k; ++kh) {
            const int yi = yo * stride - pad + kh;
            for (int kw = 0; kw < k; ++kw) {
                const int xi = xo * stride - pad + kw;
                if (yi < 0 || yi >= H || xi < 0 || xi >= W) {
                    touched_pad = true;
                    continue;
                }
                const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + (((long long)n * H + yi) * W + xi) * xp) + cv);
                const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
                for (int j = 0; j < 4; ++j) m[j] = __hmax2(m[j], h[j]);
            }
        }
        if (zero_pad && touched_pad) {
            const __half2 z = __half2half2(__float2half(0.f));
#pragma unroll
            for (int j = 0; j < 4; ++j) m[j] = __hmax2(m[j], z);
        }
        uint4 o;
        __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int j = 0; j < 4; ++j) oh[j] = m[j];
        reinterpret_cast<uint4*>(y + pix * yp)[cv] = o;
    }
}

// Stride-1 "same" pooling over a small map (the SPP block: 5/9/13 windows over the 20x20 map): one CTA owns the whole
// plane of one image x 8 channels in shared memory and does the window as two 1-D passes (k + k loads instead of k*k).
constexpr int POOL_PLANE_MAX = 576;   // <= 24 x 24 pixels
__global__ void __launch_bounds__(256) maxpool_plane_kernel(const __half* __restrict__ x, long long xp,
                                                            __half* __restrict__ y, long long yp, int H, int W, int C,
                                                            int k) {
    __shared__ __align__(16) __half sx[POOL_PLANE_MAX * 8];
    __shared__ __align__(16) __half sr[POOL_PLANE_MAX * 8];
    const int CV = C / 8;
    const int n = blockIdx.x / CV, cv = blockIdx.x - n * CV;
    const int HW = H * W, pad = (k - 1) / 2;
    for (int i = threadIdx.x; i < HW; i += blockDim.x)
        reinterpret_cast<uint4*>(sx)[i] = __ldg(reinterpret_cast<const uint4*>(x + ((long long)n * HW + i) * xp) + cv);
    __syncthreads();
    for (int i = threadIdx.x; i < HW * 8; i += blockDim.x) {
        const int c = i & 7, pix = i >> 3;
        const int yi = pix / W, xo = pix - yi * W;
        const int x0 = max(xo - pad, 0), x1 = min(xo - pad + k, W);
        __half m = sx[(yi * W + x0) * 8 + c];
        for (int xi = x0 + 1; xi < x1; ++xi) m = __hmax(m, sx[(yi * W + xi) * 8 + c]);
        sr[i] = m;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < HW * 8; i += blockDim.x) {
        const int c = i & 7, pix = i >> 3;
        const int yo = pix / W, xo = pix - yo * W;
        const int y0 = max(yo - pad, 0), y1 = min(yo - pad + k, H);
        __half m = sr[(y0 * W + xo) * 8 + c];
        for (int yi = y0 + 1; yi < y1; ++yi) m = __hmax(m, sr[(yi * W + xo) * 8 + c]);
        sx[i] = m;      // every thread reads sr only in this pass: sx is free to take the result
    }
    __syncthreads();
    for (int i = threadIdx.x; i < HW; i += blockDim.x)
        reinterpret_cast<uint4*>(y + ((long long)n * HW + i) * yp)[cv] = reinterpret_cast<const uint4*>(sx)[i];
}

extern "C" int b2y_maxpool(const void* x, long long x_pitch, void* y, long long y_pitch, int batch, int in_h, int in_w,
                           int c, int ksize, int stride, int pad_mode, void* stream) {
    if (!x || !y || c % 8 != 0 || x_pitch % 8 != 0 || y_pitch % 8 != 0 || ksize < 1 || stride < 1)
        return B2Y_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15)) return B2Y_ERR_INVALID;
    int pad, Ho, Wo;
    if (pad_mode == 1) {  // ZeroPad2d((0,1,0,1)) + MaxPool2d(k, stride, 0)
        pad = 0;
        Ho = (in_h + 1 - ksize) / stride + 1;
        Wo = (in_w + 1 - ksize) / stride + 1;
    } else {
        pad = (ksize - 1) / 2;
        Ho = (in_h + 2 * pad - ksize) / stride + 1;
        Wo = (in_w + 2 * pad - ksize) / stride + 1;
    }
    const long long total = (long long)batch * Ho * Wo * (c / 8);
    if (pad_mode != 1 && stride == 1 && (ksize & 1) && in_h * in_w <= POOL_PLANE_MAX &&
        (long long)batch * (c / 8) <= 0x7fffffffLL) {
        maxpool_plane_kernel<<<batch * (c / 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
            reinterpret_cast<const __half*>(x), x_pitch, reinterpret_cast<__half*>(y), y_pitch, in_h, in_w, c, ksize);
        B2Y_CUDA_CHECK(cudaGetLastError());
        return B2Y_OK;
    }
    maxpool_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const __half*>(x), x_pitch, reinterpret_cast<__half*>(y), y_pitch, batch, in_h, in_w, c,
        ksize, stride, pad, Ho, Wo, pad_mode == 1 ? 1 : 0);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// ------------------------------------------------------------------------------------------------
// channel copy / add
// ------------------------------------------------------------------------------------------------
__global__ void copy_channels_kernel(const __half* __restrict__ x, long long xp, __half* __restrict__ y, long long yp,
                                     long long pixels, int C) {
    const int CV = C / 8;
    const long long total = pixels * CV;
    const long long stride = (long long)gridDim.x * blockDim.x;
    // four independent 16-byte loads per thread before the first store (one per iteration left the copy latency bound)
    for (long long idx0 = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx0 < total; idx0 += 4 * stride) {
        uint4 v[4];
        uint4* dst[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const long long idx = idx0 + u * stride;
            dst[u] = nullptr;
            if (idx < total) {
                const int cv = (int)(idx % CV);
                const long long pix = idx / CV;
                v[u] = __ldg(reinterpret_cast<const uint4*>(x + pix * xp) + cv);
                dst[u] = reinterpret_cast<uint4*>(y + pix * yp) + cv;
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (dst[u] != nullptr) *dst[u] = v[u];
    }
}

extern "C" int b2y_copy_channels(const void* x, long long x_pitch, void* y, long long y_pitch, long long pixels, int c,
                                 void* stream) {
    if (!x || !y || c % 8 != 0 || x_pitch % 8 != 0 || y_pitch % 8 != 0) return B2Y_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15)) return B2Y_ERR_INVALID;
    copy_channels_kernel<<<grid_for((pixels * (c / 8) + 3) / 4, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const __half*>(x), x_pitch, reinterpret_cast<__half*>(y), y_pitch, pixels, c);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

template <typename T>
__global__ void add_kernel(const T* __restrict__ a, long long ap, const T* __restrict__ b, long long bp,
                           T* __restrict__ y, long long yp, long long pixels, int C) {
    const int CV = C / 8;
    const long long total = pixels * CV;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long idx0 = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx0 < total; idx0 += 2 * stride) {
        uint4 va[2], vb[2];
        T* dst[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const long long idx = idx0 + u * stride;
            dst[u] = nullptr;
            if (idx < total) {
                const int cv = (int)(idx % CV);
                const long long pix = idx / CV;
                va[u] = *reinterpret_cast<const uint4*>(a + pix * ap + cv * 8);
                vb[u] = *reinterpret_cast<const uint4*>(b + pix * bp + cv * 8);
                dst[u] = y + pix * yp + cv * 8;
            }
        }
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            if (dst[u] == nullptr) continue;
            // fp32 add then a single rounding (the reference adds fp32 tensors)
            float fa[8], fb[8];
            Half8<T>::unpack(va[u], fa);
            Half8<T>::unpack(vb[u], fb);
#pragma unroll
            for (int j = 0; j < 8; ++j) fa[j] += fb[j];
            Half8<T>::store(dst[u], fa);
        }
    }
}

extern "C" int b2y_add(const void* a, long long a_pitch, const void* b, long long b_pitch, void* y, long long y_pitch,
                       long long pixels, int c, int dtype, void* stream) {
    if (!a || !b || !y || c % 8 != 0 || a_pitch % 8 != 0 || b_pitch % 8 != 0 || y_pitch % 8 != 0)
        return B2Y_ERR_INVALID;
    if (dtype == B2Y_DT_BF16)
        add_kernel<__nv_bfloat16><<<grid_for((pixels * (c / 8) + 1) / 2, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
            reinterpret_cast<const __nv_bfloat16*>(a), a_pitch, reinterpret_cast<const __nv_bfloat16*>(b), b_pitch,
            reinterpret_cast<__nv_bfloat16*>(y), y_pitch, pixels, c);
    else
        add_kernel<__half><<<grid_for((pixels * (c / 8) + 1) / 2, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
            reinterpret_cast<const __half*>(a), a_pitch, reinterpret_cast<const __half*>(b), b_pitch,
            reinterpret_cast<__half*>(y), y_pitch, pixels, c);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// ------------------------------------------------------------------------------------------------
// standalone activations, fp32 (Mish fwd/bwd: utils/layers.py:117-128, 146-148)
// ------------------------------------------------------------------------------------------------
__global__ void act_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, int act,
                               float slope) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x)
        y[i] = apply_act(x[i], act, slope);
}
__global__ void act_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx,
                               long long n, int act, float slope) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x)
        dx[i] = dy[i] * act_grad(x[i], act, slope);
}
extern "C" int b2y_act_fwd_f32(const float* x, float* y, long long n, int act, float slope, void* stream) {
    if (!x || !y || n < 0) return B2Y_ERR_INVALID;
    act_fwd_kernel<<<grid_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, y, n, act, slope);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}
extern "C" int b2y_act_bwd_f32(const float* x, const float* dy, float* dx, long long n, int act, float slope,
                               void* stream) {
    if (!x || !dy || !dx || n < 0) return B2Y_ERR_INVALID;
    act_bwd_kernel<<<grid_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, dy, dx, n, act, slope);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// ------------------------------------------------------------------------------------------------
// layout converters (32x32 smem-tiled transposes between [C][HW] and [HW][C])
// ------------------------------------------------------------------------------------------------
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, __half* __restrict__ y, long long yp, int C,
                                    int HW) {
    __shared__ float tile[32][33];
    const int n = blockIdx.z;
    const int hw0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const float* xb = x + (long long)n * C * HW;
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        const int c = c0 + j, hw = hw0 + threadIdx.x;
        tile[j][threadIdx.x] = (c < C && hw < HW) ? xb[(long long)c * HW + hw] : 0.f;
    }
    __syncthreads();
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        const int hw = hw0 + j, c = c0 + threadIdx.x;
        if (c < C && hw < HW) y[((long long)n * HW + hw) * yp + c] = __float2half_rn(tile[threadIdx.x][j]);
    }
}
__global__ void nhwc_to_nchw_kernel(const __half* __restrict__ x, long long xp, float* __restrict__ y, int C,
                                    int HW) {
    __shared__ float tile[32][33];
    const int n = blockIdx.z;
    const int hw0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        const int hw = hw0 + j, c = c0 + threadIdx.x;
        tile[j][threadIdx.x] = (c < C && hw < HW) ? __half2float(x[((long long)n * HW + hw) * xp + c]) : 0.f;
    }
    __syncthreads();
    float* yb = y + (long long)n * C * HW;
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        const int c = c0 + j, hw = hw0 + threadIdx.x;
        if (c < C && hw < HW) yb[(long long)c * HW + hw] = tile[threadIdx.x][j];
    }
}
extern "C" int b2y_nchw_f32_to_nhwc_f16(const float* x, void* y, long long y_pitch, int batch, int c, int h, int w,
                                        void* stream) {
    if (!x || !y || batch <= 0 || batch > 65535) return B2Y_ERR_INVALID;
    const int HW = h * w;
    dim3 grid((HW + 31) / 32, (c + 31) / 32, batch), block(32, 8);
    if (grid.y > 65535) return B2Y_ERR_UNSUPPORTED;
    nchw_to_nhwc_kernel<<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(x, reinterpret_cast<__half*>(y),
                                                                                y_pitch, c, HW);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}
extern "C" int b2y_nhwc_f16_to_nchw_f32(const void* x, long long x_pitch, float* y, int batch, int c, int h, int w,
                                        void* stream) {
    if (!x || !y || batch <= 0 || batch > 65535) return B2Y_ERR_INVALID;
    const int HW = h * w;
    dim3 grid((HW + 31) / 32, (c + 31) / 32, batch), block(32, 8);
    if (grid.y > 65535) return B2Y_ERR_UNSUPPORTED;
    nhwc_to_nchw_kernel<<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const __half*>(x),
                                                                                x_pitch, y, c, HW);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}
