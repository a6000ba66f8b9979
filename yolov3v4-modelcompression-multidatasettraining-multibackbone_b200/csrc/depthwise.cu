// Depthwise convolution (groups == channels) and squeeze-excite, forward and backward, NHWC fp16 (C % 8 == 0).
// Reference: the `depthwise` cfg block models.py:115-197 (nn.Conv2d(groups=Cin) + BatchNorm2d + activation, k = 3 / 5,
// stride 1 / 2) and SE utils/layers.py:176-192 (avgpool -> Linear(C, C/4) -> ReLU -> Linear(C/4, C) -> HardSigmoid ->
// x * y).  0.7 % of yolov3-mobilenet's MACs but a third of its layers: these kernels are HBM / launch bound, so they run
// on the CUDA cores with 16-byte vector accesses; a thread owns one 8-channel vector (its per-channel state lives in
// registers) and walks pixels, like the BatchNorm passes in bn_train.cu.
#include "b200yolo.h"
#include "common.cuh"

using namespace b2y;

namespace {

struct Geo {
    int CV, PPB;
};
inline Geo geo_for(int c) {
    Geo g;
    g.CV = c / 8;
    g.PPB = 256 / g.CV;
    if (g.PPB < 1) g.PPB = 1;
    return g;
}
inline int sm_count() {
    static int sms[64] = {0};
    int dev = 0;
    cudaGetDevice(&dev);
    int& s = sms[dev & 63];
    if (s <= 0 && cudaDeviceGetAttribute(&s, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) s = 132;
    if (s <= 0) s = 132;
    return s;
}
inline int grid_for_rows(long long rows, int ppb, int per_sm) {
    long long g = (rows + ppb - 1) / ppb;
    const long long cap = (long long)sm_count() * per_sm;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// block-level reduction of per-thread 8-vectors over the PPB pixel rows of a CTA, then one atomic per channel into the
// fp64 stream accumulator (common.cuh stream_acc; the host adds it into the fp32 destination with acc_finalize)
__device__ __forceinline__ void block_reduce_atomic(float (&a)[8], float* red /*[256][9]*/, double* dst, int CV,
                                                    int PPB, float mul) {
    const int tid = threadIdx.x;
#pragma unroll
    for (int j = 0; j < 8; ++j) red[tid * 9 + j] = a[j];
    __syncthreads();
    for (int i = tid; i < CV * 8; i += blockDim.x) {
        const int v = i / 8, comp = i % 8;
        float s = 0.f;
        for (int k = 0; k < PPB; ++k) s += red[(v + k * CV) * 9 + comp];
        atomicAdd(dst + v * 8 + comp, (double)(s * mul));
    }
    __syncthreads();
}

// ------------------------------------------------------------------------------------------------------------
// forward: y = act(dwconv(x, w) * scale + bias); optional channel sums of the raw output (training BatchNorm) into the
// fp64 accumulator stat_acc: [0, C) sums, [C, 2C) squares.
// weights arrive as fp32 [C][k][k] (the nn.Conv2d(groups=C) parameter) and are staged as fp16 [tap][C] in smem.
__global__ void __launch_bounds__(256)
dwconv_fwd_kernel(const __half* __restrict__ x, long long xp, const float* __restrict__ w,
                  const float* __restrict__ scale, const float* __restrict__ bias, __half* __restrict__ y,
                  long long yp, double* __restrict__ stat_acc, int B, int H, int W, int C, int k,
                  int stride, int pad, int Ho, int Wo, int act, float slope, int CV, int PPB) {
    extern __shared__ uint8_t smem_dw[];
    __half* ws = reinterpret_cast<__half*>(smem_dw);                                  // [k*k][C]
    float* red = reinterpret_cast<float*>(smem_dw + (((size_t)k * k * C * 2 + 15) & ~(size_t)15));   // [256][9]
    const int k2 = k * k;
    for (int i = threadIdx.x; i < C * k2; i += blockDim.x) {
        const int c = i / k2, t = i - c * k2;
        ws[t * C + c] = __float2half_rn(__ldg(w + i));      // fp16 weights: the engine's precision policy
    }
    __syncthreads();
    const int tid = threadIdx.x;
    const bool active = tid < CV * PPB;
    const int cv = active ? tid % CV : 0, prow = tid / CV;
    float sc[8], bi[8], a1[8], a2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        sc[j] = scale != nullptr ? __ldg(scale + cv * 8 + j) : 1.f;
        bi[j] = bias != nullptr ? __ldg(bias + cv * 8 + j) : 0.f;
        a1[j] = a2[j] = 0.f;
    }
    const long long pixels = (long long)B * Ho * Wo;
    const long long stride_p = (long long)gridDim.x * PPB;
    if (active) {
        for (long long pix = (long long)blockIdx.x * PPB + prow; pix < pixels; pix += stride_p) {
            const int xo = (int)(pix % Wo);
            const int yo = (int)((pix / Wo) % Ho);
            const int n = (int)(pix / ((long long)Wo * Ho));
            float acc[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = 0.f;
            for (int r = 0; r < k; ++r) {
                const int yi = yo * stride - pad + r;
                if (yi < 0 || yi >= H) continue;
                for (int s = 0; s < k; ++s) {
                    const int xi = xo * stride - pad + s;
                    if (xi < 0 || xi >= W) continue;
                    const uint4 xv = __ldg(reinterpret_cast<const uint4*>(x + (((long long)n * H + yi) * W + xi) * xp) + cv);
                    const uint4 wv = *reinterpret_cast<const uint4*>(ws + (r * k + s) * C + cv * 8);
                    const __half2* xh = reinterpret_cast<const __half2*>(&xv);
                    const __half2* wh = reinterpret_cast<const __half2*>(&wv);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float2 xf = __half22float2(xh[j]), wf = __half22float2(wh[j]);
                        acc[2 * j] = fmaf(xf.x, wf.x, acc[2 * j]);
                        acc[2 * j + 1] = fmaf(xf.y, wf.y, acc[2 * j + 1]);
                    }
                }
            }
            float o[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                // the statistics are taken on the fp16-rounded value that is stored (what the BatchNorm pass will read)
                const float raw = fmaf(acc[j], sc[j], bi[j]);
                o[j] = apply_act(raw, act, slope);
            }
            Half8<__half>::store(y + pix * yp + cv * 8, o);
            if (stat_acc != nullptr) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float q = __half2float(__float2half_rn(o[j]));
                    a1[j] += q;
                    a2[j] = fmaf(q, q, a2[j]);
                }
            }
        }
    }
    if (stat_acc != nullptr) {
        block_reduce_atomic(a1, red, stat_acc, CV, PPB, 1.f);
        block_reduce_atomic(a2, red, stat_acc + C, CV, PPB, 1.f);
    }
}

// data gradient: dx[n,yi,xi,c] (+)= inv_s * sum_{r,s} w[c][r][s] * dz[n,(yi+pad-r)/st,(xi+pad-s)/st,c]
template <typename GT>
__global__ void __launch_bounds__(256)
dwconv_bwd_data_kernel(const __half* __restrict__ dz, long long dzp, const float* __restrict__ w, GT* __restrict__ dx,
                       long long dxp, int B, int H, int W, int C, int k, int stride, int pad, int Ho, int Wo,
                       int accumulate, const float* __restrict__ inv_scale_ptr, int CV, int PPB) {
    extern __shared__ uint8_t smem_dw[];
    __half* ws = reinterpret_cast<__half*>(smem_dw);
    const int k2 = k * k;
    for (int i = threadIdx.x; i < C * k2; i += blockDim.x) {
        const int c = i / k2, t = i - c * k2;
        ws[t * C + c] = __float2half_rn(__ldg(w + i));
    }
    __syncthreads();
    const int tid = threadIdx.x;
    if (tid >= CV * PPB) return;
    const float inv_s = inv_scale_ptr != nullptr ? __ldg(inv_scale_ptr) : 1.f;
    const int cv = tid % CV, prow = tid / CV;
    const long long pixels = (long long)B * H * W;
    const long long stride_p = (long long)gridDim.x * PPB;
    for (long long pix = (long long)blockIdx.x * PPB + prow; pix < pixels; pix += stride_p) {
        const int xi = (int)(pix % W);
        const int yi = (int)((pix / W) % H);
        const int n = (int)(pix / ((long long)W * H));
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        for (int r = 0; r < k; ++r) {
            const int ty = yi + pad - r;
            if (ty < 0 || ty % stride != 0) continue;
            const int yo = ty / stride;
            if (yo >= Ho) continue;
            for (int s = 0; s < k; ++s) {
                const int tx = xi + pad - s;
                if (tx < 0 || tx % stride != 0) continue;
                const int xo = tx / stride;
                if (xo >= Wo) continue;
                const uint4 gv = __ldg(reinterpret_cast<const uint4*>(dz + (((long long)n * Ho + yo) * Wo + xo) * dzp) + cv);
                const uint4 wv = *reinterpret_cast<const uint4*>(ws + (r * k + s) * C + cv * 8);
                const __half2* gh = reinterpret_cast<const __half2*>(&gv);
                const __half2* wh = reinterpret_cast<const __half2*>(&wv);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 gf = __half22float2(gh[j]), wf = __half22float2(wh[j]);
                    acc[2 * j] = fmaf(gf.x, wf.x, acc[2 * j]);
                    acc[2 * j + 1] = fmaf(gf.y, wf.y, acc[2 * j + 1]);
                }
            }
        }
        GT* dp = dx + pix * dxp + cv * 8;
        float o[8];
        if (accumulate) {
            Half8<GT>::load(dp, o);
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] = fmaf(acc[j], inv_s, o[j]);
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] = acc[j] * inv_s;
        }
        Half8<GT>::store(dp, o);
    }
}

// weight gradient: dw_acc[c][r][s] += alpha * inv_s * sum_pixels dz[pix][c] * x[pix @ (r,s)][c];  grid.y = tap.  dw_acc
// is the fp64 stream accumulator, added into dw by acc_finalize
__global__ void __launch_bounds__(256)
dwconv_bwd_weight_kernel(const __half* __restrict__ x, long long xp, const __half* __restrict__ dz, long long dzp,
                         double* __restrict__ dw_acc, int B, int H, int W, int C, int k, int stride, int pad, int Ho,
                         int Wo, float alpha, const float* __restrict__ inv_scale_ptr, int CV, int PPB) {
    __shared__ float red[256 * 9];
    const int tap = blockIdx.y;
    const int r = tap / k, s = tap % k;
    const int tid = threadIdx.x;
    const bool active = tid < CV * PPB;
    const int cv = active ? tid % CV : 0, prow = tid / CV;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    const long long pixels = (long long)B * Ho * Wo;
    const long long stride_p = (long long)gridDim.x * PPB;
    if (active) {
        for (long long pix = (long long)blockIdx.x * PPB + prow; pix < pixels; pix += stride_p) {
            const int xo = (int)(pix % Wo);
            const int yo = (int)((pix / Wo) % Ho);
            const int n = (int)(pix / ((long long)Wo * Ho));
            const int yi = yo * stride - pad + r, xi = xo * stride - pad + s;
            if (yi < 0 || yi >= H || xi < 0 || xi >= W) continue;
            float gf[8], xf[8];
            Half8<__half>::load(dz + pix * dzp + cv * 8, gf);
            Half8<__half>::load(x + (((long long)n * H + yi) * W + xi) * xp + cv * 8, xf);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = fmaf(gf[j], xf[j], acc[j]);
        }
    }
    const float mul = alpha * (inv_scale_ptr != nullptr ? __ldg(inv_scale_ptr) : 1.f);
#pragma unroll
    for (int j = 0; j < 8; ++j) red[tid * 9 + j] = acc[j];
    __syncthreads();
    const int k2 = k * k;
    for (int i = tid; i < CV * 8; i += blockDim.x) {
        const int v = i / 8, comp = i % 8;
        float sum = 0.f;
        for (int q = 0; q < PPB; ++q) sum += red[(v + q * CV) * 9 + comp];
        atomicAdd(dw_acc + (long long)(v * 8 + comp) * k2 + tap, (double)(sum * mul));
    }
}

// ------------------------------------------------------------------------------------------------------------
// squeeze-excite
// pooled[n][c] += sum over the image's pixels of x, into the fp64 accumulator (the mean is taken in the fc kernel)
__global__ void __launch_bounds__(256)
se_pool_kernel(const __half* __restrict__ x, long long xp, double* __restrict__ pooled, int HW, int C, int CV, int PPB) {
    __shared__ float red[256 * 9];
    const int n = blockIdx.y;
    const int tid = threadIdx.x;
    const bool active = tid < CV * PPB;
    const int cv = active ? tid % CV : 0, prow = tid / CV;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    if (active) {
        for (int p = blockIdx.x * PPB + prow; p < HW; p += gridDim.x * PPB) {
            float xf[8];
            Half8<__half>::load(x + ((long long)n * HW + p) * xp + cv * 8, xf);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] += xf[j];
        }
    }
    block_reduce_atomic(acc, red, pooled + (long long)n * C, CV, PPB, 1.f);
}

// one block per image: mean -> h = relu(W1 mean) -> s = hsigmoid(W2 h).  W1 [Cr][C], W2 [C][Cr] fp32 (nn.Linear)
__global__ void se_fc_kernel(const float* __restrict__ pooled_sum, const float* __restrict__ w1,
                             const float* __restrict__ w2, float* __restrict__ mean_out, float* __restrict__ h_out,
                             float* __restrict__ v_out, float* __restrict__ s_out, int C, int Cr, float inv_hw) {
    extern __shared__ float sh[];       // [C] mean, [Cr] h
    float* m = sh;
    float* h = sh + C;
    const int n = blockIdx.x;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        m[c] = pooled_sum[(long long)n * C + c] * inv_hw;
        if (mean_out != nullptr) mean_out[(long long)n * C + c] = m[c];
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    for (int j = warp; j < Cr; j += nw) {
        float a = 0.f;
        for (int c = lane; c < C; c += 32) a = fmaf(__ldg(w1 + (long long)j * C + c), m[c], a);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (lane == 0) {
            h[j] = fmaxf(a, 0.f);
            if (h_out != nullptr) h_out[(long long)n * Cr + j] = h[j];
        }
    }
    __syncthreads();
    for (int c = warp; c < C; c += nw) {
        float a = 0.f;
        for (int j = lane; j < Cr; j += 32) a = fmaf(__ldg(w2 + (long long)c * Cr + j), h[j], a);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (lane == 0) {
            if (v_out != nullptr) v_out[(long long)n * C + c] = a;
            s_out[(long long)n * C + c] = fminf(fmaxf(a + 3.f, 0.f), 6.f) / 6.f;     // HardSigmoid utils/layers.py:167-173
        }
    }
}

// y = x * s[n][c]
__global__ void __launch_bounds__(256)
se_scale_kernel(const __half* __restrict__ x, long long xp, const float* __restrict__ s, __half* __restrict__ y,
                long long yp, int HW, int C, long long total_vec) {
    const int CV = C / 8;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total_vec;
         idx += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(idx % CV);
        const long long pix = idx / CV;
        const int n = (int)(pix / HW);
        float xf[8];
        Half8<__half>::load(x + pix * xp + cv * 8, xf);
        const float4 sa = __ldg(reinterpret_cast<const float4*>(s + (long long)n * C + cv * 8));
        const float4 sb = __ldg(reinterpret_cast<const float4*>(s + (long long)n * C + cv * 8) + 1);
        const float sv[8] = {sa.x, sa.y, sa.z, sa.w, sb.x, sb.y, sb.z, sb.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) xf[j] *= sv[j];
        Half8<__half>::store(y + pix * yp + cv * 8, xf);
    }
}

// backward, pass 1: ds_raw[n][c] += sum_pixels dy * x, into the fp64 accumulator
template <typename GT>
__global__ void __launch_bounds__(256)
se_bwd_reduce_kernel(const __half* __restrict__ x, long long xp, const GT* __restrict__ dy, long long dyp,
                     double* __restrict__ ds, int HW, int C, int CV, int PPB) {
    __shared__ float red[256 * 9];
    const int n = blockIdx.y;
    const int tid = threadIdx.x;
    const bool active = tid < CV * PPB;
    const int cv = active ? tid % CV : 0, prow = tid / CV;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    if (active) {
        for (int p = blockIdx.x * PPB + prow; p < HW; p += gridDim.x * PPB) {
            float xf[8], gf[8];
            Half8<__half>::load(x + ((long long)n * HW + p) * xp + cv * 8, xf);
            Half8<GT>::load(dy + ((long long)n * HW + p) * dyp + cv * 8, gf);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = fmaf(xf[j], gf[j], acc[j]);
        }
    }
    block_reduce_atomic(acc, red, ds + (long long)n * C, CV, PPB, 1.f);
}

// backward of the two Linear layers, one block per image: dv = ds * hsig'(v); dh = (W2^T dv) * [h > 0];
// dmean = W1^T dh.  Outputs dv [N][C], dh [N][Cr], dmean [N][C] (the weight gradients are outer-product sums over
// the images, se_fc_wgrad_kernel).
__global__ void se_fc_bwd_kernel(const float* __restrict__ ds, const float* __restrict__ v, const float* __restrict__ h,
                                 const float* __restrict__ w1, const float* __restrict__ w2, float* __restrict__ dv_out,
                                 float* __restrict__ dh_out, float* __restrict__ dmean_out, int C, int Cr) {
    extern __shared__ float sh[];       // [C] dv, [Cr] dh
    float* dv = sh;
    float* dh = sh + C;
    const int n = blockIdx.x;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        const float vv = v[(long long)n * C + c];
        const float g = (vv > -3.f && vv < 3.f) ? (1.f / 6.f) : 0.f;
        dv[c] = ds[(long long)n * C + c] * g;
        dv_out[(long long)n * C + c] = dv[c];
    }
    __syncthreads();
    for (int j = threadIdx.x; j < Cr; j += blockDim.x) {
        float a = 0.f;
        for (int c = 0; c < C; ++c) a = fmaf(__ldg(w2 + (long long)c * Cr + j), dv[c], a);
        dh[j] = h[(long long)n * Cr + j] > 0.f ? a : 0.f;
        dh_out[(long long)n * Cr + j] = dh[j];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float a = 0.f;
        for (int j = 0; j < Cr; ++j) a = fmaf(__ldg(w1 + (long long)j * C + c), dh[j], a);
        dmean_out[(long long)n * C + c] = a;
    }
}

// dW[i][j] = alpha * sum_n a[n][i] * b[n][j]   (dW2 = dv (x) h, dW1 = dh (x) mean)
__global__ void se_fc_wgrad_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ dw,
                                   int N, int I, int J, float alpha) {
    const long long total = (long long)I * J;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(idx / J), j = (int)(idx % J);
        float s = 0.f;
        for (int n = 0; n < N; ++n) s = fmaf(a[(long long)n * I + i], b[(long long)n * J + j], s);
        dw[idx] = s * alpha;
    }
}

// backward, pass 2: dx (+)= dy * s[n][c] + dmean[n][c] / HW
template <typename GT>
__global__ void __launch_bounds__(256)
se_bwd_apply_kernel(const GT* __restrict__ dy, long long dyp, const float* __restrict__ s,
                    const float* __restrict__ dmean, GT* __restrict__ dx, long long dxp, int HW, int C, float inv_hw,
                    int accumulate, long long total_vec) {
    const int CV = C / 8;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total_vec;
         idx += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(idx % CV);
        const long long pix = idx / CV;
        const int n = (int)(pix / HW);
        float gf[8], o[8];
        Half8<GT>::load(dy + pix * dyp + cv * 8, gf);
        if (accumulate) Half8<GT>::load(dx + pix * dxp + cv * 8, o);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = cv * 8 + j;
            const float t = fmaf(gf[j], __ldg(s + (long long)n * C + c), __ldg(dmean + (long long)n * C + c) * inv_hw);
            o[j] = accumulate ? o[j] + t : t;
        }
        Half8<GT>::store(dx + pix * dxp + cv * 8, o);
    }
}

inline bool vec_ok(int c, long long p0, long long p1) { return c > 0 && c % 8 == 0 && c / 8 <= 256 && p0 % 8 == 0 && p1 % 8 == 0; }
inline size_t dw_smem(int c, int k) { return (((size_t)k * k * c * 2 + 15) & ~(size_t)15) + 256 * 9 * sizeof(float); }

template <typename K>
inline int set_smem(K kern, size_t bytes, unsigned long long& mask) {
    if (bytes > 48 * 1024 && b2y_first_use_on_device(mask))
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(200 * 1024)) != cudaSuccess)
            return -1;
    return 0;
}

// ------------------------------------------------------------------------------------------------------------
// fp32 NHWC versions for the google-QAT graph (b200yolo/qat.py), whose depthwise blocks and SE layers stay in float
// (reference models.py:115-197 under quantized=1), and for the quantised depthwise layers of the TPSQ graph.  Dense
// tensors (pitch = C), any C: MobileNet's widths 24, 40, 72, 120, 184 and 200 are not multiples of 16.  One thread per (pixel, channel), consecutive threads on consecutive channels;
// every reduction over pixels goes through chunk_reduce (common.cuh), so two runs give the same bits.

// z[n,yo,xo,c] = bias[c] + sum_{r,s} x[n, yo*st-pad+r, xo*st-pad+s, c] * w[c][r][s]
__global__ void __launch_bounds__(256)
dwconv_f32_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                      float* __restrict__ z, int H, int W, int C, int k, int stride, int pad, int Ho, int Wo,
                      long long total) {
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(idx % C);
        const long long pix = idx / C;
        const int xo = (int)(pix % Wo), yo = (int)((pix / Wo) % Ho);
        const long long n = pix / ((long long)Wo * Ho);
        const float* wc = w + (long long)c * k * k;
        float acc = 0.f;
        for (int r = 0; r < k; ++r) {
            const int yi = yo * stride - pad + r;
            if (yi < 0 || yi >= H) continue;
            for (int s = 0; s < k; ++s) {
                const int xi = xo * stride - pad + s;
                if (xi < 0 || xi >= W) continue;
                acc = fmaf(__ldg(x + ((n * H + yi) * W + xi) * C + c), __ldg(wc + r * k + s), acc);
            }
        }
        z[idx] = bias != nullptr ? acc + __ldg(bias + c) : acc;
    }
}

// dx[n,yi,xi,c] = sum_{r,s} w[c][r][s] * dz[n, (yi+pad-r)/st, (xi+pad-s)/st, c]  (+ w2 * dz2 at the same taps when dz2
// is given: the two convolutions of a TPSQ depthwise layer read the same input, so their data gradients share a gather)
__global__ void __launch_bounds__(256)
dwconv_f32_bwd_data_kernel(const float* __restrict__ dz, const float* __restrict__ w, const float* __restrict__ dz2,
                           const float* __restrict__ w2, float* __restrict__ dx, int H, int W, int C, int k, int stride,
                           int pad, int Ho, int Wo, long long total) {
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(idx % C);
        const long long pix = idx / C;
        const int xi = (int)(pix % W), yi = (int)((pix / W) % H);
        const long long n = pix / ((long long)W * H);
        const float* wc = w + (long long)c * k * k;
        const float* wc2 = dz2 != nullptr ? w2 + (long long)c * k * k : nullptr;
        float acc = 0.f;
        for (int r = 0; r < k; ++r) {
            const int ty = yi + pad - r;
            if (ty < 0 || ty % stride != 0 || ty / stride >= Ho) continue;
            for (int s = 0; s < k; ++s) {
                const int tx = xi + pad - s;
                if (tx < 0 || tx % stride != 0 || tx / stride >= Wo) continue;
                const long long o = ((n * Ho + ty / stride) * Wo + tx / stride) * C + c;
                acc = fmaf(__ldg(dz + o), __ldg(wc + r * k + s), acc);
                if (wc2 != nullptr) acc = fmaf(__ldg(dz2 + o), __ldg(wc2 + r * k + s), acc);
            }
        }
        dx[idx] = acc;
    }
}

// Batch statistics of z = dwconv(x, w) + bias, z recomputed here (never stored): the taps accumulate in double (the
// fp32 x fp32 products are exact there) and z and z^2 go to chunk_reduce as doubles, so a channel whose |mean| is many
// times its standard deviation keeps its variance.
struct DwStatOp {
    const float* x;
    const float* w;
    const float* bias;
    int H, W, C, k, stride, pad, Ho, Wo;
    __device__ void operator()(int, long long pix, int c, double (&v)[2]) const {
        const int xo = (int)(pix % Wo), yo = (int)((pix / Wo) % Ho);
        const long long n = pix / ((long long)Wo * Ho);
        const float* wc = w + (long long)c * k * k;
        double z = bias != nullptr ? (double)__ldg(bias + c) : 0.0;
        for (int r = 0; r < k; ++r) {
            const int yi = yo * stride - pad + r;
            if (yi < 0 || yi >= H) continue;
            for (int s = 0; s < k; ++s) {
                const int xi = xo * stride - pad + s;
                if (xi < 0 || xi >= W) continue;
                z = fma((double)__ldg(x + ((n * H + yi) * W + xi) * C + c), (double)__ldg(wc + r * k + s), z);
            }
        }
        v[0] = z;
        v[1] = z * z;
    }
};
__global__ void __launch_bounds__(256) dwconv_f32_stats_kernel(DwStatOp op, long long rows, double* part) {
    chunk_reduce<2, DwStatOp, double>(op, rows, op.C, part);
}
// part [chunk][2][C] -> mean, unbiased variance (torch.var), formed in double
__global__ void dwconv_f32_stats_finish_kernel(const double* __restrict__ part, long long count, float* __restrict__ mean,
                                               float* __restrict__ var, int C) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double s1 = 0.0, s2 = 0.0;
    for (int ch = 0; ch < F32_CHUNKS; ++ch) {
        s1 += part[((long long)ch * 2) * C + c];
        s2 += part[((long long)ch * 2 + 1) * C + c];
    }
    const double m = s1 / (double)count;
    mean[c] = (float)m;
    var[c] = count > 1 ? (float)(fmax(s2 - s1 * m, 0.0) / (double)(count - 1)) : 0.f;
}

// gradient into z = dwconv(x, w) + bias through its batch statistics:
// gs = g_mean / n + 2 g_var (z - mean) / (n - 1), z recomputed (k^2 MACs per output, as in the forward)
__global__ void __launch_bounds__(256)
dwconv_f32_stats_grad_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                             const float* __restrict__ mean, const float* __restrict__ g_mean,
                             const float* __restrict__ g_var, float* __restrict__ gs, int H, int W, int C, int k,
                             int stride, int pad, int Ho, int Wo, long long total) {
    const double n = (double)(total / C);
    const float inv_n = (float)(1.0 / n), two_inv_n1 = n > 1.0 ? (float)(2.0 / (n - 1.0)) : 0.f;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(idx % C);
        const long long pix = idx / C;
        float g = g_mean != nullptr ? __ldg(g_mean + c) * inv_n : 0.f;
        if (g_var != nullptr) {
            const int xo = (int)(pix % Wo), yo = (int)((pix / Wo) % Ho);
            const long long nn = pix / ((long long)Wo * Ho);
            const float* wc = w + (long long)c * k * k;
            float z = 0.f;
            for (int r = 0; r < k; ++r) {
                const int yi = yo * stride - pad + r;
                if (yi < 0 || yi >= H) continue;
                for (int s = 0; s < k; ++s) {
                    const int xi = xo * stride - pad + s;
                    if (xi < 0 || xi >= W) continue;
                    z = fmaf(__ldg(x + ((nn * H + yi) * W + xi) * C + c), __ldg(wc + r * k + s), z);
                }
            }
            // z - mean as (conv - (mean - bias)): the bias cancels before any rounding of the large terms
            const float centred = z - (__ldg(mean + c) - (bias != nullptr ? __ldg(bias + c) : 0.f));
            g = fmaf(__ldg(g_var + c) * two_inv_n1, centred, g);
        }
        gs[idx] = g;
    }
}

// weight gradient, group = tap (r, s): rows are output pixels, value dz * x at the tap's input pixel
struct DwWgradOp {
    const float* x;
    const float* dz;
    int H, W, C, k, stride, pad, Ho, Wo;
    __device__ void operator()(int tap, long long pix, int c, float (&v)[1]) const {
        const int xo = (int)(pix % Wo), yo = (int)((pix / Wo) % Ho);
        const long long n = pix / ((long long)Wo * Ho);
        const int yi = yo * stride - pad + tap / k, xi = xo * stride - pad + tap % k;
        v[0] = (yi < 0 || yi >= H || xi < 0 || xi >= W) ? 0.f
                                                         : __ldg(dz + pix * C + c) * __ldg(x + ((n * H + yi) * W + xi) * C + c);
    }
};
__global__ void __launch_bounds__(256) dwconv_f32_wgrad_reduce_kernel(DwWgradOp op, long long rows, double* part) {
    chunk_reduce<1>(op, rows, op.C, part);
}
// part [tap][chunk][C] -> dw [C][k*k]
__global__ void dwconv_f32_wgrad_finish_kernel(const double* __restrict__ part, float* __restrict__ dw, int C, int k2) {
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < C * k2; idx += gridDim.x * blockDim.x) {
        const int c = idx / k2, tap = idx % k2;
        double s = 0.0;
        for (int ch = 0; ch < F32_CHUNKS; ++ch) s += part[((long long)tap * F32_CHUNKS + ch) * C + c];
        dw[idx] = (float)s;
    }
}

// squeeze-excite, group = image: pool sums x, the backward sums dy * x
struct SePoolOp {
    const float* x;
    const float* dy;
    int C;
    long long HW;
    __device__ void operator()(int n, long long p, int c, float (&v)[1]) const {
        const long long i = ((long long)n * HW + p) * C + c;
        v[0] = dy != nullptr ? __ldg(x + i) * __ldg(dy + i) : __ldg(x + i);
    }
};
__global__ void __launch_bounds__(256) se_f32_reduce_kernel(SePoolOp op, double* part) {
    chunk_reduce<1>(op, op.HW, op.C, part);
}

// forward y = x * s[n][c];  backward dx = dy * s[n][c] + dmean[n][c] / HW
__global__ void __launch_bounds__(256)
se_f32_apply_kernel(const float* __restrict__ x, const float* __restrict__ s, const float* __restrict__ dmean,
                    float* __restrict__ y, long long HW, int C, float inv_hw, long long total) {
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(idx % C);
        const long long nc = idx / C / HW * C + c;
        const float t = __ldg(x + idx) * __ldg(s + nc);
        y[idx] = dmean != nullptr ? fmaf(__ldg(dmean + nc), inv_hw, t) : t;
    }
}

inline bool dw_f32_ok(const b2y_conv_desc* d) {
    return d->in_c == d->out_c && d->in_c > 0 && d->in_pitch == d->in_c && d->out_pitch == d->out_c && d->ksize >= 1 &&
           d->ksize <= 7 && d->stride >= 1 && d->batch > 0;
}

}  // namespace

extern "C" int b2y_dwconv_fwd(const b2y_conv_desc* d, const void* x, const float* w, const float* scale,
                              const float* bias, void* y, float* stat_sum, float* stat_sqsum, void* stream) {
    if (!d || !x || !w || !y) return B2Y_ERR_INVALID;
    if ((stat_sum == nullptr) != (stat_sqsum == nullptr)) return B2Y_ERR_INVALID;
    if (d->in_c != d->out_c || !vec_ok(d->in_c, d->in_pitch, d->out_pitch) || d->ksize < 1 || d->ksize > 7)
        return B2Y_ERR_UNSUPPORTED;
    const Geo g = geo_for(d->in_c);
    const long long pixels = (long long)d->batch * d->out_h * d->out_w;
    const size_t smem = dw_smem(d->in_c, d->ksize);
    if (smem > 200 * 1024) return B2Y_ERR_UNSUPPORTED;
    static unsigned long long mask = 0;
    if (set_smem(dwconv_fwd_kernel, smem, mask) != 0) return B2Y_ERR_CUDA;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int c = d->in_c;
    double* acc = nullptr;
    if (stat_sum != nullptr && (acc = stream_acc(st, 2LL * c)) == nullptr) return B2Y_ERR_CUDA;
    dwconv_fwd_kernel<<<grid_for_rows(pixels, g.PPB, 4), 256, smem, st>>>(
        reinterpret_cast<const __half*>(x), d->in_pitch, w, scale, bias, reinterpret_cast<__half*>(y), d->out_pitch,
        acc, d->batch, d->in_h, d->in_w, c, d->ksize, d->stride, d->pad, d->out_h, d->out_w, d->act, d->slope, g.CV,
        g.PPB);
    B2Y_CUDA_CHECK(cudaGetLastError());
    if (acc == nullptr) return B2Y_OK;
    const int rc = acc_finalize(acc, stat_sum, c, st);
    if (rc != B2Y_OK) return rc;
    return acc_finalize(acc + c, stat_sqsum, c, st);
}

extern "C" int b2y_dwconv_bwd_data(const b2y_conv_desc* d, const void* dz, const float* w, void* dx, int accumulate,
                                   int out_dtype, const float* inv_scale_ptr, void* stream) {
    if (!d || !dz || !w || !dx) return B2Y_ERR_INVALID;
    if (d->in_c != d->out_c || !vec_ok(d->in_c, d->in_pitch, d->out_pitch) || d->ksize < 1 || d->ksize > 7)
        return B2Y_ERR_UNSUPPORTED;
    const Geo g = geo_for(d->in_c);
    const long long pixels = (long long)d->batch * d->in_h * d->in_w;
    const size_t smem = dw_smem(d->in_c, d->ksize);
    if (smem > 200 * 1024) return B2Y_ERR_UNSUPPORTED;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int grid = grid_for_rows(pixels, g.PPB, 4);
    static unsigned long long m16 = 0, mbf = 0;
    if (out_dtype == B2Y_DT_BF16) {
        if (set_smem(dwconv_bwd_data_kernel<__nv_bfloat16>, smem, mbf) != 0) return B2Y_ERR_CUDA;
        dwconv_bwd_data_kernel<__nv_bfloat16><<<grid, 256, smem, st>>>(
            reinterpret_cast<const __half*>(dz), d->out_pitch, w, reinterpret_cast<__nv_bfloat16*>(dx), d->in_pitch,
            d->batch, d->in_h, d->in_w, d->in_c, d->ksize, d->stride, d->pad, d->out_h, d->out_w, accumulate,
            inv_scale_ptr, g.CV, g.PPB);
    } else {
        if (set_smem(dwconv_bwd_data_kernel<__half>, smem, m16) != 0) return B2Y_ERR_CUDA;
        dwconv_bwd_data_kernel<__half><<<grid, 256, smem, st>>>(
            reinterpret_cast<const __half*>(dz), d->out_pitch, w, reinterpret_cast<__half*>(dx), d->in_pitch, d->batch,
            d->in_h, d->in_w, d->in_c, d->ksize, d->stride, d->pad, d->out_h, d->out_w, accumulate, inv_scale_ptr,
            g.CV, g.PPB);
    }
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_dwconv_bwd_weight(const b2y_conv_desc* d, const void* x, const void* dz, float* dw, float alpha,
                                     const float* inv_scale_ptr, void* stream) {
    if (!d || !x || !dz || !dw) return B2Y_ERR_INVALID;
    if (d->in_c != d->out_c || !vec_ok(d->in_c, d->in_pitch, d->out_pitch) || d->ksize < 1 || d->ksize > 7)
        return B2Y_ERR_UNSUPPORTED;
    const Geo g = geo_for(d->in_c);
    const long long pixels = (long long)d->batch * d->out_h * d->out_w;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long n = (long long)d->in_c * d->ksize * d->ksize;
    double* acc = stream_acc(st, n);
    if (acc == nullptr) return B2Y_ERR_CUDA;
    dim3 grid(grid_for_rows(pixels, g.PPB, 1), d->ksize * d->ksize);
    dwconv_bwd_weight_kernel<<<grid, 256, 0, st>>>(
        reinterpret_cast<const __half*>(x), d->in_pitch, reinterpret_cast<const __half*>(dz), d->out_pitch, acc,
        d->batch, d->in_h, d->in_w, d->in_c, d->ksize, d->stride, d->pad, d->out_h, d->out_w, alpha, inv_scale_ptr,
        g.CV, g.PPB);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return acc_finalize(acc, dw, n, st);
}

extern "C" int b2y_se_fwd(const void* x, long long x_pitch, const float* w1, const float* w2, void* y,
                          long long y_pitch, int batch, int hw, int c, int cr, float* ws /* fp32 [batch][3c+cr] */,
                          void* stream) {
    if (!x || !w1 || !w2 || !y || !ws || batch <= 0 || hw <= 0 || cr <= 0) return B2Y_ERR_INVALID;
    if (!vec_ok(c, x_pitch, y_pitch)) return B2Y_ERR_UNSUPPORTED;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // workspace layout: pooled sum / mean [N][C] | v [N][C] | s [N][C] | h [N][Cr].  h goes last: se_scale_kernel
    // reads s with float4 loads, and N * Cr is not a multiple of 4 for every batch (e.g. N = 3, Cr = 18)
    float* pooled = ws;
    float* v = pooled + (long long)batch * c;
    float* s = v + (long long)batch * c;
    float* h = s + (long long)batch * c;
    B2Y_CUDA_CHECK(cudaMemsetAsync(pooled, 0, sizeof(float) * (size_t)batch * c, st));
    double* acc = stream_acc(st, (long long)batch * c);
    if (acc == nullptr) return B2Y_ERR_CUDA;
    const Geo g = geo_for(c);
    int gx = (hw + g.PPB - 1) / g.PPB;
    const int cap = (sm_count() * 4 + batch - 1) / batch;
    if (gx > cap) gx = cap;
    if (gx < 1) gx = 1;
    se_pool_kernel<<<dim3(gx, batch), 256, 0, st>>>(reinterpret_cast<const __half*>(x), x_pitch, acc, hw, c, g.CV,
                                                    g.PPB);
    B2Y_CUDA_CHECK(cudaGetLastError());
    const int rc = acc_finalize(acc, pooled, (long long)batch * c, st);
    if (rc != B2Y_OK) return rc;
    se_fc_kernel<<<batch, 256, sizeof(float) * (c + cr), st>>>(pooled, w1, w2, pooled, h, v, s, c, cr, 1.f / (float)hw);
    const long long total = (long long)batch * hw * (c / 8);
    long long gs = (total + 255) / 256;
    if (gs > (long long)sm_count() * 8) gs = (long long)sm_count() * 8;
    se_scale_kernel<<<(int)gs, 256, 0, st>>>(reinterpret_cast<const __half*>(x), x_pitch, s, reinterpret_cast<__half*>(y),
                                             y_pitch, hw, c, total);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_se_bwd(const void* x, long long x_pitch, const void* dy, long long dy_pitch, const float* w1,
                          const float* w2, const float* ws /* from b2y_se_fwd */, float* ws_bwd /* fp32 [batch][3c+cr] */,
                          void* dx, long long dx_pitch, int accumulate, float* dw1, float* dw2, float grad_scale,
                          int batch, int hw, int c, int cr, int grad_dtype, void* stream) {
    if (!x || !dy || !w1 || !w2 || !ws || !ws_bwd || !dx || !dw1 || !dw2) return B2Y_ERR_INVALID;
    if (!vec_ok(c, x_pitch, dy_pitch) || dx_pitch % 8 != 0) return B2Y_ERR_UNSUPPORTED;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float* mean = ws;                               // layout of b2y_se_fwd
    const float* v = mean + (long long)batch * c;
    const float* s = v + (long long)batch * c;
    const float* h = s + (long long)batch * c;
    float* ds = ws_bwd;                                   // [N][C]  sum dy*x, then reused as dv
    float* dh = ds + (long long)batch * c;                // [N][Cr]
    float* dmean = dh + (long long)batch * cr;            // [N][C]
    float* dv = dmean + (long long)batch * c;             // [N][C]
    B2Y_CUDA_CHECK(cudaMemsetAsync(ds, 0, sizeof(float) * (size_t)batch * c, st));
    double* acc = stream_acc(st, (long long)batch * c);
    if (acc == nullptr) return B2Y_ERR_CUDA;
    const Geo g = geo_for(c);
    int gx = (hw + g.PPB - 1) / g.PPB;
    const int cap = (sm_count() * 4 + batch - 1) / batch;
    if (gx > cap) gx = cap;
    if (gx < 1) gx = 1;
    const long long total = (long long)batch * hw * (c / 8);
    long long gs = (total + 255) / 256;
    if (gs > (long long)sm_count() * 8) gs = (long long)sm_count() * 8;
    if (grad_dtype == B2Y_DT_BF16)
        se_bwd_reduce_kernel<__nv_bfloat16><<<dim3(gx, batch), 256, 0, st>>>(
            reinterpret_cast<const __half*>(x), x_pitch, reinterpret_cast<const __nv_bfloat16*>(dy), dy_pitch, acc, hw, c,
            g.CV, g.PPB);
    else
        se_bwd_reduce_kernel<__half><<<dim3(gx, batch), 256, 0, st>>>(
            reinterpret_cast<const __half*>(x), x_pitch, reinterpret_cast<const __half*>(dy), dy_pitch, acc, hw, c, g.CV,
            g.PPB);
    B2Y_CUDA_CHECK(cudaGetLastError());
    const int rc = acc_finalize(acc, ds, (long long)batch * c, st);
    if (rc != B2Y_OK) return rc;
    se_fc_bwd_kernel<<<batch, 256, sizeof(float) * (c + cr), st>>>(ds, v, h, w1, w2, dv, dh, dmean, c, cr);
    {
        const long long t2 = (long long)c * cr;
        int gw = (int)((t2 + 255) / 256);
        se_fc_wgrad_kernel<<<gw, 256, 0, st>>>(dv, h, dw2, batch, c, cr, grad_scale);        // dW2 [C][Cr]
        se_fc_wgrad_kernel<<<gw, 256, 0, st>>>(dh, mean, dw1, batch, cr, c, grad_scale);     // dW1 [Cr][C]
    }
    if (grad_dtype == B2Y_DT_BF16)
        se_bwd_apply_kernel<__nv_bfloat16><<<(int)gs, 256, 0, st>>>(
            reinterpret_cast<const __nv_bfloat16*>(dy), dy_pitch, s, dmean, reinterpret_cast<__nv_bfloat16*>(dx), dx_pitch,
            hw, c, 1.f / (float)hw, accumulate, total);
    else
        se_bwd_apply_kernel<__half><<<(int)gs, 256, 0, st>>>(
            reinterpret_cast<const __half*>(dy), dy_pitch, s, dmean, reinterpret_cast<__half*>(dx), dx_pitch, hw, c,
            1.f / (float)hw, accumulate, total);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_dwconv_fwd_f32(const b2y_conv_desc* d, const float* x, const float* w, const float* bias, float* z,
                                  void* stream) {
    if (!d || !x || !w || !z) return B2Y_ERR_INVALID;
    if (!dw_f32_ok(d)) return B2Y_ERR_UNSUPPORTED;
    const long long total = (long long)d->batch * d->out_h * d->out_w * d->out_c;
    dwconv_f32_fwd_kernel<<<grid_1d(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        x, w, bias, z, d->in_h, d->in_w, d->in_c, d->ksize, d->stride, d->pad, d->out_h, d->out_w, total);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_dwconv_bwd_f32(const b2y_conv_desc* d, const float* x, const float* dz, const float* w, float* dx,
                                  float* dw, void* stream) {
    if (!d || !dz || !w || (!dx && !dw) || (dw && !x)) return B2Y_ERR_INVALID;
    if (!dw_f32_ok(d)) return B2Y_ERR_UNSUPPORTED;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (dx != nullptr) {
        const long long total = (long long)d->batch * d->in_h * d->in_w * d->in_c;
        dwconv_f32_bwd_data_kernel<<<grid_1d(total), 256, 0, st>>>(dz, w, nullptr, nullptr, dx, d->in_h, d->in_w,
                                                                  d->in_c, d->ksize, d->stride, d->pad, d->out_h,
                                                                  d->out_w, total);
    }
    if (dw != nullptr) {
        const int k2 = d->ksize * d->ksize;
        double* part = chunk_ws(st, k2, 1, d->in_c);
        if (part == nullptr) return B2Y_ERR_CUDA;
        const DwWgradOp op{x, dz, d->in_h, d->in_w, d->in_c, d->ksize, d->stride, d->pad, d->out_h, d->out_w};
        dwconv_f32_wgrad_reduce_kernel<<<chunk_grid(d->in_c, k2), dim3(32, 8), 0, st>>>(
            op, (long long)d->batch * d->out_h * d->out_w, part);
        dwconv_f32_wgrad_finish_kernel<<<grid_1d((long long)d->in_c * k2), 256, 0, st>>>(part, dw, d->in_c, k2);
    }
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_dwconv_stats_f32(const b2y_conv_desc* d, const float* x, const float* w, const float* bias,
                                    float* mean, float* var, void* stream) {
    if (!d || !x || !w || !mean || !var) return B2Y_ERR_INVALID;
    if (!dw_f32_ok(d)) return B2Y_ERR_UNSUPPORTED;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int c = d->in_c;
    double* part = chunk_ws(st, 1, 2, c);
    if (part == nullptr) return B2Y_ERR_CUDA;
    const long long rows = (long long)d->batch * d->out_h * d->out_w;
    const DwStatOp op{x, w, bias, d->in_h, d->in_w, c, d->ksize, d->stride, d->pad, d->out_h, d->out_w};
    dwconv_f32_stats_kernel<<<chunk_grid(c, 1), dim3(32, 8), 0, st>>>(op, rows, part);
    dwconv_f32_stats_finish_kernel<<<(c + 127) / 128, 128, 0, st>>>(part, rows, mean, var, c);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_dwconv_stats_bwd_f32(const b2y_conv_desc* d, const float* x, const float* w, const float* bias,
                                        const float* mean, const float* g_mean, const float* g_var, const float* dz2,
                                        const float* w2, float* gs, float* dx, float* dw, void* stream) {
    if (!d || !x || !w || !mean || !gs || (!dx && !dw) || (dz2 && !w2)) return B2Y_ERR_INVALID;
    if (!dw_f32_ok(d)) return B2Y_ERR_UNSUPPORTED;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int c = d->in_c;
    const long long total = (long long)d->batch * d->out_h * d->out_w * c;
    dwconv_f32_stats_grad_kernel<<<grid_1d(total), 256, 0, st>>>(x, w, bias, mean, g_mean, g_var, gs, d->in_h, d->in_w,
                                                                 c, d->ksize, d->stride, d->pad, d->out_h, d->out_w,
                                                                 total);
    if (dx != nullptr) {
        const long long tin = (long long)d->batch * d->in_h * d->in_w * c;
        dwconv_f32_bwd_data_kernel<<<grid_1d(tin), 256, 0, st>>>(gs, w, dz2, w2, dx, d->in_h, d->in_w, c, d->ksize,
                                                                d->stride, d->pad, d->out_h, d->out_w, tin);
    }
    if (dw != nullptr) {
        const int k2 = d->ksize * d->ksize;
        double* part = chunk_ws(st, k2, 1, c);
        if (part == nullptr) return B2Y_ERR_CUDA;
        const DwWgradOp op{x, gs, d->in_h, d->in_w, c, d->ksize, d->stride, d->pad, d->out_h, d->out_w};
        dwconv_f32_wgrad_reduce_kernel<<<chunk_grid(c, k2), dim3(32, 8), 0, st>>>(
            op, (long long)d->batch * d->out_h * d->out_w, part);
        dwconv_f32_wgrad_finish_kernel<<<grid_1d((long long)c * k2), 256, 0, st>>>(part, dw, c, k2);
    }
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_se_fwd_f32(const float* x, const float* w1, const float* w2, float* y, int batch, int hw, int c,
                              int cr, float* ws /* fp32 [batch][3c+cr] */, void* stream) {
    if (!x || !w1 || !w2 || !y || !ws || batch <= 0 || hw <= 0 || c <= 0 || cr <= 0) return B2Y_ERR_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float* pooled = ws;                  // layout of b2y_se_fwd: mean [N][C] | v [N][C] | s [N][C] | h [N][Cr]
    float* v = pooled + (long long)batch * c;
    float* s = v + (long long)batch * c;
    float* h = s + (long long)batch * c;
    double* part = chunk_ws(st, batch, 1, c);
    if (part == nullptr) return B2Y_ERR_CUDA;
    se_f32_reduce_kernel<<<chunk_grid(c, batch), dim3(32, 8), 0, st>>>(SePoolOp{x, nullptr, c, hw}, part);
    chunk_sum_kernel<0><<<grid_1d((long long)batch * c), 256, 0, st>>>(part, pooled, c, batch, 1.f);
    se_fc_kernel<<<batch, 256, sizeof(float) * (c + cr), st>>>(pooled, w1, w2, pooled, h, v, s, c, cr, 1.f / (float)hw);
    const long long total = (long long)batch * hw * c;
    se_f32_apply_kernel<<<grid_1d(total), 256, 0, st>>>(x, s, nullptr, y, hw, c, 0.f, total);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_se_bwd_f32(const float* x, const float* dy, const float* w1, const float* w2,
                              const float* ws /* from b2y_se_fwd_f32 */, float* ws_bwd /* fp32 [batch][3c+cr] */,
                              float* dx, float* dw1, float* dw2, int batch, int hw, int c, int cr, void* stream) {
    if (!x || !dy || !w1 || !w2 || !ws || !ws_bwd || !dx || !dw1 || !dw2 || batch <= 0 || hw <= 0 || c <= 0 || cr <= 0)
        return B2Y_ERR_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float* mean = ws;
    const float* v = mean + (long long)batch * c;
    const float* s = v + (long long)batch * c;
    const float* h = s + (long long)batch * c;
    float* ds = ws_bwd;                                   // [N][C]  sum dy*x
    float* dh = ds + (long long)batch * c;                // [N][Cr]
    float* dmean = dh + (long long)batch * cr;            // [N][C]
    float* dv = dmean + (long long)batch * c;             // [N][C]
    double* part = chunk_ws(st, batch, 1, c);
    if (part == nullptr) return B2Y_ERR_CUDA;
    se_f32_reduce_kernel<<<chunk_grid(c, batch), dim3(32, 8), 0, st>>>(SePoolOp{x, dy, c, hw}, part);
    chunk_sum_kernel<0><<<grid_1d((long long)batch * c), 256, 0, st>>>(part, ds, c, batch, 1.f);
    se_fc_bwd_kernel<<<batch, 256, sizeof(float) * (c + cr), st>>>(ds, v, h, w1, w2, dv, dh, dmean, c, cr);
    const int gw = grid_1d((long long)c * cr);
    se_fc_wgrad_kernel<<<gw, 256, 0, st>>>(dv, h, dw2, batch, c, cr, 1.f);        // dW2 [C][Cr]
    se_fc_wgrad_kernel<<<gw, 256, 0, st>>>(dh, mean, dw1, batch, cr, c, 1.f);     // dW1 [Cr][C]
    const long long total = (long long)batch * hw * c;
    se_f32_apply_kernel<<<grid_1d(total), 256, 0, st>>>(dy, s, dmean, dx, hw, c, 1.f / (float)hw, total);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}
