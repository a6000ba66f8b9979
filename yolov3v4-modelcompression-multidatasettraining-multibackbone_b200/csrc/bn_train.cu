// Training-mode BatchNorm + activation, bandwidth-oriented versions (three HBM passes per layer and step).
// Reference semantics: nn.BatchNorm2d(momentum=0.1, eps=1e-5) + activation under autograd (models.py:100-113):
// normalise with the biased batch variance, update running_var with the unbiased one.
//
//   forward      y  = act(z*scale + shift) [+ residual]       scale/shift derived from the conv epilogue's channel sums
//                                                             inside this kernel (no separate finalize launch)
//   bwd reduce   S1 = sum du, S2 = sum du*xhat                du = dy * act'(z*scale+shift), xhat = (z-mean)*invstd
//   bwd apply    dz = gamma*invstd*(du - S1/N - xhat*S2/N)    written as fp16 * 2^k (k chosen on the device), and the
//                                                             parameter gradients dgamma = S2, dbeta = S1 emitted
//
// Layout: NHWC, C % 8 == 0.  A thread owns ONE 8-channel vector for the whole kernel (its per-channel coefficients
// live in registers) and walks pixels with a fixed stride; U independent 16-byte loads per operand are issued before
// any arithmetic so that enough bytes are in flight per SM to cover HBM latency (the round-1 kernels issued one load
// per operand per iteration and were latency bound).  Block = CV * (256 / CV) threads (CV = C/8 <= 256), grid = one
// wave of 2 CTAs per SM.
#include "b200yolo.h"
#include "common.cuh"

#include <type_traits>

using namespace b2y;

namespace {

constexpr int ACT_RT = -1;   // activation resolved at run time (relu6 / h_swish / swish / relu)

template <int ACT>
__device__ __forceinline__ float actf(float v, int act_rt, float slope) {
    return apply_act(v, ACT == ACT_RT ? act_rt : ACT, slope);
}
template <int ACT>
__device__ __forceinline__ float actg(float v, int act_rt, float slope) {
    return act_grad(v, ACT == ACT_RT ? act_rt : ACT, slope);
}

// L2 prefetch of the 16-byte vector a thread will load one iteration ahead: the register file caps the loads in flight at
// U per operand (2 CTAs x 256 threads x ~120 registers), prefetches cost no registers and double the bytes in flight.
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

struct Geo {
    int CV, PPB, T;     // channel vectors, pixel rows per block, active threads
};
inline Geo geo_for(int c) {
    Geo g;
    g.CV = c / 8;
    g.PPB = 256 / g.CV;
    g.T = g.CV * g.PPB;
    return g;
}
inline int wave_grid(long long pixels, int ppb, int ctas_per_sm) {
    static int sm_count[64] = {0};
    int dev = 0;
    cudaGetDevice(&dev);
    int& sms = sm_count[dev & 63];
    if (sms <= 0 && cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) sms = 132;
    if (sms <= 0) sms = 132;
    long long g = (pixels + ppb - 1) / ppb;
    const long long cap = (long long)sms * ctas_per_sm;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// ------------------------------------------------------------------------------------------------------------
template <int ACT, int U>
__global__ void __launch_bounds__(256, 2)
bn_train_fwd_kernel(const __half* __restrict__ z, long long zp, const float* __restrict__ s1,
                    const float* __restrict__ s2, const float* __restrict__ gamma, const float* __restrict__ beta,
                    float count, float eps, float momentum, float* __restrict__ rmean, float* __restrict__ rvar,
                    float* __restrict__ save, const __half* __restrict__ res, long long rp, __half* __restrict__ y,
                    long long yp, long long pixels, int CV, int PPB, int act_rt, float slope, int c_logical) {
    pdl_wait();                     // launched as a programmatic dependent (launch_pdl): the statistics / z come from
    pdl_launch_dependents();        // the previous kernel
    const int tid = threadIdx.x;
    if (tid >= CV * PPB) return;
    const int cv = tid % CV, prow = tid / CV;
    const int C = CV * 8;
    float sc[8], sh[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int c = cv * 8 + j;
        if (c >= c_logical) {       // pad channel of a pruned width: y = act(0) (+ a zero residual pad) = 0
            sc[j] = sh[j] = 0.f;
            continue;
        }
        const float mean = __ldg(s1 + c) / count;
        const float var = fmaxf(__ldg(s2 + c) / count - mean * mean, 0.f);      // biased: used for normalisation
        const float invstd = 1.f / sqrtf(var + eps);
        const float g = gamma != nullptr ? __ldg(gamma + c) : 1.f;
        sc[j] = g * invstd;
        sh[j] = (beta != nullptr ? __ldg(beta + c) : 0.f) - mean * sc[j];
        if (blockIdx.x == 0 && prow == 0) {
            save[c] = mean;
            save[C + c] = invstd;
            save[2 * C + c] = sc[j];
            save[3 * C + c] = sh[j];
            if (rmean != nullptr) {
                const float unbiased = count > 1.f ? var * (count / (count - 1.f)) : var;
                rmean[c] = (1.f - momentum) * rmean[c] + momentum * mean;
                rvar[c] = (1.f - momentum) * rvar[c] + momentum * unbiased;
            }
        }
    }
    const long long stride = (long long)gridDim.x * PPB;
    for (long long p0 = (long long)blockIdx.x * PPB + prow; p0 < pixels; p0 += stride * U) {
        uint4 v[U], r[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const long long pix = p0 + u * stride;
            if (pix < pixels) {
                v[u] = __ldg(reinterpret_cast<const uint4*>(z + pix * zp) + cv);
                if (res != nullptr) r[u] = __ldg(reinterpret_cast<const uint4*>(res + pix * rp) + cv);
            }
            const long long nxt = pix + stride * U;
            if (nxt < pixels) {
                prefetch_l2(reinterpret_cast<const uint4*>(z + nxt * zp) + cv);
                if (res != nullptr) prefetch_l2(reinterpret_cast<const uint4*>(res + nxt * rp) + cv);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const long long pix = p0 + u * stride;
            if (pix < pixels) {
                const __half2* h = reinterpret_cast<const __half2*>(&v[u]);
                const __half2* rh = reinterpret_cast<const __half2*>(&r[u]);
                uint4 o;
                __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 f = __half22float2(h[j]);
                    float a = actf<ACT>(fmaf(f.x, sc[2 * j], sh[2 * j]), act_rt, slope);
                    float b = actf<ACT>(fmaf(f.y, sc[2 * j + 1], sh[2 * j + 1]), act_rt, slope);
                    if (res != nullptr) {
                        const float2 rf = __half22float2(rh[j]);
                        a += rf.x;
                        b += rf.y;
                    }
                    oh[j] = __floats2half2_rn(a, b);
                }
                reinterpret_cast<uint4*>(y + pix * yp)[cv] = o;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------------------
template <typename GT, int ACT, int U>
__global__ void __launch_bounds__(256, 2)
bn_train_bwd_reduce_kernel(const __half* __restrict__ z, long long zp, const GT* __restrict__ dy, long long dp,
                           const float* __restrict__ save, double* __restrict__ sums, float* __restrict__ du_absmax,
                           long long pixels, int CV, int PPB, int act_rt, float slope) {
    __shared__ float red[256][17];
    pdl_wait();
    pdl_launch_dependents();
    const int tid = threadIdx.x;
    const int C = CV * 8;
    const bool active = tid < CV * PPB;
    const int cv = active ? tid % CV : 0, prow = tid / CV;
    float sc[8], sh[8], mu[8], a1[8], a2[8], dmax[8];   // dmax: max |z - mean| per channel
    float amax = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int c = cv * 8 + j;
        mu[j] = __ldg(save + c);
        sc[j] = __ldg(save + 2 * C + c);
        sh[j] = __ldg(save + 3 * C + c);
        a1[j] = a2[j] = dmax[j] = 0.f;
    }
    const long long stride = (long long)gridDim.x * PPB;
    if (active) {
        for (long long p0 = (long long)blockIdx.x * PPB + prow; p0 < pixels; p0 += stride * U) {
            uint4 v[U], g[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const long long pix = p0 + u * stride;
                if (pix < pixels) {
                    v[u] = __ldg(reinterpret_cast<const uint4*>(z + pix * zp) + cv);
                    g[u] = __ldg(reinterpret_cast<const uint4*>(dy + pix * dp) + cv);
                }
                const long long nxt = pix + stride * U;
                if (nxt < pixels) {
                    prefetch_l2(reinterpret_cast<const uint4*>(z + nxt * zp) + cv);
                    prefetch_l2(reinterpret_cast<const uint4*>(dy + nxt * dp) + cv);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const long long pix = p0 + u * stride;
                if (pix < pixels) {
                    float xf[8], gf[8];
                    Half8<__half>::unpack(v[u], xf);
                    Half8<GT>::unpack(g[u], gf);
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const float du = gf[j] * actg<ACT>(fmaf(xf[j], sc[j], sh[j]), act_rt, slope);
                        const float d = xf[j] - mu[j];
                        a1[j] += du;
                        a2[j] = fmaf(du, d, a2[j]);
                        amax = fmaxf(amax, fabsf(du));
                        dmax[j] = fmaxf(dmax[j], fabsf(d));
                    }
                }
            }
        }
    }
    if (du_absmax != nullptr) {   // [0] max|du|, [3] max|xhat|: non-negative floats order like their bit patterns
        float xmax = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) xmax = fmaxf(xmax, dmax[j] * __ldg(save + C + cv * 8 + j));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
            xmax = fmaxf(xmax, __shfl_xor_sync(0xffffffffu, xmax, o));
        }
        if ((tid & 31) == 0 && amax > 0.f) atomicMax(reinterpret_cast<unsigned int*>(du_absmax), __float_as_uint(amax));
        if ((tid & 31) == 0 && xmax > 0.f)
            atomicMax(reinterpret_cast<unsigned int*>(du_absmax + 3), __float_as_uint(xmax));
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        red[tid][j] = a1[j];
        red[tid][8 + j] = a2[j];
    }
    __syncthreads();
    // one (channel vector, component) per thread, summed over the PPB pixel rows of the CTA; one atomic per channel
    for (int i = tid; i < CV * 16; i += 256) {
        const int v = i / 16, comp = i % 16;
        float sum = 0.f;
        for (int k = 0; k < PPB; ++k) sum += red[v + k * CV][comp];
        if (comp < 8)
            atomicAdd(sums + v * 8 + comp, (double)sum);
        else   // * invstd -> sum du*xhat
            atomicAdd(sums + C + v * 8 + comp - 8, (double)(sum * __ldg(save + C + v * 8 + comp - 8)));
    }
}

// ------------------------------------------------------------------------------------------------------------
// dz = A*du + Bx*z + Cc   with  A = s*gamma*invstd, Bx = -A*invstd*S2/N, Cc = A*(-S1/N + mean*invstd*S2/N)
// The data gradient dz feeds two tensor-core GEMMs whose operands share one 16-bit format with the fp16 activations /
// weights, so it is written in fp16 times a per-layer power of two s derived on the device from a bound on max|dz|
// (no host sync); the GEMM epilogues multiply by 1/s (scale_out[1]) read from device memory.  du_absmax holds the
// reduce's [max|du|, -, -, max|xhat|] (scale_out is its slots 1 and 2 in the training plan).
template <typename GT, int ACT, int U>
__global__ void __launch_bounds__(256, 2)
bn_train_bwd_apply_kernel(const __half* __restrict__ z, long long zp, const GT* __restrict__ dy, long long dp,
                          const float* __restrict__ gamma, const float* __restrict__ save,
                          const float* __restrict__ sums, __half* __restrict__ dz, long long dzp, long long pixels,
                          int CV, int PPB, int act_rt, float slope, const float* __restrict__ du_absmax,
                          float* __restrict__ scale_out, float* __restrict__ dgamma_out,
                          float* __restrict__ dbeta_out, float grad_out_scale) {
    pdl_wait();
    pdl_launch_dependents();
    const int C = CV * 8;
    const int tid = threadIdx.x;
    const float inv_n = 1.f / (float)pixels;
    __shared__ float s_red[8];
    __shared__ float s_scale;
    {   // every CTA derives the same scale from a bound on max|dz|, since |xhat| <= max|xhat|:
        //   bound = max_c |gamma_c*invstd_c| * (max|du| + |S1_c|/N + max|xhat| * |S2_c|/N)
        // Without the reduce's maxima, max|du| is taken as 1 and max|xhat| as sqrt(N) (sum xhat^2 <= N).
        float bound = 0.f;
        const float dumax = du_absmax != nullptr ? du_absmax[0] : 1.f;
        const float xhmax = du_absmax != nullptr ? du_absmax[3] : sqrtf((float)pixels);
        for (int c = tid; c < C; c += 256) {
            const float g = gamma != nullptr ? gamma[c] : 1.f;
            const float b = fabsf(g * save[C + c]) * (dumax + fabsf(sums[c]) * inv_n + xhmax * fabsf(sums[C + c]) * inv_n);
            bound = fmaxf(bound, b);
            if (blockIdx.x == 0) {
                if (dbeta_out != nullptr) dbeta_out[c] = sums[c] * grad_out_scale;
                if (dgamma_out != nullptr) dgamma_out[c] = sums[C + c] * grad_out_scale;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) bound = fmaxf(bound, __shfl_xor_sync(0xffffffffu, bound, o));
        if ((tid & 31) == 0) s_red[tid >> 5] = bound;
        __syncthreads();
        if (tid == 0) {
            float m = 0.f;
            for (int w = 0; w < 8; ++w) m = fmaxf(m, s_red[w]);
            float sc = 1.f;
            if (m > 0.f && m < 3.0e38f) sc = exp2f(floorf(log2f(4096.f / m)));   // target max |dz|*s <= 2^12
            sc = fminf(fmaxf(sc, 1.0e-30f), 1.0e30f);
            s_scale = sc;
            if (blockIdx.x == 0 && scale_out != nullptr) {
                scale_out[0] = sc;
                scale_out[1] = 1.f / sc;
            }
        }
        __syncthreads();
    }
    if (tid >= CV * PPB) return;
    const float scl = s_scale;
    const int cv = tid % CV, prow = tid / CV;
    float sc[8], sh[8], A[8], Bx[8], Cc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int c = cv * 8 + j;
        const float mean = __ldg(save + c), is = __ldg(save + C + c);
        sc[j] = __ldg(save + 2 * C + c);
        sh[j] = __ldg(save + 3 * C + c);
        const float db = __ldg(sums + c) * inv_n, dg = __ldg(sums + C + c) * inv_n;
        A[j] = scl * (gamma != nullptr ? __ldg(gamma + c) : 1.f) * is;
        Bx[j] = -A[j] * is * dg;
        Cc[j] = A[j] * (mean * is * dg - db);
    }
    const long long stride = (long long)gridDim.x * PPB;
    for (long long p0 = (long long)blockIdx.x * PPB + prow; p0 < pixels; p0 += stride * U) {
        uint4 v[U], g[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const long long pix = p0 + u * stride;
            if (pix < pixels) {
                v[u] = __ldg(reinterpret_cast<const uint4*>(z + pix * zp) + cv);
                g[u] = __ldg(reinterpret_cast<const uint4*>(dy + pix * dp) + cv);
            }
            const long long nxt = pix + stride * U;
            if (nxt < pixels) {
                prefetch_l2(reinterpret_cast<const uint4*>(z + nxt * zp) + cv);
                prefetch_l2(reinterpret_cast<const uint4*>(dy + nxt * dp) + cv);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const long long pix = p0 + u * stride;
            if (pix < pixels) {
                float xf[8], gf[8], r[8];
                Half8<__half>::unpack(v[u], xf);
                Half8<GT>::unpack(g[u], gf);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float du = gf[j] * actg<ACT>(fmaf(xf[j], sc[j], sh[j]), act_rt, slope);
                    r[j] = fmaf(A[j], du, fmaf(Bx[j], xf[j], Cc[j]));
                }
                Half8<__half>::store(dz + pix * dzp + cv * 8, r);
            }
        }
    }
}

template <typename F>
inline void dispatch_act(int act, F&& f) {
    // compile-time activation for the three that dominate Darknet (yolov3: leaky, yolov4: mish, heads/mobilenet: linear)
    if (act == B2Y_ACT_LEAKY) f(std::integral_constant<int, B2Y_ACT_LEAKY>{});
    else if (act == B2Y_ACT_MISH) f(std::integral_constant<int, B2Y_ACT_MISH>{});
    else if (act == B2Y_ACT_LINEAR) f(std::integral_constant<int, B2Y_ACT_LINEAR>{});
    else f(std::integral_constant<int, ACT_RT>{});
}

inline bool shape_ok(int c, long long p0, long long p1, long long p2 = 8) {
    return c > 0 && c % 8 == 0 && c / 8 <= 256 && p0 % 8 == 0 && p1 % 8 == 0 && p2 % 8 == 0;
}

// ------------------------------------------------------------------------------------------------------------
// fp32 NHWC BatchNorm + activation of the google-QAT graph's float depthwise blocks (b200yolo/qat.py), any C, dense.
// save [4][C] = mean, invstd, scale, shift: the batch statistics in training, the running ones in eval.  Sums over pixels
// go through chunk_reduce (common.cuh, fixed order, double).
struct BnF32StatOp {
    const float* z;
    int C;
    __device__ void operator()(int, long long p, int c, float (&v)[2]) const {
        const float t = __ldg(z + p * C + c);
        v[0] = t;
        v[1] = t * t;
    }
};
__global__ void __launch_bounds__(256) bn_f32_stat_kernel(BnF32StatOp op, long long rows, double* part) {
    chunk_reduce<2>(op, rows, op.C, part);
}

// training: batch mean / biased variance for the normalisation, running statistics updated with the unbiased variance
// (nn.BatchNorm2d); eval: the running statistics
__global__ void bn_f32_finalize_kernel(const double* __restrict__ part, long long count, const float* __restrict__ gamma,
                                       const float* __restrict__ beta, float eps, float momentum,
                                       float* __restrict__ rmean, float* __restrict__ rvar, float* __restrict__ save,
                                       int C, int training) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    float mean, var;
    if (training) {
        double s1 = 0.0, s2 = 0.0;
        for (int ch = 0; ch < F32_CHUNKS; ++ch) {
            s1 += part[((long long)ch * 2) * C + c];
            s2 += part[((long long)ch * 2 + 1) * C + c];
        }
        const double m = s1 / (double)count;
        const double vb = fmax(s2 / (double)count - m * m, 0.0);
        mean = (float)m;
        var = (float)vb;
        const float unbiased = count > 1 ? (float)(vb * ((double)count / (double)(count - 1))) : var;
        rmean[c] = (1.f - momentum) * rmean[c] + momentum * mean;
        rvar[c] = (1.f - momentum) * rvar[c] + momentum * unbiased;
    } else {
        mean = rmean[c];
        var = rvar[c];
    }
    const float invstd = 1.f / sqrtf(var + eps);
    const float sc = gamma[c] * invstd;
    save[c] = mean;
    save[C + c] = invstd;
    save[2 * C + c] = sc;
    save[3 * C + c] = beta[c] - mean * sc;
}

__global__ void __launch_bounds__(256)
bn_f32_apply_kernel(const float* __restrict__ z, const float* __restrict__ save, float* __restrict__ y, int C,
                    long long total, int act, float slope) {
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(idx % C);
        y[idx] = apply_act(fmaf(__ldg(z + idx), __ldg(save + 2 * C + c), __ldg(save + 3 * C + c)), act, slope);
    }
}

// backward sums: S1 = sum du, S2 = sum du * (z - mean), du = dy * act'(z * scale + shift)
struct BnF32BwdOp {
    const float* z;
    const float* dy;
    const float* save;
    int C, act;
    float slope;
    __device__ void operator()(int, long long p, int c, float (&v)[2]) const {
        const float t = __ldg(z + p * C + c);
        const float du = __ldg(dy + p * C + c) * act_grad(fmaf(t, __ldg(save + 2 * C + c), __ldg(save + 3 * C + c)), act, slope);
        v[0] = du;
        v[1] = du * (t - __ldg(save + c));
    }
};
__global__ void __launch_bounds__(256) bn_f32_bwd_stat_kernel(BnF32BwdOp op, long long rows, double* part) {
    chunk_reduce<2>(op, rows, op.C, part);
}

// sums [2][C] in fp32 (dbeta, dgamma) and the double coefficients of dz = A du + Bx z + Cc per channel
__global__ void bn_f32_bwd_finalize_kernel(const double* __restrict__ part, long long count,
                                           const float* __restrict__ gamma, const float* __restrict__ save,
                                           float* __restrict__ coef, float* __restrict__ dgamma,
                                           float* __restrict__ dbeta, int C, int training) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double s1 = 0.0, s2 = 0.0;
    for (int ch = 0; ch < F32_CHUNKS; ++ch) {
        s1 += part[((long long)ch * 2) * C + c];
        s2 += part[((long long)ch * 2 + 1) * C + c];
    }
    const double is = save[C + c], mean = save[c];
    dbeta[c] = (float)s1;
    dgamma[c] = (float)(s2 * is);
    const double A = (double)gamma[c] * is;
    if (training) {   // dz = A (du - S1/N - xhat * (S2 * invstd) / N),  xhat = (z - mean) invstd
        const double db = s1 / (double)count, dg = s2 * is * is / (double)count;
        coef[c] = (float)A;
        coef[C + c] = (float)(-A * dg);
        coef[2 * C + c] = (float)(A * (mean * dg - db));
    } else {          // running statistics are constants: dz = A du
        coef[c] = (float)A;
        coef[C + c] = 0.f;
        coef[2 * C + c] = 0.f;
    }
}

__global__ void __launch_bounds__(256)
bn_f32_bwd_apply_kernel(const float* __restrict__ z, const float* __restrict__ dy, const float* __restrict__ save,
                        const float* __restrict__ coef, float* __restrict__ dz, int C, long long total, int act,
                        float slope) {
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(idx % C);
        const float t = __ldg(z + idx);
        const float du = __ldg(dy + idx) * act_grad(fmaf(t, __ldg(save + 2 * C + c), __ldg(save + 3 * C + c)), act, slope);
        dz[idx] = fmaf(__ldg(coef + c), du, fmaf(__ldg(coef + C + c), t, __ldg(coef + 2 * C + c)));
    }
}

}  // namespace

extern "C" int b2y_bn_train_fwd_lw(const void* z, long long z_pitch, const float* stat_sum, const float* stat_sqsum,
                                   long long count, const float* gamma, const float* beta, float eps, float momentum,
                                   float* running_mean, float* running_var, float* save, const void* residual,
                                   long long res_pitch, void* y, long long y_pitch, long long pixels, int c,
                                   int c_logical, int act, float slope, void* stream) {
    if (!z || !y || !stat_sum || !stat_sqsum || !save || count <= 0 || pixels <= 0) return B2Y_ERR_INVALID;
    if (!shape_ok(c, z_pitch, y_pitch, residual ? res_pitch : 8)) return B2Y_ERR_UNSUPPORTED;
    if (c_logical < 1 || c_logical > c || c - c_logical >= 8) return B2Y_ERR_INVALID;
    const Geo g = geo_for(c);
    const int grid = wave_grid(pixels, g.PPB, 2);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    dispatch_act(act, [&](auto A) {
        launch_pdl(bn_train_fwd_kernel<decltype(A)::value, 4>, dim3(grid), dim3(256), 0, st, 
            reinterpret_cast<const __half*>(z), z_pitch, stat_sum, stat_sqsum, gamma, beta, (float)count, eps, momentum,
            running_mean, running_var, save, reinterpret_cast<const __half*>(residual), res_pitch,
            reinterpret_cast<__half*>(y), y_pitch, pixels, g.CV, g.PPB, act, slope, c_logical);
    });
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_bn_train_fwd(const void* z, long long z_pitch, const float* stat_sum, const float* stat_sqsum,
                                long long count, const float* gamma, const float* beta, float eps, float momentum,
                                float* running_mean, float* running_var, float* save, const void* residual,
                                long long res_pitch, void* y, long long y_pitch, long long pixels, int c, int act,
                                float slope, void* stream) {
    return b2y_bn_train_fwd_lw(z, z_pitch, stat_sum, stat_sqsum, count, gamma, beta, eps, momentum, running_mean,
                               running_var, save, residual, res_pitch, y, y_pitch, pixels, c, c, act, slope, stream);
}

extern "C" int b2y_bn_train_bwd_reduce(const void* z, long long z_pitch, const void* dy, long long dy_pitch,
                                       const float* save, float* sums, float* du_absmax, long long pixels, int c,
                                       int act, float slope, int grad_dtype, void* stream) {
    if (!z || !dy || !save || !sums || pixels <= 0) return B2Y_ERR_INVALID;
    if (!shape_ok(c, z_pitch, dy_pitch)) return B2Y_ERR_UNSUPPORTED;
    const Geo g = geo_for(c);
    const int grid = wave_grid(pixels, g.PPB, 2);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    double* acc = stream_acc(st, 2LL * c);     // [0, C) sum du, [C, 2C) sum du*xhat
    if (acc == nullptr) return B2Y_ERR_CUDA;
    dispatch_act(act, [&](auto A) {
        constexpr int ACT = decltype(A)::value;
        if (grad_dtype == B2Y_DT_BF16)
            launch_pdl(bn_train_bwd_reduce_kernel<__nv_bfloat16, ACT, 4>, dim3(grid), dim3(256), 0, st, 
                reinterpret_cast<const __half*>(z), z_pitch, reinterpret_cast<const __nv_bfloat16*>(dy), dy_pitch, save,
                acc, du_absmax, pixels, g.CV, g.PPB, act, slope);
        else
            launch_pdl(bn_train_bwd_reduce_kernel<__half, ACT, 4>, dim3(grid), dim3(256), 0, st, 
                reinterpret_cast<const __half*>(z), z_pitch, reinterpret_cast<const __half*>(dy), dy_pitch, save, acc,
                du_absmax, pixels, g.CV, g.PPB, act, slope);
    });
    B2Y_CUDA_CHECK(cudaGetLastError());
    return acc_finalize(acc, sums, 2LL * c, st);
}

extern "C" int b2y_bn_train_bwd_apply(const void* z, long long z_pitch, const void* dy, long long dy_pitch,
                                      const float* gamma, const float* save, const float* sums, void* dz,
                                      long long dz_pitch, long long pixels, int c, int act, float slope,
                                      int grad_dtype, const float* du_absmax, float* scale_out, float* dgamma_out,
                                      float* dbeta_out, float grad_out_scale, void* stream) {
    if (!z || !dy || !save || !sums || !dz || pixels <= 0) return B2Y_ERR_INVALID;
    if (!shape_ok(c, z_pitch, dy_pitch, dz_pitch)) return B2Y_ERR_UNSUPPORTED;
    const Geo g = geo_for(c);
    const int grid = wave_grid(pixels, g.PPB, 2);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    dispatch_act(act, [&](auto A) {
        constexpr int ACT = decltype(A)::value;
        if (grad_dtype == B2Y_DT_BF16)
            launch_pdl(bn_train_bwd_apply_kernel<__nv_bfloat16, ACT, 4>, dim3(grid), dim3(256), 0, st, 
                reinterpret_cast<const __half*>(z), z_pitch, reinterpret_cast<const __nv_bfloat16*>(dy), dy_pitch, gamma,
                save, sums, reinterpret_cast<__half*>(dz), dz_pitch, pixels, g.CV, g.PPB, act, slope, du_absmax,
                scale_out, dgamma_out, dbeta_out, grad_out_scale);
        else
            launch_pdl(bn_train_bwd_apply_kernel<__half, ACT, 4>, dim3(grid), dim3(256), 0, st, 
                reinterpret_cast<const __half*>(z), z_pitch, reinterpret_cast<const __half*>(dy), dy_pitch, gamma, save,
                sums, reinterpret_cast<__half*>(dz), dz_pitch, pixels, g.CV, g.PPB, act, slope, du_absmax, scale_out,
                dgamma_out, dbeta_out, grad_out_scale);
    });
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_bn_f32_fwd(const float* z, long long pixels, int c, const float* gamma, const float* beta, float eps,
                              float momentum, float* running_mean, float* running_var, int training, float* save,
                              float* y, int act, float slope, void* stream) {
    if (!z || !gamma || !beta || !running_mean || !running_var || !save || !y || pixels <= 0 || c <= 0)
        return B2Y_ERR_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    double* part = nullptr;
    if (training) {
        part = chunk_ws(st, 1, 2, c);
        if (part == nullptr) return B2Y_ERR_CUDA;
        bn_f32_stat_kernel<<<chunk_grid(c, 1), dim3(32, 8), 0, st>>>(BnF32StatOp{z, c}, pixels, part);
    }
    bn_f32_finalize_kernel<<<(c + 127) / 128, 128, 0, st>>>(part, pixels, gamma, beta, eps, momentum, running_mean,
                                                             running_var, save, c, training);
    bn_f32_apply_kernel<<<grid_1d(pixels * c), 256, 0, st>>>(z, save, y, c, pixels * c, act, slope);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_bn_f32_bwd(const float* z, const float* dy, long long pixels, int c, const float* gamma,
                              const float* save, int training, float* coef /* [3][c] */, float* dz, float* dgamma,
                              float* dbeta, int act, float slope, void* stream) {
    if (!z || !dy || !gamma || !save || !coef || !dz || !dgamma || !dbeta || pixels <= 0 || c <= 0)
        return B2Y_ERR_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    double* part = chunk_ws(st, 1, 2, c);
    if (part == nullptr) return B2Y_ERR_CUDA;
    bn_f32_bwd_stat_kernel<<<chunk_grid(c, 1), dim3(32, 8), 0, st>>>(BnF32BwdOp{z, dy, save, c, act, slope}, pixels,
                                                                      part);
    bn_f32_bwd_finalize_kernel<<<(c + 127) / 128, 128, 0, st>>>(part, pixels, gamma, save, coef, dgamma, dbeta, c,
                                                                 training);
    bn_f32_bwd_apply_kernel<<<grid_1d(pixels * c), 256, 0, st>>>(z, dy, save, coef, dz, c, pixels * c, act, slope);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}
