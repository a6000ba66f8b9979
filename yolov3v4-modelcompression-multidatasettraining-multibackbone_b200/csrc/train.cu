// Training-mode backward helpers on NHWC fp16 tensors (the per-channel (BatchNorm/bias) + activation gradient reduce,
// the YOLO-head, upsample and max-pool gradients), the fused SGD-Nesterov step over a flat fp32 parameter buffer and the
// per-parameter-group SGD / Adam steps over the same buffers.
// Reference semantics: activation under autograd (models.py:100-113), optimizer train.py:135-144.  The BatchNorm
// training passes of the conv layers are in bn_train.cu.
#include "b200yolo.h"
#include "common.cuh"

using namespace b2y;

static inline int grid_for(long long n, int block, int cap = 132 * 16) {
    long long g = (n + block - 1) / block;
    if (g < 1) g = 1;
    if (g > cap) g = cap;
    return (int)g;
}

// v2 layout: a thread owns ONE 8-channel vector (its per-channel coefficients live in registers for the whole kernel)
// and walks the pixels with a fixed stride; the activation is resolved at compile time.  Needs 256 % (C/8) == 0.
static inline int v2_grid(long long pixels, int CV) {
    const int ppb = 256 / CV;
    long long g = (pixels + ppb - 1) / ppb;
    const long long cap = 132 * 8;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}
static inline bool v2_ok(int c) { return c % 8 == 0 && c / 8 <= 256 && 256 % (c / 8) == 0; }

// ------------------------------------------------------------------------------------------------
// backward pass 1: dbeta[c] = sum du, dgamma[c] = sum du * xhat   with  u = x*scale+shift, du = dy*act'(u)
// grid.y tiles the channels in slabs of 256 (32 lanes x 8 channels); each warp walks a strip of pixels.
// ------------------------------------------------------------------------------------------------
template <typename GT>
__global__ void __launch_bounds__(256)
bn_act_bwd_reduce_kernel(const __half* __restrict__ x, long long xp, const GT* __restrict__ dy, long long dp,
                         const float* __restrict__ scale, const float* __restrict__ shift,
                         const float* __restrict__ mean, const float* __restrict__ invstd,
                         double* __restrict__ dgamma, double* __restrict__ dbeta, float* __restrict__ du_absmax,
                         long long pixels, int C, int act, float slope) {
    __shared__ float red[8][32][17];
    float amax = 0.f;
    const int CV = C / 8;
    const int cv0 = blockIdx.y * 32;
    const int cvn = min(32, CV - cv0);                 // channel vectors in this slab
    // lanes -> (pixel sub-index, channel vector); pack several pixels per warp when the slab is narrow
    int lanes_c = 1;
    while (lanes_c < cvn) lanes_c <<= 1;               // next pow2 >= cvn (<= 32)
    const int ppw = 32 / lanes_c;                      // pixels per warp iteration
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int lc = lane % lanes_c, lp = lane / lanes_c;
    const bool active = lc < cvn;
    const int cv = cv0 + lc;
    float sc[8], sh[8], mu[8], is[8], gb[8], gg[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        gb[j] = gg[j] = 0.f;
        const int c = cv * 8 + j;
        sc[j] = active ? scale[c] : 0.f;
        sh[j] = active ? shift[c] : 0.f;
        mu[j] = (active && mean) ? mean[c] : 0.f;
        is[j] = (active && invstd) ? invstd[c] : 1.f;
    }
    const long long warps_total = (long long)gridDim.x * 8;
    const long long wid = (long long)blockIdx.x * 8 + warp;
    for (long long p0 = wid * ppw; p0 < pixels; p0 += warps_total * ppw) {
        const long long pix = p0 + lp;
        if (active && pix < pixels) {
            float xf8[8], g8[8];
            Half8<__half>::load(x + pix * xp + cv * 8, xf8);
            Half8<GT>::load(dy + pix * dp + cv * 8, g8);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float xf = xf8[j];
                const float u = fmaf(xf, sc[j], sh[j]);
                const float du = g8[j] * act_grad(u, act, slope);
                gb[j] += du;
                gg[j] += du * ((xf - mu[j]) * is[j]);
                amax = fmaxf(amax, fabsf(du));
            }
        }
    }
    if (du_absmax != nullptr) {   // max |du| over the tensor (non-negative floats order like their bit patterns)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        if (lane == 0 && amax > 0.f) atomicMax(reinterpret_cast<unsigned int*>(du_absmax), __float_as_uint(amax));
    }
    // combine the pixel sub-lanes of a warp, then the 8 warps of the CTA, then one atomic per channel
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        for (int o = lanes_c; o < 32; o <<= 1) {
            gb[j] += __shfl_xor_sync(0xffffffffu, gb[j], o);
            gg[j] += __shfl_xor_sync(0xffffffffu, gg[j], o);
        }
    }
    if (lp == 0) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            red[warp][lc][j] = gb[j];
            red[warp][lc][8 + j] = gg[j];
        }
    }
    __syncthreads();
    if (warp == 0 && lp == 0 && active) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float b = 0.f, g = 0.f;
#pragma unroll
            for (int w = 0; w < 8; ++w) {
                b += red[w][lc][j];
                g += red[w][lc][8 + j];
            }
            atomicAdd(dbeta + cv * 8 + j, (double)b);
            if (dgamma != nullptr) atomicAdd(dgamma + cv * 8 + j, (double)g);
        }
    }
}

template <typename GT, int ACT>
__global__ void __launch_bounds__(256)
bn_act_bwd_reduce_v2_kernel(const __half* __restrict__ x, long long xp, const GT* __restrict__ dy, long long dp,
                            const float* __restrict__ scale, const float* __restrict__ shift,
                            const float* __restrict__ mean, const float* __restrict__ invstd,
                            double* __restrict__ dgamma, double* __restrict__ dbeta, float* __restrict__ du_absmax,
                            long long pixels, int CV, float slope) {
    __shared__ float red[256][17];
    const int cv = threadIdx.x % CV;
    const int ppb = 256 / CV;
    float sc[8], sh[8], mu[8], is[8], gb[8], gg[8];
    float amax = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        gb[j] = gg[j] = 0.f;
        const int c = cv * 8 + j;
        sc[j] = __ldg(scale + c);
        sh[j] = __ldg(shift + c);
        mu[j] = mean ? __ldg(mean + c) : 0.f;
        is[j] = invstd ? __ldg(invstd + c) : 1.f;
    }
    for (long long pix = (long long)blockIdx.x * ppb + threadIdx.x / CV; pix < pixels; pix += (long long)gridDim.x * ppb) {
        float xf8[8], g8[8];
        Half8<__half>::load(x + pix * xp + cv * 8, xf8);
        Half8<GT>::load(dy + pix * dp + cv * 8, g8);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float xf = xf8[j];
            const float u = fmaf(xf, sc[j], sh[j]);
            const float du = g8[j] * act_grad(u, ACT, slope);
            gb[j] += du;
            gg[j] += du * ((xf - mu[j]) * is[j]);
            amax = fmaxf(amax, fabsf(du));
        }
    }
    if (du_absmax != nullptr) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        if ((threadIdx.x & 31) == 0 && amax > 0.f) atomicMax(reinterpret_cast<unsigned int*>(du_absmax), __float_as_uint(amax));
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        red[threadIdx.x][j] = gb[j];
        red[threadIdx.x][8 + j] = gg[j];
    }
    __syncthreads();
    // threads 0 .. CV*16-1: one (channel vector, component) each, summed over the 256/CV pixel sub-rows of the CTA
    for (int i = threadIdx.x; i < CV * 16; i += 256) {
        const int v = i / 16, comp = i % 16;
        float sum = 0.f;
        for (int k = 0; k < ppb; ++k) sum += red[v + k * CV][comp];
        if (comp < 8)
            atomicAdd(dbeta + v * 8 + comp, (double)sum);
        else if (dgamma != nullptr)
            atomicAdd(dgamma + v * 8 + comp - 8, (double)sum);
    }
}

static int bn_act_bwd_reduce_launch(const void* x, long long x_pitch, const void* dy, long long dy_pitch,
                                    const float* scale, const float* shift, const float* save_mean,
                                    const float* save_invstd, double* dgamma, double* dbeta, float* du_absmax,
                                    long long pixels, int c, int act, float slope, int grad_dtype, void* stream) {
    if (!x || !dy || !scale || !shift || !dbeta || c % 8 != 0 || x_pitch % 8 != 0 || dy_pitch % 8 != 0)
        return B2Y_ERR_INVALID;
    const int CV = c / 8;
    if (v2_ok(c) && (act == B2Y_ACT_LEAKY || act == B2Y_ACT_MISH || act == B2Y_ACT_LINEAR)) {
        const int g2 = v2_grid(pixels, CV);
        cudaStream_t st = static_cast<cudaStream_t>(stream);
#define B2Y_RED_V2(T, A)                                                                                               \
    bn_act_bwd_reduce_v2_kernel<T, A><<<g2, 256, 0, st>>>(reinterpret_cast<const __half*>(x), x_pitch,                  \
                                                          reinterpret_cast<const T*>(dy), dy_pitch, scale, shift,      \
                                                          save_mean, save_invstd, dgamma, dbeta, du_absmax, pixels,   \
                                                          CV, slope)
        if (grad_dtype == B2Y_DT_BF16) {
            if (act == B2Y_ACT_LEAKY) B2Y_RED_V2(__nv_bfloat16, B2Y_ACT_LEAKY);
            else if (act == B2Y_ACT_MISH) B2Y_RED_V2(__nv_bfloat16, B2Y_ACT_MISH);
            else B2Y_RED_V2(__nv_bfloat16, B2Y_ACT_LINEAR);
        } else {
            if (act == B2Y_ACT_LEAKY) B2Y_RED_V2(__half, B2Y_ACT_LEAKY);
            else if (act == B2Y_ACT_MISH) B2Y_RED_V2(__half, B2Y_ACT_MISH);
            else B2Y_RED_V2(__half, B2Y_ACT_LINEAR);
        }
#undef B2Y_RED_V2
        B2Y_CUDA_CHECK(cudaGetLastError());
        return B2Y_OK;
    }
    dim3 grid(1, (CV + 31) / 32);
    long long want = (pixels + 63) / 64;
    grid.x = (unsigned)(want < 1 ? 1 : (want > 132 * 4 ? 132 * 4 : want));
    if (grad_dtype == B2Y_DT_BF16)
        bn_act_bwd_reduce_kernel<__nv_bfloat16><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
            reinterpret_cast<const __half*>(x), x_pitch, reinterpret_cast<const __nv_bfloat16*>(dy), dy_pitch, scale,
            shift, save_mean, save_invstd, dgamma, dbeta, du_absmax, pixels, c, act, slope);
    else
        bn_act_bwd_reduce_kernel<__half><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
            reinterpret_cast<const __half*>(x), x_pitch, reinterpret_cast<const __half*>(dy), dy_pitch, scale, shift,
            save_mean, save_invstd, dgamma, dbeta, du_absmax, pixels, c, act, slope);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_bn_act_bwd_reduce(const void* x, long long x_pitch, const void* dy, long long dy_pitch,
                                     const float* scale, const float* shift, const float* save_mean,
                                     const float* save_invstd, float* dgamma, float* dbeta, float* du_absmax,
                                     long long pixels, int c, int act, float slope, int grad_dtype, void* stream) {
    if (!dbeta) return B2Y_ERR_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    double* acc = stream_acc(st, 2LL * c);     // [0, C) dbeta, [C, 2C) dgamma
    if (acc == nullptr) return B2Y_ERR_CUDA;
    int rc = bn_act_bwd_reduce_launch(x, x_pitch, dy, dy_pitch, scale, shift, save_mean, save_invstd,
                                      dgamma != nullptr ? acc + c : nullptr, acc, du_absmax, pixels, c, act, slope,
                                      grad_dtype, stream);
    if (rc != B2Y_OK) return rc;
    rc = acc_finalize(acc, dbeta, c, st);
    if (rc != B2Y_OK || dgamma == nullptr) return rc;
    return acc_finalize(acc + c, dgamma, c, st);
}

// ------------------------------------------------------------------------------------------------
// Grouped optimiser steps (train.py:120-150 parameter groups, per-group burn-in at :356-365).  One CTA per tile of the
// table; a tile lies inside one parameter tensor, so its group's hyper-parameters are uniform.  Its unaligned head and
// tail (< 4 elements each) are scalar, the rest goes in 16-byte vectors, OPT_VEC of them per thread loaded before any is
// updated.  HBM traffic per element: SGD reads p, g, buf and writes p, buf (20 B; 16 B on the first step, which does
// not read buf); Adam reads p, g, m, v and writes p, m, v (28 B); the EMA adds 8 B.
//
// Order of operations per element (g is the NCCL sum of the per-rank gradients):
//   1. g += (s / gs) * sign(w)  on L1 tiles -- BNOptimizer.updateBN on the averaged gradient (prune_utils.py:133-138)
//   2. g  = g * gs              -- DDP's mean over ranks
//   3. SGD:  g = g + wd*w ; buf = first ? g : mu*buf + g ; w -= lr * (g + mu*buf)
//      Adam: g = g + wd*w                                   (grad.add(param, alpha=weight_decay))
//            m = m + (1-b1)*(g - m)                         (exp_avg.lerp_(grad, 1-beta1))
//            v = v*b2 + (1-b2)*g*g                          (exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1-beta2))
//            w = w - step_size * m / (sqrt(v)/bc2_sqrt + eps)   step_size = lr/(1-b1^t), bc2_sqrt = sqrt(1-b2^t)
//   4. ema = d*ema + (1-d)*w    -- ModelEMA.update on the new weight
// ------------------------------------------------------------------------------------------------
constexpr int OPT_THREADS = 256;
constexpr int OPT_VEC = B2Y_OPT_TILE / (4 * OPT_THREADS);
static_assert(OPT_VEC * 4 * OPT_THREADS == B2Y_OPT_TILE, "a tile is OPT_VEC float4 per thread");

template <bool ADAM>
__device__ __forceinline__ float opt_elem(float w, float g, float& s0, float& s1, const B2YOptGroup& G,
                                          const B2YOptStep& hp, bool l1) {
    if (l1) g = fmaf(hp.l1_coeff, (float)((w > 0.f) - (w < 0.f)), g);       // torch.sign: 0 at 0
    const float gr = fmaf(G.weight_decay, w, g * hp.grad_scale);
    if (!ADAM) {                                                            // s0 = buf (ignored on the first step)
        s0 = hp.first_step ? gr : fmaf(G.momentum, s0, gr);
        return w - G.lr * fmaf(G.momentum, s0, gr);
    }
    s0 = fmaf(G.one_minus_beta1, gr - s0, s0);
    s1 = fmaf(G.one_minus_beta2, gr * gr, s1 * G.beta2);
    const float denom = sqrtf(s1) / G.bc2_sqrt + G.eps;
    return w - G.step_size * (s0 / denom);
}

// ModelEMA.update (utils/torch_utils.py:171-183) fused into the optimiser pass: ema = d*ema + (1-d)*w_new
__device__ __forceinline__ float ema_elem(float e, float wn, float d) { return fmaf(d, e, (1.f - d) * wn); }

template <bool ADAM, bool EMA>
__global__ void __launch_bounds__(OPT_THREADS)
opt_grouped_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ s0, float* __restrict__ s1,
                   float* __restrict__ ema, const B2YOptTile* __restrict__ tiles, const B2YOptStep hp) {
    const B2YOptTile t = tiles[blockIdx.x];
    const B2YOptGroup G = hp.group[t.flags & (B2Y_OPT_MAX_GROUPS - 1)];
    const bool l1 = (t.flags & B2Y_OPT_TILE_L1) != 0;
    const bool load_s0 = ADAM || !hp.first_step;
    const long long s = t.start, e = s + t.len;
    const long long a0 = min(e, (s + 3) & ~3LL), a1 = max(a0, e & ~3LL);   // [a0, a1): whole float4s
    const int tid = threadIdx.x;

    auto scalar = [&](long long i) {
        float m0 = load_s0 ? s0[i] : 0.f, m1 = ADAM ? s1[i] : 0.f;
        const float wn = opt_elem<ADAM>(p[i], g[i], m0, m1, G, hp, l1);
        p[i] = wn;
        s0[i] = m0;
        if (ADAM) s1[i] = m1;
        if (EMA) ema[i] = ema_elem(ema[i], wn, hp.ema_decay);
    };
    if (tid < a0 - s) scalar(s + tid);
    if (tid < e - a1) scalar(a1 + tid);

    float4* p4 = reinterpret_cast<float4*>(p);
    const float4* g4 = reinterpret_cast<const float4*>(g);
    float4* s04 = reinterpret_cast<float4*>(s0);
    float4* s14 = reinterpret_cast<float4*>(s1);
    float4* e4 = reinterpret_cast<float4*>(ema);
    const long long v0 = a0 >> 2, nv = (a1 - a0) >> 2;
    float4 vp[OPT_VEC], vg[OPT_VEC], va[OPT_VEC], vb[OPT_VEC], ve[OPT_VEC];
#pragma unroll
    for (int k = 0; k < OPT_VEC; ++k) {
        const long long j = tid + k * OPT_THREADS;
        if (j < nv) {
            vp[k] = p4[v0 + j];
            vg[k] = g4[v0 + j];
            va[k] = load_s0 ? s04[v0 + j] : make_float4(0.f, 0.f, 0.f, 0.f);
            if (ADAM) vb[k] = s14[v0 + j];
            if (EMA) ve[k] = e4[v0 + j];
        }
    }
#pragma unroll
    for (int k = 0; k < OPT_VEC; ++k) {
        const long long j = tid + k * OPT_THREADS;
        if (j < nv) {
            float4 w = vp[k], a = va[k], b = ADAM ? vb[k] : make_float4(0.f, 0.f, 0.f, 0.f);
            w.x = opt_elem<ADAM>(w.x, vg[k].x, a.x, b.x, G, hp, l1);
            w.y = opt_elem<ADAM>(w.y, vg[k].y, a.y, b.y, G, hp, l1);
            w.z = opt_elem<ADAM>(w.z, vg[k].z, a.z, b.z, G, hp, l1);
            w.w = opt_elem<ADAM>(w.w, vg[k].w, a.w, b.w, G, hp, l1);
            p4[v0 + j] = w;
            s04[v0 + j] = a;
            if (ADAM) s14[v0 + j] = b;
            if (EMA) {
                float4 em = ve[k];
                em.x = ema_elem(em.x, w.x, hp.ema_decay);
                em.y = ema_elem(em.y, w.y, hp.ema_decay);
                em.z = ema_elem(em.z, w.z, hp.ema_decay);
                em.w = ema_elem(em.w, w.w, hp.ema_decay);
                e4[v0 + j] = em;
            }
        }
    }
}

static bool opt_args_ok(const void* const* bufs, int nbufs, const B2YOptTile* tiles, int n_tiles, const B2YOptStep* hp) {
    if (n_tiles < 0 || hp == nullptr || (n_tiles > 0 && tiles == nullptr)) return false;
    for (int i = 0; i < nbufs; ++i)
        if (bufs[i] == nullptr || (reinterpret_cast<uintptr_t>(bufs[i]) & 15) != 0) return false;
    return true;
}

template <bool ADAM>
static int opt_grouped_launch(float* param, const float* grad, float* s0, float* s1, float* ema,
                              const B2YOptTile* tiles, int n_tiles, const B2YOptStep* hp, void* stream) {
    if (n_tiles == 0) return B2Y_OK;
    auto st = static_cast<cudaStream_t>(stream);
    if (ema != nullptr)
        opt_grouped_kernel<ADAM, true><<<n_tiles, OPT_THREADS, 0, st>>>(param, grad, s0, s1, ema, tiles, *hp);
    else
        opt_grouped_kernel<ADAM, false><<<n_tiles, OPT_THREADS, 0, st>>>(param, grad, s0, s1, nullptr, tiles, *hp);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_sgd_grouped(float* param, const float* grad, float* momentum_buf, float* ema,
                               const B2YOptTile* tiles_dev, int n_tiles, const B2YOptStep* hp, void* stream) {
    const void* bufs[] = {param, grad, momentum_buf};
    if (!opt_args_ok(bufs, 3, tiles_dev, n_tiles, hp) || (reinterpret_cast<uintptr_t>(ema) & 15) != 0)
        return B2Y_ERR_INVALID;
    return opt_grouped_launch<false>(param, grad, momentum_buf, nullptr, ema, tiles_dev, n_tiles, hp, stream);
}

extern "C" int b2y_adam_grouped(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, float* ema,
                                const B2YOptTile* tiles_dev, int n_tiles, const B2YOptStep* hp, void* stream) {
    const void* bufs[] = {param, grad, exp_avg, exp_avg_sq};
    if (!opt_args_ok(bufs, 4, tiles_dev, n_tiles, hp) || (reinterpret_cast<uintptr_t>(ema) & 15) != 0)
        return B2Y_ERR_INVALID;
    return opt_grouped_launch<true>(param, grad, exp_avg, exp_avg_sq, ema, tiles_dev, n_tiles, hp, stream);
}

// ------------------------------------------------------------------------------------------------
// backward of the data-movement layers (gradients are NHWC fp16, accumulated in place)
// ------------------------------------------------------------------------------------------------
// YOLO head: dp fp32 [B][na][ny][nx][no] -> d(raw) fp16 [B][ny][nx][pitch] (channel a*no+o), times `scale`
template <typename GT>
__global__ void yolo_grad_to_raw_kernel(const float* __restrict__ dp, GT* __restrict__ draw, long long pitch,
                                        int B, int na, int no, int ny, int nx, float scale,
                                        const float* __restrict__ scale_ptr) {
    if (scale_ptr != nullptr) scale *= __ldg(scale_ptr);
    const long long total = (long long)B * ny * nx * pitch;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(idx % pitch);
        long long t = idx / pitch;
        const int x = (int)(t % nx);
        t /= nx;
        const int y = (int)(t % ny);
        const int b = (int)(t / ny);
        float v = 0.f;
        if (c < na * no) {
            const int a = c / no, o = c - a * no;
            v = dp[((((long long)b * na + a) * ny + y) * nx + x) * no + o] * scale;
        }
        draw[idx] = Half8<GT>::from_f(v);
    }
}
// The same permutation, one warp per PIXEL (pitch <= 256): the (anchor, output) split of every element is computed once
// per thread, a lane issues its 8 loads (three contiguous runs of `no` floats in dp) back to back and the warp writes one
// contiguous 512-byte row -- no per-element index divisions.
template <typename GT>
__global__ void __launch_bounds__(256) yolo_grad_to_raw_pixel_kernel(const float* __restrict__ dp, GT* __restrict__ draw,
                                                                     long long pitch, int B, int na, int no, int ny,
                                                                     int nx, float scale,
                                                                     const float* __restrict__ scale_ptr) {
    if (scale_ptr != nullptr) scale *= __ldg(scale_ptr);
    const int lane = threadIdx.x & 31;
    const unsigned plane = (unsigned)(ny * nx);
    const unsigned pixels = (unsigned)B * plane;
    const unsigned warps = (gridDim.x * blockDim.x) >> 5;
    const int nel = na * no;
    long long eoff[8];       // offset of element e inside dp relative to the pixel's (b, a = 0, y, x, o = 0) entry, or -1
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int e = lane + 32 * i;
        const int a = e / no;
        eoff[i] = e < nel ? (long long)a * plane * no + (e - a * no) : -1;
    }
    for (unsigned pix = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; pix < pixels; pix += warps) {
        const unsigned b = pix / plane, yx = pix - b * plane;
        const float* src = dp + ((long long)b * na * plane + yx) * no;
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = eoff[i] >= 0 ? __ldg(src + eoff[i]) * scale : 0.f;
        GT* dst = draw + (long long)pix * pitch;
#pragma unroll
        for (int i = 0; i < 8; ++i)
            if (lane + 32 * i < pitch) dst[lane + 32 * i] = Half8<GT>::from_f(v[i]);
    }
}

extern "C" int b2y_yolo_grad_to_raw(const float* dp, void* draw, long long raw_pitch, int batch, int na, int no,
                                    int ny, int nx, float scale, const float* scale_ptr, int grad_dtype,
                                    void* stream) {
    if (!dp || !draw || raw_pitch < (long long)na * no) return B2Y_ERR_INVALID;
    const long long total = (long long)batch * ny * nx * raw_pitch;
    if (raw_pitch <= 256 && (long long)batch * ny * nx < 0x7fffffffLL) {
        long long pb = ((long long)batch * ny * nx + 7) / 8;
        if (pb > 132 * 8) pb = 132 * 8;
        if (grad_dtype == B2Y_DT_BF16)
            yolo_grad_to_raw_pixel_kernel<__nv_bfloat16><<<(int)pb, 256, 0, static_cast<cudaStream_t>(stream)>>>(
                dp, reinterpret_cast<__nv_bfloat16*>(draw), raw_pitch, batch, na, no, ny, nx, scale, scale_ptr);
        else
            yolo_grad_to_raw_pixel_kernel<__half><<<(int)pb, 256, 0, static_cast<cudaStream_t>(stream)>>>(
                dp, reinterpret_cast<__half*>(draw), raw_pitch, batch, na, no, ny, nx, scale, scale_ptr);
        B2Y_CUDA_CHECK(cudaGetLastError());
        return B2Y_OK;
    }
    if (grad_dtype == B2Y_DT_BF16)
        yolo_grad_to_raw_kernel<__nv_bfloat16><<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
            dp, reinterpret_cast<__nv_bfloat16*>(draw), raw_pitch, batch, na, no, ny, nx, scale, scale_ptr);
    else
        yolo_grad_to_raw_kernel<__half><<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
            dp, reinterpret_cast<__half*>(draw), raw_pitch, batch, na, no, ny, nx, scale, scale_ptr);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// nearest upsample backward: dx[n,y,x,:] += sum_{dy,dx<s} dup[n, y*s+dy, x*s+dx, :]
template <typename GT>
__global__ void upsample_bwd_kernel(const GT* __restrict__ dy, long long dyp, GT* __restrict__ dx,
                                    long long dxp, int B, int H, int W, int C, int s) {
    const int CV = C / 8;
    const long long total = (long long)B * H * W * CV;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(idx % CV);
        long long pix = idx / CV;
        const int x = (int)(pix % W);
        const int y = (int)((pix / W) % H);
        const int n = (int)(pix / ((long long)W * H));
        float acc[8], t8[8];
        Half8<GT>::load(dx + pix * dxp + cv * 8, acc);
        for (int a = 0; a < s; ++a)
            for (int b = 0; b < s; ++b) {
                const long long op = ((long long)n * H * s + (y * s + a)) * (W * s) + (x * s + b);
                Half8<GT>::load(dy + op * dyp + cv * 8, t8);
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] += t8[j];
            }
        Half8<GT>::store(dx + pix * dxp + cv * 8, acc);
    }
}
extern "C" int b2y_upsample_nearest_bwd(const void* dy, long long dy_pitch, void* dx, long long dx_pitch, int batch,
                                        int in_h, int in_w, int c, int scale, int grad_dtype, void* stream) {
    if (!dy || !dx || c % 8 != 0 || dy_pitch % 8 != 0 || dx_pitch % 8 != 0 || scale < 1) return B2Y_ERR_INVALID;
    const long long total = (long long)batch * in_h * in_w * (c / 8);
    if (grad_dtype == B2Y_DT_BF16)
        upsample_bwd_kernel<__nv_bfloat16><<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
            reinterpret_cast<const __nv_bfloat16*>(dy), dy_pitch, reinterpret_cast<__nv_bfloat16*>(dx), dx_pitch, batch,
            in_h, in_w, c, scale);
    else
        upsample_bwd_kernel<__half><<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
            reinterpret_cast<const __half*>(dy), dy_pitch, reinterpret_cast<__half*>(dx), dx_pitch, batch, in_h, in_w,
            c, scale);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// maxpool backward: every output pixel re-finds its arg-max (first maximum in row-major window order, as
// torch's max_pool2d does) and adds its gradient there (windows overlap for stride 1 -> fp16x2 atomics).
template <typename GT, typename GT2>
__global__ void maxpool_bwd_kernel(const __half* __restrict__ x, long long xp, const GT* __restrict__ dy,
                                   long long dyp, GT* __restrict__ dx, long long dxp, int B, int H, int W, int C,
                                   int k, int stride, int pad, int Ho, int Wo, int zero_pad) {
    const int CV = C / 2;
    const long long total = (long long)B * Ho * Wo * CV;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(idx % CV);
        long long pix = idx / CV;
        const int xo = (int)(pix % Wo);
        const int yo = (int)((pix / Wo) % Ho);
        const int n = (int)(pix / ((long long)Wo * Ho));
        float best0 = -INFINITY, best1 = -INFINITY;
        long long arg0 = -1, arg1 = -1;
        for (int kh = 0; kh < k; ++kh) {
            const int yi = yo * stride - pad + kh;
            for (int kw = 0; kw < k; ++kw) {
                const int xi = xo * stride - pad + kw;
                if (yi < 0 || yi >= H || xi < 0 || xi >= W) {
                    if (zero_pad) {  // the zero padding competes (and swallows the gradient when it wins)
                        if (0.f > best0) { best0 = 0.f; arg0 = -1; }
                        if (0.f > best1) { best1 = 0.f; arg1 = -1; }
                    }
                    continue;
                }
                const long long ip = ((long long)n * H + yi) * W + xi;
                const __half2 v = *reinterpret_cast<const __half2*>(x + ip * xp + cv * 2);
                const float a = __low2float(v), b = __high2float(v);
                if (a > best0) { best0 = a; arg0 = ip; }
                if (b > best1) { best1 = b; arg1 = ip; }
            }
        }
        const GT g0 = dy[pix * dyp + cv * 2], g1 = dy[pix * dyp + cv * 2 + 1];
        const GT zero = Half8<GT>::from_f(0.f);
        GT2 v;
        if (arg0 >= 0 && arg0 == arg1) {
            v.x = g0;
            v.y = g1;
            atomicAdd(reinterpret_cast<GT2*>(dx + arg0 * dxp + cv * 2), v);
        } else {
            if (arg0 >= 0) {
                v.x = g0;
                v.y = zero;
                atomicAdd(reinterpret_cast<GT2*>(dx + arg0 * dxp + cv * 2), v);
            }
            if (arg1 >= 0) {
                v.x = zero;
                v.y = g1;
                atomicAdd(reinterpret_cast<GT2*>(dx + arg1 * dxp + cv * 2), v);
            }
        }
    }
}
// Stride-1 "same" pooling over a small map (SPP: 5/9/13 over 20x20): one CTA owns the plane of one image x 8 channels.
// Pass 1 finds, per input row and window position, the row-window maximum and its FIRST column; pass 2 walks the window
// rows with a strict '>' -- together the first maximum in row-major window order, as the k*k scan of the general kernel
// (and torch's max_pool2d) finds it, with k + k loads.  Gradients are summed in shared memory (fp32) and added to dx by
// the owner, so there are no global atomics and the result does not depend on scheduling.
constexpr int POOL_PLANE_MAX = 576;
template <typename GT>
__global__ void __launch_bounds__(256) maxpool_plane_bwd_kernel(const __half* __restrict__ x, long long xp,
                                                                const GT* __restrict__ dy, long long dyp,
                                                                GT* __restrict__ dx, long long dxp, int H, int W,
                                                                int C, int k) {
    __shared__ __align__(16) __half sx[POOL_PLANE_MAX * 8];
    __shared__ __align__(16) __half sr[POOL_PLANE_MAX * 8];
    __shared__ unsigned char sa[POOL_PLANE_MAX * 8];
    __shared__ unsigned short sarg[POOL_PLANE_MAX * 8];   // argmax pixel (y * W + x) of every output
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
        float m = __half2float(sx[(yi * W + x0) * 8 + c]);
        int a = x0;
        for (int xi = x0 + 1; xi < x1; ++xi) {
            const float v = __half2float(sx[(yi * W + xi) * 8 + c]);
            if (v > m) { m = v; a = xi; }
        }
        sr[i] = __float2half(m);        // exact: m is one of the fp16 inputs
        sa[i] = (unsigned char)a;
    }
    __syncthreads();
    // sx is dead now: stage the plane of dy in it with 16-byte loads (the scalar 2-byte global loads of the first version
    // put one DRAM round trip into every iteration of the pass below)
    GT* sdy = reinterpret_cast<GT*>(sx);
    for (int i = threadIdx.x; i < HW; i += blockDim.x)
        reinterpret_cast<uint4*>(sdy)[i] = __ldg(reinterpret_cast<const uint4*>(dy + ((long long)n * HW + i) * dyp) + cv);
    __syncthreads();
    for (int i = threadIdx.x; i < HW * 8; i += blockDim.x) {
        const int c = i & 7, pix = i >> 3;
        const int yo = pix / W, xo = pix - yo * W;
        const int y0 = max(yo - pad, 0), y1 = min(yo - pad + k, H);
        float m = __half2float(sr[(y0 * W + xo) * 8 + c]);
        int ay = y0;
        for (int yi = y0 + 1; yi < y1; ++yi) {
            const float v = __half2float(sr[(yi * W + xo) * 8 + c]);
            if (v > m) { m = v; ay = yi; }
        }
        // NaN rows never win a strict '>' (same as the general kernel, whose -inf start is replaced by the first value)
        const int ax = sa[(ay * W + xo) * 8 + c];
        sarg[i] = (unsigned short)(ay * W + ax);
    }
    __syncthreads();
    // gather: every input sums the gradients of the outputs whose window maximum it is, in a fixed order (no atomics, so
    // the sum does not depend on scheduling)
    for (int i = threadIdx.x; i < HW; i += blockDim.x) {
        const int yi = i / W, xi = i - yi * W;
        const int ya = max(yi + pad - k + 1, 0), yb = min(yi + pad, H - 1);
        const int xa = max(xi + pad - k + 1, 0), xb = min(xi + pad, W - 1);
        float s[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int yo = ya; yo <= yb; ++yo)
            for (int xo = xa; xo <= xb; ++xo) {
                const int o = yo * W + xo;
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    if (sarg[o * 8 + j] == i) s[j] += Half8<GT>::to_f(sdy[o * 8 + j]);
            }
        GT* d = dx + ((long long)n * HW + i) * dxp + cv * 8;
        float f[8];
        Half8<GT>::load(d, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] += s[j];
        Half8<GT>::store(d, f);
    }
}

extern "C" int b2y_maxpool_bwd(const void* x, long long x_pitch, const void* dy, long long dy_pitch, void* dx,
                               long long dx_pitch, int batch, int in_h, int in_w, int c, int ksize, int stride,
                               int pad_mode, int grad_dtype, void* stream) {
    if (!x || !dy || !dx || c % 2 != 0 || x_pitch % 2 != 0 || dy_pitch % 2 != 0 || dx_pitch % 2 != 0)
        return B2Y_ERR_INVALID;
    int pad, Ho, Wo;
    if (pad_mode == 1) {
        pad = 0;
        Ho = (in_h + 1 - ksize) / stride + 1;
        Wo = (in_w + 1 - ksize) / stride + 1;
    } else {
        pad = (ksize - 1) / 2;
        Ho = (in_h + 2 * pad - ksize) / stride + 1;
        Wo = (in_w + 2 * pad - ksize) / stride + 1;
    }
    const long long total = (long long)batch * Ho * Wo * (c / 2);
    if (pad_mode != 1 && stride == 1 && (ksize & 1) && c % 8 == 0 && x_pitch % 8 == 0 && in_w <= 255 &&
        in_h * in_w <= POOL_PLANE_MAX && dy_pitch % 8 == 0 && dx_pitch % 8 == 0 &&
        ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dx)) & 15) == 0) {
        const int grid = batch * (c / 8);
        if (grad_dtype == B2Y_DT_BF16)
            maxpool_plane_bwd_kernel<__nv_bfloat16><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
                reinterpret_cast<const __half*>(x), x_pitch, reinterpret_cast<const __nv_bfloat16*>(dy), dy_pitch,
                reinterpret_cast<__nv_bfloat16*>(dx), dx_pitch, in_h, in_w, c, ksize);
        else
            maxpool_plane_bwd_kernel<__half><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
                reinterpret_cast<const __half*>(x), x_pitch, reinterpret_cast<const __half*>(dy), dy_pitch,
                reinterpret_cast<__half*>(dx), dx_pitch, in_h, in_w, c, ksize);
        B2Y_CUDA_CHECK(cudaGetLastError());
        return B2Y_OK;
    }
    if (grad_dtype == B2Y_DT_BF16)
        maxpool_bwd_kernel<__nv_bfloat16, __nv_bfloat162><<<grid_for(total, 256), 256, 0,
                                                            static_cast<cudaStream_t>(stream)>>>(
            reinterpret_cast<const __half*>(x), x_pitch, reinterpret_cast<const __nv_bfloat16*>(dy), dy_pitch,
            reinterpret_cast<__nv_bfloat16*>(dx), dx_pitch, batch, in_h, in_w, c, ksize, stride, pad, Ho, Wo,
            pad_mode == 1);
    else
        maxpool_bwd_kernel<__half, __half2><<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
            reinterpret_cast<const __half*>(x), x_pitch, reinterpret_cast<const __half*>(dy), dy_pitch,
            reinterpret_cast<__half*>(dx), dx_pitch, batch, in_h, in_w, c, ksize, stride, pad, Ho, Wo, pad_mode == 1);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// ------------------------------------------------------------------------------------------------
// stem weight gradient (Cin <= 4, NCHW fp32 image): dW[co][ci][kh][kw] += scale * sum_pix dz[pix][co] * x[...]
// CTA = 32 output channels x 8 tap groups; each thread keeps <= TPG taps of one output channel in registers.
// ------------------------------------------------------------------------------------------------
template <int TPG, typename GT>
__global__ void __launch_bounds__(256)
stem_wgrad_kernel(const float* __restrict__ x, const GT* __restrict__ dz, long long dzp, double* __restrict__ dw,
                  int B, int Cin, int H, int W, int Cout, int k, int stride, int pad, int Ho, int Wo, float scale) {
    const int taps = Cin * k * k;
    const int co_l = threadIdx.x & 31;
    const int grp = threadIdx.x >> 5;  // 0..7
    const long long M = (long long)B * Ho * Wo;
    for (int co0 = 0; co0 < Cout; co0 += 32) {
        const int co = co0 + co_l;
        float acc[TPG];
        int t_ci[TPG], t_kh[TPG], t_kw[TPG];
#pragma unroll
        for (int j = 0; j < TPG; ++j) {
            acc[j] = 0.f;
            const int t = grp * TPG + j;
            t_ci[j] = t / (k * k);
            t_kh[j] = (t / k) % k;
            t_kw[j] = t % k;
        }
        const long long per = (M + gridDim.x - 1) / gridDim.x;
        const long long m0 = (long long)blockIdx.x * per;
        const long long m1 = m0 + per < M ? m0 + per : M;
        for (long long m = m0; m < m1; ++m) {
            const int xo = (int)(m % Wo);
            const int yo = (int)((m / Wo) % Ho);
            const int n = (int)(m / ((long long)Wo * Ho));
            const float g = co < Cout ? Half8<GT>::to_f(dz[m * dzp + co]) : 0.f;
#pragma unroll
            for (int j = 0; j < TPG; ++j) {
                if (grp * TPG + j < taps) {
                    const int yi = yo * stride - pad + t_kh[j], xi = xo * stride - pad + t_kw[j];
                    float v = 0.f;
                    if (yi >= 0 && yi < H && xi >= 0 && xi < W)
                        v = __ldg(x + (((long long)n * Cin + t_ci[j]) * H + yi) * W + xi);
                    acc[j] = fmaf(g, v, acc[j]);
                }
            }
        }
        if (co < Cout) {
#pragma unroll
            for (int j = 0; j < TPG; ++j)
                if (grp * TPG + j < taps) atomicAdd(dw + (long long)co * taps + grp * TPG + j, (double)(acc[j] * scale));
        }
    }
}
extern "C" int b2y_stem_conv_bwd_weight(const b2y_conv_desc* d, const float* x_nchw, const void* dz, float* dw_oihw,
                                        float scale, int grad_dtype, void* stream) {
    if (!d || !x_nchw || !dz || !dw_oihw) return B2Y_ERR_INVALID;
    const int taps = d->in_c * d->ksize * d->ksize;
    if (d->in_c > 4 || taps > 8 * 5) return B2Y_ERR_UNSUPPORTED;
    double* acc = stream_acc(static_cast<cudaStream_t>(stream), (long long)d->out_c * taps);
    if (acc == nullptr) return B2Y_ERR_CUDA;
    const long long M = (long long)d->batch * d->out_h * d->out_w;
    int grid = (int)((M + 1023) / 1024);
    if (grid > 132 * 8) grid = 132 * 8;
    if (grid < 1) grid = 1;
    if (grad_dtype == B2Y_DT_BF16)
        stem_wgrad_kernel<5, __nv_bfloat16><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
            x_nchw, reinterpret_cast<const __nv_bfloat16*>(dz), d->out_pitch, acc, d->batch, d->in_c, d->in_h,
            d->in_w, d->out_c, d->ksize, d->stride, d->pad, d->out_h, d->out_w, scale);
    else
        stem_wgrad_kernel<5, __half><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
            x_nchw, reinterpret_cast<const __half*>(dz), d->out_pitch, acc, d->batch, d->in_c, d->in_h, d->in_w,
            d->out_c, d->ksize, d->stride, d->pad, d->out_h, d->out_w, scale);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return acc_finalize(acc, dw_oihw, (long long)d->out_c * taps, static_cast<cudaStream_t>(stream));
}
