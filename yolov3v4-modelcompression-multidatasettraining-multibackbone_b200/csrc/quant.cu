// Power-of-two fake quantisation, calibration reductions and int8 weight packing
// (reference utils/quantized/quantized_ptq_cos.py:14-113, utils/quantized/quantized_google.py:16-219).
// All HBM-bound: one pass over the data, 16-byte vector accesses, warp-shuffle + one atomic per CTA for reductions.
#include "b200yolo.h"
#include <cmath>

#include "common.cuh"

using namespace b2y;

static inline int grid_for(long long n, int block) {
    long long g = (n + block - 1) / block;
    if (g < 1) g = 1;
    if (g > 132LL * 16) g = 132LL * 16;
    return (int)g;
}

__device__ __forceinline__ float rha(float x) { return copysignf(floorf(fabsf(x) + 0.5f), x); }  // ptq_cos.py:14-20

// y = clamp(round(x / s), lo, hi) * s      (ptq_cos.py:44-62, 89-92; the division is a true division, not
// a multiply by 1/s, although for power-of-two s both are exact)
__global__ void fakequant_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, float scale,
                                 float lo, float hi) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x) {
        float q = rha(x[i] / scale);
        y[i] = fminf(fmaxf(q, lo), hi) * scale;
    }
}

extern "C" int b2y_fakequant_f32(const float* x, float* y, long long n, float scale, float lo, float hi,
                                 void* stream) {
    if (!x || !y || n < 0 || !(scale > 0.f)) return B2Y_ERR_INVALID;
    fakequant_kernel<<<grid_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, y, n, scale, lo, hi);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// Straight-through backward of the fake-quantiser (google.py:81-92 Round STE + torch.clamp's gradient mask):
//   dx = g * [lo <= round(x / s) <= hi] * gain       (gain = 1 for the symmetric power-of-two quantisers)
__global__ void fakequant_bwd_kernel(const float* __restrict__ x, const float* __restrict__ g, float* __restrict__ dx,
                                     long long n, float scale, float lo, float hi, float gain) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x) {
        const float q = rha(x[i] / scale);
        dx[i] = (q >= lo && q <= hi) ? g[i] * gain : 0.f;
    }
}

extern "C" int b2y_fakequant_bwd_f32(const float* x, const float* g, float* dx, long long n, float scale, float lo,
                                     float hi, float gain, void* stream) {
    if (!x || !g || !dx || n < 0 || !(scale > 0.f)) return B2Y_ERR_INVALID;
    fakequant_bwd_kernel<<<grid_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, g, dx, n, scale, lo, hi,
                                                                                         gain);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// TPSQ quantiser (quantized_TPSQ.py:66-130): soft clamp to [-P, P], q = round(c * qmax / P), y = q * P / 2^(bits-1)
//   forward:  y;   backward pieces for the learned range P:  dy/dx = [|x| < P] * qmax / 2^(bits-1),
//   dy/dP = q / 2^(bits-1) + (qmax / 2^(bits-1)) * (sign(x) [|x| >= P] - c / P)       -> sum(g * dy/dP) in *dp_sum (double)
__global__ void tpsq_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, float P, float qmax,
                                float qden) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x) {
        const float v = x[i];
        const float c = 0.5f * (fabsf(v + P) - fabsf(v - P));
        y[i] = rha(c * qmax / P) * P / qden;
    }
}
__global__ void tpsq_bwd_kernel(const float* __restrict__ x, const float* __restrict__ g, float* __restrict__ dx,
                                double* __restrict__ dp_sum, long long n, float P, float qmax, float qden) {
    double acc = 0.0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x) {
        const float v = x[i], gi = g[i];
        const float c = 0.5f * (fabsf(v + P) - fabsf(v - P));
        const float q = rha(c * qmax / P);
        // d c / d x = 0.5 (sign(x+P) - sign(x-P)),  d c / d P = 0.5 (sign(x+P) + sign(x-P))   (torch.abs' subgradient)
        const float sp = (v + P > 0.f) - (v + P < 0.f), sm = (v - P > 0.f) - (v - P < 0.f);
        const float dcdx = 0.5f * (sp - sm), dcdp = 0.5f * (sp + sm);
        if (dx != nullptr) dx[i] = gi * dcdx * qmax / qden;
        acc += (double)gi * ((double)q / qden + (double)(qmax / qden) * ((double)dcdp - (double)c / P));
    }
    __shared__ double sh[256];
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) atomicAdd(dp_sum, sh[0]);
}

extern "C" int b2y_tpsq_fwd_f32(const float* x, float* y, long long n, float range_pow2, int bits, void* stream) {
    if (!x || !y || n < 0 || !(range_pow2 > 0.f) || bits < 2 || bits > 16) return B2Y_ERR_INVALID;
    tpsq_fwd_kernel<<<grid_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        x, y, n, range_pow2, (float)((1 << (bits - 1)) - 1), (float)(1 << (bits - 1)));
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}
extern "C" int b2y_tpsq_bwd_f32(const float* x, const float* g, float* dx, double* dp_sum, long long n, float range_pow2,
                                int bits, void* stream) {
    if (!x || !g || !dp_sum || n < 0 || !(range_pow2 > 0.f) || bits < 2 || bits > 16) return B2Y_ERR_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    B2Y_CUDA_CHECK(cudaMemsetAsync(dp_sum, 0, sizeof(double), st));
    tpsq_bwd_kernel<<<grid_for(n, 256), 256, 0, st>>>(x, g, dx, dp_sum, n, range_pow2, (float)((1 << (bits - 1)) - 1),
                                                      (float)(1 << (bits - 1)));
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// fp16 NHWC -> int8 NHWC integer codes
__global__ void quantize_f16_i8_kernel(const __half* __restrict__ x, long long xp, int8_t* __restrict__ q,
                                       long long qp, long long pixels, int C, float scale, float lo, float hi) {
    const int CV = C / 8;
    const long long total = pixels * CV;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(idx % CV);
        const long long pix = idx / CV;
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + pix * xp) + cv);
        const __half* h = reinterpret_cast<const __half*>(&v);
        uint2 o;
        int8_t* ob = reinterpret_cast<int8_t*>(&o);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float r = rha(__half2float(h[j]) / scale);
            ob[j] = (int8_t)(int)fminf(fmaxf(r, lo), hi);
        }
        *reinterpret_cast<uint2*>(q + pix * qp + cv * 8) = o;
    }
}

extern "C" int b2y_quantize_f16_to_i8(const void* x, long long x_pitch, void* q, long long q_pitch, long long pixels,
                                      int c, float scale, float lo, float hi, void* stream) {
    if (!x || !q || c % 8 != 0 || x_pitch % 8 != 0 || q_pitch % 8 != 0 || !(scale > 0.f)) return B2Y_ERR_INVALID;
    quantize_f16_i8_kernel<<<grid_for(pixels * (c / 8), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const __half*>(x), x_pitch, reinterpret_cast<int8_t*>(q), q_pitch, pixels, c, scale, lo, hi);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// COSPTQ calibration (ptq_cos.py:71-87): all candidate power-of-two scales in ONE pass over x.
// Per candidate k: dot_k = sum x*q_k, qq_k = sum q_k^2 ; xx = sum x^2.  cos_k = dot_k / sqrt(xx*qq_k).
// Accumulated in double so that the argmax matches torch.cosine_similarity on the ties the reference resolves
// with a strict '>'.
#define B2Y_MAX_CAND 24
__global__ void cos_search_kernel(const float* __restrict__ x, long long n, int bits, int n_cand, int step0,
                                  double* __restrict__ acc /* [1 + 2*n_cand] */) {
    __shared__ double sh[(1 + 2 * B2Y_MAX_CAND)];
    for (int i = threadIdx.x; i < 1 + 2 * n_cand; i += blockDim.x) sh[i] = 0.0;
    __syncthreads();
    const float lo = -(float)(1 << (bits - 1)), hi = (float)((1 << (bits - 1)) - 1);
    float xx = 0.f;
    float dot[B2Y_MAX_CAND], qq[B2Y_MAX_CAND];
#pragma unroll
    for (int k = 0; k < B2Y_MAX_CAND; ++k) dot[k] = qq[k] = 0.f;
    int cnt = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x) {
        const float v = x[i];
        xx += v * v;
#pragma unroll
        for (int k = 0; k < B2Y_MAX_CAND; ++k) {
            if (k < n_cand) {
                const float scale = exp2f((float)(k + step0)) / (float)(1 << (bits - 1));
                const float q = fminf(fmaxf(rha(v / scale), lo), hi) * scale;
                dot[k] += v * q;
                qq[k] += q * q;
            }
        }
        // flush fp32 partials into double every 64 elements to bound the rounding error
        if (++cnt == 64) {
            cnt = 0;
            atomicAdd(&sh[0], (double)xx);
            xx = 0.f;
#pragma unroll
            for (int k = 0; k < B2Y_MAX_CAND; ++k)
                if (k < n_cand) {
                    atomicAdd(&sh[1 + k], (double)dot[k]);
                    atomicAdd(&sh[1 + n_cand + k], (double)qq[k]);
                    dot[k] = qq[k] = 0.f;
                }
        }
    }
    atomicAdd(&sh[0], (double)xx);
#pragma unroll
    for (int k = 0; k < B2Y_MAX_CAND; ++k)
        if (k < n_cand) {
            atomicAdd(&sh[1 + k], (double)dot[k]);
            atomicAdd(&sh[1 + n_cand + k], (double)qq[k]);
        }
    __syncthreads();
    for (int i = threadIdx.x; i < 1 + 2 * n_cand; i += blockDim.x) atomicAdd(acc + i, sh[i]);
}

__global__ void cos_finalize_kernel(const double* __restrict__ acc, int n_cand, float* __restrict__ out) {
    const int k = threadIdx.x;
    if (k < n_cand) {
        const double xx = acc[0], dot = acc[1 + k], qq = acc[1 + n_cand + k];
        // torch.cosine_similarity: dot / max(||x||*||q||, eps), eps = 1e-8
        const double den = fmax(sqrt(xx) * sqrt(qq), 1e-8);
        out[k] = (float)(dot / den);
    }
}

// candidate k uses float_range = 2^(k + step0): the conv quantisers search step0 = -5 over bits+7 candidates
// (ptq_cos.py:71-87), the shortcut quantisers step0 = 0 over `bits` candidates (ptq_cos.py:836-868, 1158-1197)
extern "C" int b2y_cos_scale_search_ex(const float* x, long long n, int bits, int n_cand, int step0, float* out_cos,
                                       void* workspace, size_t workspace_bytes, void* stream) {
    if (!x || !out_cos || !workspace || n_cand < 1 || n_cand > B2Y_MAX_CAND || bits < 2 || bits > 16)
        return B2Y_ERR_INVALID;
    if (workspace_bytes < sizeof(double) * (1 + 2 * (size_t)n_cand)) return B2Y_ERR_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    double* acc = reinterpret_cast<double*>(workspace);
    B2Y_CUDA_CHECK(cudaMemsetAsync(acc, 0, sizeof(double) * (1 + 2 * n_cand), st));
    int grid = grid_for(n, 256);
    if (grid > 132 * 4) grid = 132 * 4;
    cos_search_kernel<<<grid, 256, 0, st>>>(x, n, bits, n_cand, step0, acc);
    cos_finalize_kernel<<<1, 32, 0, st>>>(acc, n_cand, out_cos);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_cos_scale_search(const float* x, long long n, int bits, int n_cand, float* out_cos,
                                    void* workspace, size_t workspace_bytes, void* stream) {
    return b2y_cos_scale_search_ex(x, n, bits, n_cand, -5, out_cos, workspace, workspace_bytes, stream);
}

// min / max trackers (google.py:16-77): per tensor ('L') or per output channel ('C' = per row of [rows][cols])
__device__ __forceinline__ void atomic_min_f(float* a, float v) {
    int* ai = reinterpret_cast<int*>(a);
    int old = *ai;
    while (v < __int_as_float(old)) {
        int assumed = old;
        old = atomicCAS(ai, assumed, __float_as_int(v));
        if (old == assumed) break;
    }
}
__device__ __forceinline__ void atomic_max_f(float* a, float v) {
    int* ai = reinterpret_cast<int*>(a);
    int old = *ai;
    while (v > __int_as_float(old)) {
        int assumed = old;
        old = atomicCAS(ai, assumed, __float_as_int(v));
        if (old == assumed) break;
    }
}
__global__ void minmax_init_kernel(float* out, long long n_pairs) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_pairs;
         i += (long long)gridDim.x * blockDim.x) {
        out[2 * i] = __int_as_float(0x7f800000);      // +inf
        out[2 * i + 1] = __int_as_float(0xff800000);  // -inf
    }
}
__global__ void minmax_kernel(const float* __restrict__ x, long long rows, long long cols, int per_row,
                              float* __restrict__ out) {
    // grid.y strides over rows (per_row) ; the tensor-level mode uses a single "row" of rows*cols elements
    const long long nrow = per_row ? rows : 1;
    const long long ncol = per_row ? cols : rows * cols;
    for (long long r = blockIdx.y; r < nrow; r += gridDim.y) {
        float mn = __int_as_float(0x7f800000), mx = __int_as_float(0xff800000);
        const float* xr = x + r * ncol;
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < ncol;
             i += (long long)gridDim.x * blockDim.x) {
            const float v = xr[i];
            mn = fminf(mn, v);
            mx = fmaxf(mx, v);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        }
        if ((threadIdx.x & 31) == 0) {
            atomic_min_f(out + 2 * r, mn);
            atomic_max_f(out + 2 * r + 1, mx);
        }
    }
}

extern "C" int b2y_minmax_f32(const float* x, long long rows, long long cols, int per_row, float* out_minmax,
                              void* stream) {
    if (!x || !out_minmax || rows <= 0 || cols <= 0) return B2Y_ERR_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long nrow = per_row ? rows : 1;
    const long long ncol = per_row ? cols : rows * cols;
    minmax_init_kernel<<<grid_for(nrow, 256), 256, 0, st>>>(out_minmax, nrow);
    dim3 grid((unsigned)((ncol + 256 * 8 - 1) / (256 * 8) > 0 ? (ncol + 256 * 8 - 1) / (256 * 8) : 1),
              (unsigned)(nrow > 65535 ? 65535 : nrow));
    if (grid.x > 592) grid.x = 592;
    minmax_kernel<<<grid, 256, 0, st>>>(x, rows, cols, per_row, out_minmax);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// OIHW fp32 (already BN-folded) -> int8 [O][kh][kw][I] codes at scale w_scale
__global__ void pack_qweights_kernel(const float* __restrict__ w, int O, int I, int k, float scale, float lo, float hi,
                                     int8_t* __restrict__ out) {
    const long long total = (long long)O * I * k * k;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(idx % I);
        long long t = idx / I;
        const int kw = (int)(t % k);
        t /= k;
        const int kh = (int)(t % k);
        const int o = (int)(t / k);
        const float v = w[(((long long)o * I + i) * k + kh) * k + kw];
        out[idx] = (int8_t)(int)fminf(fmaxf(rha(v / scale), lo), hi);
    }
}

extern "C" int b2y_pack_qconv_weights(const float* w_oihw_folded, int out_c, int in_c, int ksize, float w_scale,
                                      float lo, float hi, void* w_i8, void* stream) {
    if (!w_oihw_folded || !w_i8 || out_c <= 0 || in_c <= 0 || ksize <= 0 || !(w_scale > 0.f)) return B2Y_ERR_INVALID;
    const long long total = (long long)out_c * in_c * ksize * ksize;
    pack_qweights_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        w_oihw_folded, out_c, in_c, ksize, w_scale, lo, hi, reinterpret_cast<int8_t*>(w_i8));
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// ------------------------------------------------------------------------------------------------
// int8 data-movement layers of the quantised graph (eval): shortcut and concat requantisation
// reference: COSPTQuantizedShortcut_min.forward (ptq_cos.py:876-884, 931-933, 1031) and
//            COSPTQuantizedFeatureConcat.forward eval branch (ptq_cos.py:1540-1546)
// ------------------------------------------------------------------------------------------------
// out = clamp(round((round(x*sx_in/scale_x)*scale_x + round(a*sa_in/scale_a)*scale_a) / scale_sum))
__global__ void qshortcut_kernel(const int8_t* __restrict__ x, long long xp, const int8_t* __restrict__ a,
                                 long long ap, int8_t* __restrict__ out, long long op, long long pixels, int C,
                                 float sx_in, float scale_x, float sa_in, float scale_a, float scale_sum, float lo,
                                 float hi) {
    const int CV = C / 16;
    const long long total = pixels * CV;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(idx % CV);
        const long long pix = idx / CV;
        const uint4 xv = __ldg(reinterpret_cast<const uint4*>(x + pix * xp) + cv);
        const uint4 av = __ldg(reinterpret_cast<const uint4*>(a + pix * ap) + cv);
        const int8_t* xb = reinterpret_cast<const int8_t*>(&xv);
        const int8_t* ab = reinterpret_cast<const int8_t*>(&av);
        uint4 ov;
        int8_t* ob = reinterpret_cast<int8_t*>(&ov);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const float xf = rha(((float)xb[j] * sx_in) / scale_x) * scale_x;   // rounded, NOT clamped
            const float af = rha(((float)ab[j] * sa_in) / scale_a) * scale_a;
            const float q = rha((xf + af) / scale_sum);
            ob[j] = (int8_t)(int)fminf(fmaxf(q, lo), hi);
        }
        reinterpret_cast<uint4*>(out + pix * op)[cv] = ov;
    }
}
// v2: a thread owns one 16-channel vector and strides the pixels (no index divisions).  EXACT_MUL: all three scales are
// powers of two (what the COSPTQ quantiser produces, ptq_cos.py:60-75), so x / s == x * (1/s) bit for bit and the three
// IEEE divisions per element become multiplications; other scales keep the divisions.
template <bool EXACT_MUL>
__global__ void __launch_bounds__(256)
qshortcut_v2_kernel(const int8_t* __restrict__ x, long long xp, const int8_t* __restrict__ a, long long ap,
                    int8_t* __restrict__ out, long long op, long long pixels, int CV, float sx_in, float scale_x,
                    float sa_in, float scale_a, float scale_sum, float lo, float hi) {
    const int cv = threadIdx.x % CV;
    const int ppb = 256 / CV;
    const float rx = 1.f / scale_x, ra = 1.f / scale_a, rs = 1.f / scale_sum;
    for (long long pix = (long long)blockIdx.x * ppb + threadIdx.x / CV; pix < pixels; pix += (long long)gridDim.x * ppb) {
        const uint4 xv = __ldg(reinterpret_cast<const uint4*>(x + pix * xp) + cv);
        const uint4 av = __ldg(reinterpret_cast<const uint4*>(a + pix * ap) + cv);
        const int8_t* xb = reinterpret_cast<const int8_t*>(&xv);
        const int8_t* ab = reinterpret_cast<const int8_t*>(&av);
        uint4 ov;
        int8_t* ob = reinterpret_cast<int8_t*>(&ov);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const float xs = (float)xb[j] * sx_in, as = (float)ab[j] * sa_in;
            const float xf = rha(EXACT_MUL ? xs * rx : xs / scale_x) * scale_x;   // rounded, NOT clamped
            const float af = rha(EXACT_MUL ? as * ra : as / scale_a) * scale_a;
            const float q = rha(EXACT_MUL ? (xf + af) * rs : (xf + af) / scale_sum);
            ob[j] = (int8_t)(int)fminf(fmaxf(q, lo), hi);
        }
        reinterpret_cast<uint4*>(out + pix * op)[cv] = ov;
    }
}
static inline bool is_pow2f(float v) {
    int e = 0;
    return v > 0.f && frexpf(v, &e) == 0.5f;
}

extern "C" int b2y_qshortcut_i8(const void* x, long long x_pitch, const void* a, long long a_pitch, void* out,
                                long long out_pitch, long long pixels, int c, float sx_in, float scale_x,
                                float sa_in, float scale_a, float scale_sum, float lo, float hi, void* stream) {
    if (!x || !a || !out || c % 16 != 0 || x_pitch % 16 != 0 || a_pitch % 16 != 0 || out_pitch % 16 != 0)
        return B2Y_ERR_INVALID;
    const int CV = c / 16;
    if (CV <= 256 && 256 % CV == 0) {
        const int ppb = 256 / CV;
        long long g = (pixels + ppb - 1) / ppb;
        if (g > 132 * 8) g = 132 * 8;
        if (g < 1) g = 1;
        const bool exact = is_pow2f(scale_x) && is_pow2f(scale_a) && is_pow2f(scale_sum);
        cudaStream_t st = static_cast<cudaStream_t>(stream);
        if (exact)
            qshortcut_v2_kernel<true><<<(int)g, 256, 0, st>>>(
                reinterpret_cast<const int8_t*>(x), x_pitch, reinterpret_cast<const int8_t*>(a), a_pitch,
                reinterpret_cast<int8_t*>(out), out_pitch, pixels, CV, sx_in, scale_x, sa_in, scale_a, scale_sum, lo, hi);
        else
            qshortcut_v2_kernel<false><<<(int)g, 256, 0, st>>>(
                reinterpret_cast<const int8_t*>(x), x_pitch, reinterpret_cast<const int8_t*>(a), a_pitch,
                reinterpret_cast<int8_t*>(out), out_pitch, pixels, CV, sx_in, scale_x, sa_in, scale_a, scale_sum, lo, hi);
        B2Y_CUDA_CHECK(cudaGetLastError());
        return B2Y_OK;
    }
    qshortcut_kernel<<<grid_for(pixels * (c / 16), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const int8_t*>(x), x_pitch, reinterpret_cast<const int8_t*>(a), a_pitch,
        reinterpret_cast<int8_t*>(out), out_pitch, pixels, c, sx_in, scale_x, sa_in, scale_a, scale_sum, lo, hi);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// out = clamp(round(x * s_in / s_out))   (channel-slice copy with requantisation; s_in == s_out is a plain copy)
__global__ void requant_kernel(const int8_t* __restrict__ x, long long xp, int8_t* __restrict__ out, long long op,
                               long long pixels, int C, float s_in, float s_out, float lo, float hi) {
    const int CV = C / 16;
    const long long total = pixels * CV;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(idx % CV);
        const long long pix = idx / CV;
        const uint4 xv = __ldg(reinterpret_cast<const uint4*>(x + pix * xp) + cv);
        const int8_t* xb = reinterpret_cast<const int8_t*>(&xv);
        uint4 ov;
        int8_t* ob = reinterpret_cast<int8_t*>(&ov);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const float q = rha(((float)xb[j] * s_in) / s_out);
            ob[j] = (int8_t)(int)fminf(fmaxf(q, lo), hi);
        }
        reinterpret_cast<uint4*>(out + pix * op)[cv] = ov;
    }
}
extern "C" int b2y_requant_i8(const void* x, long long x_pitch, void* out, long long out_pitch, long long pixels,
                              int c, float s_in, float s_out, float lo, float hi, void* stream) {
    if (!x || !out || c % 16 != 0 || x_pitch % 16 != 0 || out_pitch % 16 != 0) return B2Y_ERR_INVALID;
    requant_kernel<<<grid_for(pixels * (c / 16), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const int8_t*>(x), x_pitch, reinterpret_cast<int8_t*>(out), out_pitch, pixels, c, s_in, s_out,
        lo, hi);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// nearest upsample of int8 NHWC codes (scale unchanged)
__global__ void upsample_i8_kernel(const int8_t* __restrict__ x, long long xp, int8_t* __restrict__ y, long long yp,
                                   int B, int H, int W, int C, int s) {
    const int CV = C / 16;
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
        reinterpret_cast<uint4*>(y + pix * yp)[cv] = __ldg(reinterpret_cast<const uint4*>(x + ipix * xp) + cv);
    }
}
extern "C" int b2y_upsample_nearest_i8(const void* x, long long x_pitch, void* y, long long y_pitch, int batch,
                                       int in_h, int in_w, int c, int scale, void* stream) {
    if (!x || !y || c % 16 != 0 || x_pitch % 16 != 0 || y_pitch % 16 != 0 || scale < 1) return B2Y_ERR_INVALID;
    const long long total = (long long)batch * in_h * scale * in_w * scale * (c / 16);
    upsample_i8_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const int8_t*>(x), x_pitch, reinterpret_cast<int8_t*>(y), y_pitch, batch, in_h, in_w, c,
        scale);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// Max-pool of int8 NHWC codes (the plain nn.MaxPool2d of the google-QAT graph, models.py:207-214).  Every input sits on
// one power-of-two grid, so the max of the codes is the code of the max.  16 channels (one 16-byte vector) per thread,
// four signed-byte maxima per __vmaxs4.
__device__ __forceinline__ uint4 vmax_s8x16(uint4 a, uint4 b) {
    return make_uint4(__vmaxs4(a.x, b.x), __vmaxs4(a.y, b.y), __vmaxs4(a.z, b.z), __vmaxs4(a.w, b.w));
}

// any window: out-of-range taps are skipped (-inf padding); zero_pad adds code 0 when the window touches the right or
// bottom pad of ZeroPad2d((0,1,0,1))
__global__ void maxpool_i8_kernel(const int8_t* __restrict__ x, long long xp, int8_t* __restrict__ y, long long yp,
                                  int H, int W, int CV, int k, int stride, int pad, int Ho, int Wo, long long total,
                                  int zero_pad) {
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int cv = (int)(idx % CV);
        const long long pix = idx / CV;
        const int xo = (int)(pix % Wo);
        const int yo = (int)((pix / Wo) % Ho);
        const long long n = pix / ((long long)Wo * Ho);
        uint4 m = make_uint4(0x80808080u, 0x80808080u, 0x80808080u, 0x80808080u);
        bool touched_pad = false;
        for (int kh = 0; kh < k; ++kh) {
            const int yi = yo * stride - pad + kh;
            for (int kw = 0; kw < k; ++kw) {
                const int xi = xo * stride - pad + kw;
                if (yi < 0 || yi >= H || xi < 0 || xi >= W) {
                    touched_pad = true;
                    continue;
                }
                m = vmax_s8x16(m, __ldg(reinterpret_cast<const uint4*>(x + ((n * H + yi) * W + xi) * xp) + cv));
            }
        }
        if (zero_pad && touched_pad) m = vmax_s8x16(m, make_uint4(0u, 0u, 0u, 0u));
        reinterpret_cast<uint4*>(y + pix * yp)[cv] = m;
    }
}

// Stride-1 "same" pooling (SPP: k = 5 / 9 / 13) over a map of up to POOL_PLANE_I8_MAX pixels: one CTA holds the plane of
// one image x 16 channels in shared memory and takes the window as a row pass then a column pass (2k loads, not k*k),
// as maxpool_plane_kernel does for fp16.  Clipping the window at the border is the -inf padding.
constexpr int POOL_PLANE_I8_MAX = 1024;   // 32 x 32 pixels, 2 x 16 KB of shared memory
__global__ void __launch_bounds__(256) maxpool_i8_plane_kernel(const int8_t* __restrict__ x, long long xp,
                                                               int8_t* __restrict__ y, long long yp, int H, int W,
                                                               int CV, int k) {
    __shared__ uint4 sx[POOL_PLANE_I8_MAX];
    __shared__ uint4 sr[POOL_PLANE_I8_MAX];
    const long long n = blockIdx.x / CV;
    const int cv = blockIdx.x - (int)(n * CV);
    const int HW = H * W, pad = (k - 1) / 2;
    for (int i = threadIdx.x; i < HW; i += blockDim.x)
        sx[i] = __ldg(reinterpret_cast<const uint4*>(x + (n * HW + i) * xp) + cv);
    __syncthreads();
    for (int i = threadIdx.x; i < HW; i += blockDim.x) {
        const int yi = i / W, xo = i - yi * W;
        const int x0 = max(xo - pad, 0), x1 = min(xo - pad + k, W);
        uint4 m = sx[yi * W + x0];
        for (int xi = x0 + 1; xi < x1; ++xi) m = vmax_s8x16(m, sx[yi * W + xi]);
        sr[i] = m;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < HW; i += blockDim.x) {
        const int yo = i / W, xo = i - yo * W;
        const int y0 = max(yo - pad, 0), y1 = min(yo - pad + k, H);
        uint4 m = sr[y0 * W + xo];
        for (int yi = y0 + 1; yi < y1; ++yi) m = vmax_s8x16(m, sr[yi * W + xo]);
        reinterpret_cast<uint4*>(y + (n * HW + i) * yp)[cv] = m;
    }
}

extern "C" int b2y_maxpool_i8(const void* x, long long x_pitch, void* y, long long y_pitch, int batch, int in_h,
                              int in_w, int c, int ksize, int stride, int pad_mode, void* stream) {
    if (!x || !y || batch < 1 || in_h < 1 || in_w < 1 || c < 16 || c % 16 != 0 || x_pitch < c || y_pitch < c ||
        x_pitch % 16 != 0 || y_pitch % 16 != 0 || ksize < 1 || stride < 1 || (pad_mode != 0 && pad_mode != 1))
        return B2Y_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15)) return B2Y_ERR_INVALID;
    const int pad = pad_mode == 1 ? 0 : (ksize - 1) / 2;
    const int extra = pad_mode == 1 ? 1 : 2 * pad;      // ZeroPad2d((0,1,0,1)) widens by one on one side only
    if (in_h + extra < ksize || in_w + extra < ksize) return B2Y_ERR_INVALID;
    const int Ho = (in_h + extra - ksize) / stride + 1, Wo = (in_w + extra - ksize) / stride + 1;
    const int CV = c / 16;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (pad_mode == 0 && stride == 1 && (ksize & 1) && in_h * in_w <= POOL_PLANE_I8_MAX &&
        (long long)batch * CV <= 0x7fffffffLL) {
        maxpool_i8_plane_kernel<<<batch * CV, 256, 0, st>>>(reinterpret_cast<const int8_t*>(x), x_pitch,
                                                            reinterpret_cast<int8_t*>(y), y_pitch, in_h, in_w, CV, ksize);
    } else {
        const long long total = (long long)batch * Ho * Wo * CV;
        maxpool_i8_kernel<<<grid_for(total, 256), 256, 0, st>>>(reinterpret_cast<const int8_t*>(x), x_pitch,
                                                               reinterpret_cast<int8_t*>(y), y_pitch, in_h, in_w, CV,
                                                               ksize, stride, pad, Ho, Wo, total, pad_mode);
    }
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// First quantised layer: the image is float (not on an int8 grid), so conv 0 runs in fp32 on the fake-quantised
// weights (exactly what the reference does, ptq_cos.py:288-296) and only its output is requantised to int8.
__global__ void __launch_bounds__(128)
stem_conv_q_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                   int8_t* __restrict__ y, int B, int Cin, int H, int W, int Cout, int k, int stride, int pad, int Ho,
                   int Wo, long long out_pitch, int act, float slope, float out_scale, float lo, float hi) {
    constexpr int CO = 32;
    extern __shared__ float sw[];
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
            int8_t* op = y + m * out_pitch + co0;
#pragma unroll
            for (int c = 0; c < CO; ++c) {
                if (co0 + c < Cout) {
                    const float v = apply_act(acc[c] + sw[taps * CO + c], act, slope);
                    op[c] = (int8_t)(int)fminf(fmaxf(rha(v / out_scale), lo), hi);
                }
            }
        }
    }
}
extern "C" int b2y_stem_conv_fwd_q(const b2y_conv_desc* d, const float* x_nchw, const float* w_q, const float* bias_q,
                                   void* y_i8, float out_scale, float lo, float hi, void* stream) {
    if (!d || !x_nchw || !w_q || !y_i8 || !(out_scale > 0.f)) return B2Y_ERR_INVALID;
    if (d->in_c < 1 || d->in_c > 4) return B2Y_ERR_UNSUPPORTED;
    const long long M = (long long)d->batch * d->out_h * d->out_w;
    const int taps = d->in_c * d->ksize * d->ksize;
    const size_t smem = (size_t)(taps * 32 + 32) * sizeof(float);
    if (smem > 48 * 1024) return B2Y_ERR_UNSUPPORTED;
    int grid = (int)((M + 127) / 128);
    if (grid > 132 * 16) grid = 132 * 16;
    stem_conv_q_kernel<<<grid, 128, smem, static_cast<cudaStream_t>(stream)>>>(
        x_nchw, w_q, bias_q, reinterpret_cast<int8_t*>(y_i8), d->batch, d->in_c, d->in_h, d->in_w, d->out_c, d->ksize,
        d->stride, d->pad, d->out_h, d->out_w, d->out_pitch, d->act, d->slope, out_scale, lo, hi);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}
