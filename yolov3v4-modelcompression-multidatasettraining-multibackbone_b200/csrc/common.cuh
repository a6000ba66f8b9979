// Shared device helpers for the b200yolo kernels (sm_90a).
// Thin inline-PTX wrappers around mbarrier / TMA / clusters / wgmma operands.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "b200yolo.h"  // status codes + activation ids (single source of truth)
#include "wgmma.cuh"

// (in_c, k) pairs of the first layer's two im2col kernels, stem_fused_kernel (stem_tc.cu) and stem_fullpack_kernel
// (conv_tc.cu): odd k and in_c * k * k <= 32, so that one output pixel's receptive field fits one 32-column fp16 GEMM
// row.  Each kernel's dispatch expands X(in_c, k) over this list; layout.stem_path states the same rule in Python.
#define B2Y_STEM_IM2COL_SHAPES(X) X(1, 1) X(2, 1) X(3, 1) X(4, 1) X(1, 3) X(2, 3) X(3, 3) X(1, 5)

namespace b2y {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a pipeline bug traps (kernel error) instead of hanging the GPU box.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) {  // ~2 s at 2 GHz
            __trap();
        }
    }
}

// shared-window (u32) address variants for the single-thread issue loops: no generic->shared conversion per call
__device__ __forceinline__ bool mbar_try_wait_s(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait_s(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait_s(bar, parity)) return;
    long long t0 = clock64();
    while (!mbar_try_wait_s(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) __trap();
    }
}
__device__ __forceinline__ void mbar_expect_tx_s(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// programmatic dependent launch: wait for the upstream grid's memory / let the downstream grid start its prologue
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// Host side: launch `kern` as a programmatic dependent of the previous kernel in the stream.  The grid may become
// resident while its predecessor drains, so the kernel MUST execute pdl_wait() before it touches anything the
// predecessor wrote (and should call pdl_launch_dependents() right after, so that at most one grid is ever parked
// behind a running one).  In a captured graph the edge becomes a programmatic dependency.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                              Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// one lane of a converged warp
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "elect.sync _|p, 0xffffffff;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(pred));
    return pred != 0;
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// multicast variant: the box lands at the same smem offset in every CTA of `mask` and signals each one's mbarrier
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                                      int c1, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask)
        : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// im2col-mode load of an NHWC tensor: coords (c, w, h, n) are the *base pixel*
// (already offset by the lower corner), (off_w, off_h) the filter tap.
__device__ __forceinline__ void tma_load_im2col_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c, int w,
                                                   int h, int n, uint16_t off_w, uint16_t off_h) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h),
        "r"(n), "h"(off_w), "h"(off_h)
        : "memory");
}

__device__ __forceinline__ void tma_load_2d_s(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d_multicast_s(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1,
                                                        uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "h"(mask)
        : "memory");
}
__device__ __forceinline__ void tma_load_im2col_4d_s(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c, int w, int h,
                                                     int n, uint16_t off_w, uint16_t off_h) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c), "r"(w), "r"(h), "r"(n), "h"(off_w), "h"(off_h)
        : "memory");
}

// TMA store of a smem box (written by generic stores + fence.proxy.async) to global; bulk-group completion
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(m)),
                 "r"(src), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_cta() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ uint32_t mapa_u32(uint32_t smem_addr, uint32_t cta_rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(cta_rank));
    return r;
}
// Arrive on an mbarrier of any CTA of the cluster (the stage-release of a multicast ring).  CTA-scope release, the
// default: the consumer's reads of the stage were wgmma operand reads that wgmma.wait_group has already retired, so no
// generic-proxy data is published through this arrive.  A .cluster-scope release compiles to a GPU-wide MEMBAR in
// front of every arrive, once per k-step per peer, which stalls the MMA warps.
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_bar_addr) {
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(cluster_bar_addr) : "memory");
}
// named barrier over `nthreads` threads (a multiple of 32); id 0 is __syncthreads()
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------- wgmma operands / accumulators
// Shared-memory matrix descriptor (wgmma), swizzled canonical layouts.
//   bits: [0,14) addr>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [62,64) swizzle: 1 = 128B, 2 = 64B, 3 = 32B
//   K-major: rows of `row_bytes` (= the swizzle span), 8-row groups SBO apart.  Tiles start 1024-byte aligned.
__host__ __device__ __forceinline__ uint64_t smem_desc_base(uint32_t lbo_bytes, uint32_t sbo_bytes,
                                                            uint32_t layout_type) {
    uint64_t d = 0;
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    d |= (uint64_t)(layout_type & 3) << 62;
    return d;
}
__device__ __forceinline__ uint64_t smem_desc_at(uint64_t base, uint32_t smem_addr) {
    return base | (uint64_t)((smem_addr >> 4) & 0x3FFF);
}
__host__ __device__ constexpr uint32_t swizzle_layout_type(int row_bytes) {
    return row_bytes == 128 ? 1u : (row_bytes == 64 ? 2u : (row_bytes == 32 ? 3u : 0u));
}

// fp32 accumulator staging tile [rows][N] in smem, 16-byte granules XOR-swizzled by (row & 7): conflict-free row reads
// (thread = row) and at most two-way conflicts on the fragment stores.  N >= 32.
template <int N>
__device__ __forceinline__ uint32_t stage_off(int row, int col) {   // byte offset of (row, col), col % 2 == 0
    return (uint32_t)(row * N * 4) + ((uint32_t)(((col >> 2) ^ (row & 7))) << 4) + (uint32_t)((col & 3) * 4);
}
// the wgmma accumulator fragment of this thread (64 x N block of a warpgroup, rows row0 .. row0 + 63) -> staging tile
template <int N, typename T>
__device__ __forceinline__ void frag_to_stage(const T (&d)[N / 2], uint8_t* stage, int row0, int tid_in_wg) {
    const int r = row0 + 16 * (tid_in_wg >> 5) + ((tid_in_wg & 31) >> 2);
    const int c = 2 * (tid_in_wg & 3);
#pragma unroll
    for (int i = 0; i < N / 8; ++i) {
        *reinterpret_cast<uint2*>(stage + stage_off<N>(r, 8 * i + c)) =
            make_uint2(reinterpret_cast<const uint32_t&>(d[4 * i]), reinterpret_cast<const uint32_t&>(d[4 * i + 1]));
        *reinterpret_cast<uint2*>(stage + stage_off<N>(r + 8, 8 * i + c)) =
            make_uint2(reinterpret_cast<const uint32_t&>(d[4 * i + 2]), reinterpret_cast<const uint32_t&>(d[4 * i + 3]));
    }
}
// 32 consecutive 32-bit accumulators of one row (columns c0 .. c0 + 31) from the staging tile
template <int N>
__device__ __forceinline__ void stage_row32(const uint8_t* stage, int row, int c0, uint32_t (&r)[32]) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const uint4 u = *reinterpret_cast<const uint4*>(stage + stage_off<N>(row, c0 + 4 * q));
        r[4 * q] = u.x;
        r[4 * q + 1] = u.y;
        r[4 * q + 2] = u.z;
        r[4 * q + 3] = u.w;
    }
}

// ---------------------------------------------------------------- activations (fp32)
__device__ __forceinline__ float softplus_f(float x) {
    // torch F.softplus(beta=1, threshold=20)  (reference utils/layers.py:148)
    return x > 20.f ? x : log1pf(expf(x));
}
// Mish (reference utils/layers.py:118-128, 146-148): tanh(softplus(x)) in closed form.  With e = exp(x):
//   tanh(log(1+e)) = ((1+e)^2 - 1) / ((1+e)^2 + 1) = n / (n + 2),  n = e (e + 2)
// one exponential and one division instead of exp + log1p + tanh; no cancellation for either sign of x (for x << 0 it
// tends to e like the original).  x is clamped at 20, where torch's softplus switches to the identity and tanh is 1
// in fp32 anyway.  Agreement with the literal formula: a few fp32 ulp.
__device__ __forceinline__ float mish_tanh_softplus(float x, float& e) {
    e = __expf(fminf(x, 20.f));
    const float n = e * (e + 2.f);
    return __fdividef(n, n + 2.f);
}
__device__ __forceinline__ float mish_f(float x) {
    float e;
    return x * mish_tanh_softplus(x, e);
}
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }

__device__ __forceinline__ float apply_act(float v, int act, float slope) {
    switch (act) {
        case B2Y_ACT_LEAKY: return v > 0.f ? v : v * slope;
        case B2Y_ACT_MISH: return mish_f(v);
        case B2Y_ACT_RELU: return fmaxf(v, 0.f);
        case B2Y_ACT_RELU6: return fminf(fmaxf(v, 0.f), 6.f);
        case B2Y_ACT_HSWISH: return v * (fminf(fmaxf(v + 3.f, 0.f), 6.f) / 6.f);
        case B2Y_ACT_SWISH: return v * sigmoid_f(v);
        default: return v;
    }
}
// d act(v) / dv
__device__ __forceinline__ float act_grad(float v, int act, float slope) {
    switch (act) {
        case B2Y_ACT_LEAKY: return v > 0.f ? 1.f : slope;
        case B2Y_ACT_MISH: {
            // reference utils/layers.py:123-128: fx + x * sigmoid(x) * (1 - fx^2), fx = tanh(softplus(x))
            // fx = n / (n + 2) and sigmoid(x) = e / (1 + e) share ONE reciprocal, 1 / ((n + 2)(1 + e)) (<= e^60, no
            // overflow): the backward BN passes are bound by the MUFU pipe (exp + reciprocals), this drops a third of it
            const float e = __expf(fminf(v, 20.f));
            const float n = e * (e + 2.f), d1 = n + 2.f, d2 = 1.f + e;
            const float r = __fdividef(1.f, d1 * d2);
            const float fx = n * d2 * r;
            const float sx = e * d1 * r;
            return fx + v * sx * (1.f - fx * fx);
        }
        case B2Y_ACT_RELU: return v > 0.f ? 1.f : 0.f;
        case B2Y_ACT_RELU6: return (v > 0.f && v < 6.f) ? 1.f : 0.f;
        case B2Y_ACT_HSWISH: {
            float r = fminf(fmaxf(v + 3.f, 0.f), 6.f) / 6.f;
            float dr = (v > -3.f && v < 3.f) ? (1.f / 6.f) : 0.f;
            return r + v * dr;
        }
        case B2Y_ACT_SWISH: {
            float sx = sigmoid_f(v);
            return sx * (1.f + v * (1.f - sx));
        }
        default: return 1.f;
    }
}

}  // namespace b2y

namespace b2y {
// 16-bit storage helpers so that gradient kernels can be instantiated for fp16 or bf16 tensors
template <typename T> struct Half8;
template <> struct Half8<__half> {
    __device__ static void unpack(const uint4& u, float (&f)[8]) {
        const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 t = __half22float2(h[j]);
            f[2 * j] = t.x;
            f[2 * j + 1] = t.y;
        }
    }
    __device__ static void load(const __half* p, float (&f)[8]) {
        const uint4 u = *reinterpret_cast<const uint4*>(p);
        const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 t = __half22float2(h[j]);
            f[2 * j] = t.x;
            f[2 * j + 1] = t.y;
        }
    }
    __device__ static void store(__half* p, const float (&f)[8]) {
        uint4 u;
        __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
        for (int j = 0; j < 4; ++j) h[j] = __floats2half2_rn(f[2 * j], f[2 * j + 1]);
        *reinterpret_cast<uint4*>(p) = u;
    }
    __device__ static float to_f(__half v) { return __half2float(v); }
    __device__ static __half from_f(float v) { return __float2half_rn(v); }
};
template <> struct Half8<__nv_bfloat16> {
    __device__ static void unpack(const uint4& u, float (&f)[8]) {
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 t = __bfloat1622float2(h[j]);
            f[2 * j] = t.x;
            f[2 * j + 1] = t.y;
        }
    }
    __device__ static void load(const __nv_bfloat16* p, float (&f)[8]) {
        const uint4 u = *reinterpret_cast<const uint4*>(p);
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 t = __bfloat1622float2(h[j]);
            f[2 * j] = t.x;
            f[2 * j + 1] = t.y;
        }
    }
    __device__ static void store(__nv_bfloat16* p, const float (&f)[8]) {
        uint4 u;
        __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
        for (int j = 0; j < 4; ++j) h[j] = __floats2bfloat162_rn(f[2 * j], f[2 * j + 1]);
        *reinterpret_cast<uint4*>(p) = u;
    }
    __device__ static float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
    __device__ static __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};
}  // namespace b2y

// host-side helpers ---------------------------------------------------------
// true the first time it is called for the current device with this mask (launch attributes such as
// MaxDynamicSharedMemorySize are per device; a process may drive several GPUs)
static inline bool b2y_first_use_on_device(unsigned long long& mask) {
    int dev = 0;
    cudaGetDevice(&dev);
    const unsigned long long bit = 1ull << (dev & 63);
    if (mask & bit) return false;
    mask |= bit;
    return true;
}

#define B2Y_CUDA_CHECK(expr)                       \
    do {                                           \
        cudaError_t _e = (expr);                   \
        if (_e != cudaSuccess) {                   \
            b2y_set_last_cuda_error((int)_e);      \
            return B2Y_ERR_CUDA;                   \
        }                                          \
    } while (0)

extern "C" void b2y_set_last_cuda_error(int e);

// Order-independent reductions: a kernel whose CTAs add partial sums into one fp32 result adds them into a double
// accumulator instead, and acc_finalize then adds the rounded total into the fp32 destination and clears the
// accumulator.  A double sum of fp32 terms is exact unless the terms span more than 29 binades, so in practice the result
// no longer depends on the order of the atomics: batch-statistics BatchNorm over fp16 activations magnifies last-bit
// differences step after step, and without this two runs of the same training diverge within a few steps, which would
// make the outputs of two builds impossible to compare.
//
// stream_acc(st, n) returns the zero-filled accumulator (>= n doubles) owned by the current device and stream `st`:
// launches on one stream are ordered and each finalizes (clears) what it used before the next one starts, and launches
// on different streams never share an accumulator.
double* stream_acc(cudaStream_t st, long long n);

template <int UNUSED = 0>
__global__ void acc_finalize_kernel(double* __restrict__ acc, float* __restrict__ dst, long long n) {
    b2y::pdl_wait();
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        dst[i] += (float)acc[i];
        acc[i] = 0.0;
    }
}
static inline int acc_finalize(double* acc, float* dst, long long n, cudaStream_t st) {
    long long grid = (n + 255) / 256;
    if (grid > 132 * 16) grid = 132 * 16;
    B2Y_CUDA_CHECK(b2y::launch_pdl(acc_finalize_kernel<0>, dim3((unsigned)grid), dim3(256), 0, st, acc, dst, n));
    return B2Y_OK;
}

// stream_ws(st, n) returns an fp32 workspace (>= n floats, contents undefined) owned by the current device and stream
// `st`, on the same terms as stream_acc: the weight gradient stores its split-K partial tiles there and reduces them in
// a fixed order (wgrad_tc.cu).
float* stream_ws(cudaStream_t st, long long n);

// Fixed-order per-channel reduction of the fp32 NHWC paths (QAT depthwise, BatchNorm, squeeze-excite): a CTA of 32
// channels x 8 pixel rows sums K values per (row, channel) over its chunk of the rows in double, the 8 rows are then added
// in order, and the chunk's total goes to part[((group * chunks + chunk) * K + k) * C + c].  chunk_sum_kernel adds the
// chunks in order.  No atomics, so two runs give the same bits.  grid = (ceil(C / 32), F32_CHUNKS, groups), block (32, 8).
// V is the type op writes its per-row values in (double where a value must not be rounded to fp32 first).
namespace b2y {
constexpr int F32_CHUNKS = 128;

template <int K, typename Op, typename V = float>
__device__ __forceinline__ void chunk_reduce(const Op& op, long long rows, int C, double* __restrict__ part) {
    __shared__ double red[K][8][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    const long long per = (rows + gridDim.y - 1) / gridDim.y;
    const long long r0 = (long long)blockIdx.y * per;
    const long long r1 = r0 + per < rows ? r0 + per : rows;
    double acc[K];
#pragma unroll
    for (int k = 0; k < K; ++k) acc[k] = 0.0;
    if (c < C) {
        for (long long r = r0 + threadIdx.y; r < r1; r += 8) {
            V v[K];
            op(blockIdx.z, r, c, v);
#pragma unroll
            for (int k = 0; k < K; ++k) acc[k] += (double)v[k];
        }
    }
#pragma unroll
    for (int k = 0; k < K; ++k) red[k][threadIdx.y][threadIdx.x] = acc[k];
    __syncthreads();
    if (threadIdx.y == 0 && c < C) {
#pragma unroll
        for (int k = 0; k < K; ++k) {
            double s = 0.0;
#pragma unroll
            for (int j = 0; j < 8; ++j) s += red[k][j][threadIdx.x];
            part[(((long long)blockIdx.z * gridDim.y + blockIdx.y) * K + k) * C + c] = s;
        }
    }
}

// out[g][i] = alpha * sum_{chunk} part[g][chunk][i]   (i < n = K * C), chunks added in order
template <int UNUSED = 0>
__global__ void chunk_sum_kernel(const double* __restrict__ part, float* __restrict__ out, long long n, int groups,
                                 float alpha) {
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n * groups;
         idx += (long long)gridDim.x * blockDim.x) {
        const long long g = idx / n, i = idx % n;
        double s = 0.0;
        for (int ch = 0; ch < F32_CHUNKS; ++ch) s += part[(g * F32_CHUNKS + ch) * n + i];
        out[idx] = (float)(s * alpha);
    }
}

inline dim3 chunk_grid(int c, int groups) { return dim3((unsigned)((c + 31) / 32), F32_CHUNKS, (unsigned)groups); }
inline double* chunk_ws(cudaStream_t st, long long groups, int K, int c) {
    return reinterpret_cast<double*>(stream_ws(st, 2LL * groups * F32_CHUNKS * K * c));
}
inline int grid_1d(long long n) {
    long long g = (n + 255) / 256;
    return (int)(g < 1 ? 1 : (g > 132 * 16 ? 132 * 16 : g));
}
}  // namespace b2y
