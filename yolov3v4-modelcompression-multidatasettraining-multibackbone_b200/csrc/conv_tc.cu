// Host side of the wgmma implicit-GEMM convolution: TMA tensor-map encoding, tile-shape dispatch,
// C-ABI entry points (include/b200yolo.h).
#include "conv_tc.cuh"

#include <cmath>
#include <mutex>

#include "b200yolo.h"

namespace b2y {

// ---- driver entry points (resolved lazily; the library does not link libcuda) -------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*PFN_encodeIm2col)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t,
                                     const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                     CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled g_encodeTiled = nullptr;
static PFN_encodeIm2col g_encodeIm2col = nullptr;
static int g_driver_version = 0;
static int g_num_sms = 0;
static std::once_flag g_once;

static void resolve_driver() {
    cudaDriverEntryPointQueryResult q;
    void* fn = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
        g_encodeTiled = reinterpret_cast<PFN_encodeTiled>(fn);
    fn = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
        g_encodeIm2col = reinterpret_cast<PFN_encodeIm2col>(fn);
    cudaDriverGetVersion(&g_driver_version);
    int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
}

static CUtensorMapSwizzle swizzle_enum(int kbytes) {
    return kbytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                         : (kbytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

// 2-D tiled map over a row-major [rows][cols] matrix with row pitch `pitch_elems`.
static CUtensorMapDataType tm_dtype(int esize, bool bf16) {
    if (esize == 1) return CU_TENSOR_MAP_DATA_TYPE_UINT8;
    if (esize == 4) return CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    return bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
}

static int make_map_2d(CUtensorMap* m, const void* base, int esize, long long rows, long long cols,
                       long long pitch_elems, int box_cols, int box_rows, int kbytes, bool bf16 = false) {
    if (!g_encodeTiled) return B2Y_ERR_DRIVER;
    cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t gstride[1] = {(cuuint64_t)(pitch_elems * esize)};
    cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = g_encodeTiled(m, tm_dtype(esize, bf16), 2,
                               const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                               swizzle_enum(kbytes), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? B2Y_OK : B2Y_ERR_DRIVER;
}

// im2col map over an NHWC activation tensor (dims C,W,H,N) for an RxS / stride / pad convolution.
static int make_map_im2col(CUtensorMap* m, const void* base, int esize, int N, int H, int W, int C,
                           long long pitch_elems, int lower_w, int lower_h, int upper_w, int upper_h, int stride,
                           int block_k, int kbytes, int pixels_per_column = 128, bool bf16 = false,
                           int stride_h = 0) {
    if (!g_encodeIm2col) return B2Y_ERR_DRIVER;
    cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t gstride[3] = {(cuuint64_t)(pitch_elems * esize), (cuuint64_t)(pitch_elems * esize * W),
                             (cuuint64_t)(pitch_elems * esize * W * (long long)H)};
    // bounding box of the *base pixel* (the tap with offset 0): for fprop lower = -pad, upper = pad - (filter-1)
    int lower[2] = {lower_w, lower_h};
    int upper[2] = {upper_w, upper_h};
    cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)(stride_h > 0 ? stride_h : stride), 1};
    CUresult r = g_encodeIm2col(m, tm_dtype(esize, bf16), 4,
                                const_cast<void*>(base), gdim, gstride, lower, upper, (cuuint32_t)block_k,
                                (cuuint32_t)pixels_per_column, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_enum(kbytes),
                                CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return B2Y_ERR_DRIVER;
    // Drivers <= 13.1 mis-encode im2col maps of tensors smaller than 128 KiB (same workaround as CUTLASS).
    if (g_driver_version <= 13010) {
        long long bytes = (long long)N * H * W * pitch_elems * esize;
        if (bytes < 131072) reinterpret_cast<uint64_t*>(m)[1] &= ~(1ull << 21);
    }
    return B2Y_OK;
}

// Adds the batch statistics accumulated in double (stream_acc: [0, CONV_STAT_MAX) sums, [CONV_STAT_MAX, ...) squares)
// into the caller's fp32 buffers and clears the accumulator; a programmatic dependent of the convolution.
__global__ void stats_finalize_kernel(double* __restrict__ acc, int C, float* __restrict__ sum, float* __restrict__ sqsum) {
    pdl_wait();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    sum[c] += (float)acc[c];
    sqsum[c] += (float)acc[CONV_STAT_MAX + c];
    acc[c] = 0.0;
    acc[CONV_STAT_MAX + c] = 0.0;
}

template <int BLOCK_N, int KBYTES, int KIND, int CLUSTER>
static int launch_cfg(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const ConvTcParams& p,
                      cudaStream_t st) {
    using Cfg = ConvTcCfg<BLOCK_N, KBYTES>;
    auto kern = conv_tc_kernel<BLOCK_N, KBYTES, KIND, CLUSTER>;
    static unsigned long long attr_set = 0;      // one bit per device: the attribute is per (function, device)
    if (b2y_first_use_on_device(attr_set)) {
        B2Y_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    }
    const int items = ((p.num_m_tiles + CLUSTER - 1) / CLUSTER) * p.num_n_tiles;
    const int max_clusters = g_num_sms / CLUSTER;
    const int clusters = items < max_clusters ? items : max_clusters;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(clusters * CLUSTER);
    cfg.blockDim = dim3(ConvTcEpi::THREADS);
    cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    int na = 0;
    if (CLUSTER > 1) {
        attr[na].id = cudaLaunchAttributeClusterDimension;
        attr[na].val.clusterDim.x = CLUSTER;
        attr[na].val.clusterDim.y = 1;
        attr[na].val.clusterDim.z = 1;
        ++na;
    }
    // the kernel's prologue (and its static weight loads) may start while the previous kernel drains; it executes
    // griddepcontrol.wait before touching activations
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
    cfg.attrs = attr;
    cfg.numAttrs = na;
    B2Y_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, tmA, tmB, tmC, p));
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

template <int KIND>
static int dispatch(int block_n, int kbytes, int cluster, const CUtensorMap& a, const CUtensorMap& b,
                    const CUtensorMap& c, const ConvTcParams& p, cudaStream_t st) {
#define B2Y_CASE(BN, KB) \
    if (block_n == BN && kbytes == KB && cluster == 1) return launch_cfg<BN, KB, KIND, 1>(a, b, c, p, st);
    B2Y_CASE(32, 32) B2Y_CASE(32, 64) B2Y_CASE(32, 128)
    B2Y_CASE(64, 32) B2Y_CASE(64, 64) B2Y_CASE(64, 128)
    B2Y_CASE(128, 32) B2Y_CASE(128, 64) B2Y_CASE(128, 128)
#undef B2Y_CASE
    // weight-multicast clusters exist for the wide, deep tiles only (KBYTES = 128)
    if (kbytes == 128 && block_n == 128 && cluster == 2) return launch_cfg<128, 128, KIND, 2>(a, b, c, p, st);
    return B2Y_ERR_UNSUPPORTED;
}

// cluster size for a launch: 2 when the tile shape supports multicast and there is more than one M tile per cluster to
// share the weights across
static int pick_cluster(int block_n, int kbytes, int num_m_tiles) {
    if (kbytes != 128 || block_n < 128) return 1;
    if (num_m_tiles < 4) return 1;
    return 2;
}

struct EpilogueArgs {
    const float* bias = nullptr;
    int act = 0;
    float slope = 0.1f;
    float acc_scale = 1.f;
    const void* res = nullptr;
    long long res_pitch = 0;
    void* out = nullptr;
    long long out_pitch = 0;
    int out_dtype = OUT_F16;
    float out_scale = 1.f;
    int out_fakequant = 0;
    float q_lo = -128.f, q_hi = 127.f;
    float* stat_sum = nullptr;
    float* stat_sqsum = nullptr;
    int res_bf16 = 0;
    const float* acc_scale_ptr = nullptr;
    // int8 graph: quantised shortcut folded into the epilogue (see ConvTcParams::qres)
    const void* qres = nullptr;
    long long qres_pitch = 0;
    float qs_a_in = 1.f, qs_x = 1.f, qs_a = 1.f, qs_sum = 1.f, qs_lo = -128.f, qs_hi = 127.f;
    int qs_clamp = 0;
};

// Generic implicit-GEMM launch description: A = NHWC activation-like tensor gathered tap by tap, B = [Nout][ntaps*C].
struct GemmConvSpec {
    int kind = CONV_KIND_F16;
    const void* a = nullptr;
    int N = 0, H = 0, W = 0, C = 0;
    long long a_pitch = 0;
    int MH = 0, MW = 0;          // base-pixel grid per image (GEMM rows = N*MH*MW)
    int stride = 1;              // TMA traversal stride (along W; along H too unless stride_h is set)
    int stride_h = 0;            // 0: same as stride
    int lower_w = 0, lower_h = 0, upper_w = 0, upper_h = 0;
    int ntaps = 1;
    unsigned char tap_ow[16] = {0}, tap_oh[16] = {0};
    bool pointwise = false;      // plain GEMM over [N*H*W][C] (2-D tiled TMA)
    bool a_bf16 = false, b_bf16 = false;   // 16-bit operand formats (wgmma: both the same)
    const void* w = nullptr;
    int Nout = 0;
    int out_identity = 1, out_OH = 0, out_OW = 0, out_ys = 1, out_xs = 1, out_y0 = 0, out_x0 = 0;
};

int gemm_conv_launch(const GemmConvSpec& g, const EpilogueArgs& e, cudaStream_t st) {
    std::call_once(g_once, resolve_driver);
    const int esize = g.kind == CONV_KIND_F16 ? 2 : 1;
    if (!g.a || !g.w || !e.out) return B2Y_ERR_INVALID;
    if (g.N <= 0 || g.C <= 0 || g.Nout <= 0 || g.ntaps < 1 || g.ntaps > 16) return B2Y_ERR_INVALID;
    const long long kb_total = (long long)g.C * esize;
    if (kb_total % 32 != 0) return B2Y_ERR_UNSUPPORTED;
    const int kbytes = kb_total % 128 == 0 ? 128 : (kb_total % 64 == 0 ? 64 : 32);
    if ((g.a_pitch * esize) % 16 != 0) return B2Y_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(g.a) & 15) || (reinterpret_cast<uintptr_t>(g.w) & 15)) return B2Y_ERR_INVALID;
    const long long M = (long long)g.N * g.MH * g.MW;
    if (M <= 0 || M > 0x7fffff00LL) return B2Y_ERR_UNSUPPORTED;
    if (g.kind == CONV_KIND_F16 && g.a_bf16 != g.b_bf16) return B2Y_ERR_UNSUPPORTED;
    // N tiles of at most 128 columns: a 128 x 128 fp32 accumulator is 64 registers per thread of the two consumer
    // warpgroups and 64 KB of epilogue staging, which leaves room for a 4-deep ring of 32 KB k-step stages
    const int block_n = g.Nout <= 32 ? 32 : (g.Nout <= 64 ? 64 : 128);
    const int block_k = kbytes / esize;

    ConvTcParams p{};
    p.M_total = (int)M;
    p.Cout = g.Nout;
    p.num_m_tiles = (int)((M + 127) / 128);
    p.num_n_tiles = (g.Nout + block_n - 1) / block_n;
    p.k_chunks = (int)(kb_total / kbytes);
    p.Cin = g.C;
    p.ntaps = g.ntaps;
    p.MH = g.MH;
    p.MW = g.MW;
    p.stride = g.stride;
    p.stride_h = g.stride_h > 0 ? g.stride_h : g.stride;
    p.lower_w = g.lower_w;
    p.lower_h = g.lower_h;
    for (int t = 0; t < 16; ++t) {
        if (g.tap_ow[t] > 15 || g.tap_oh[t] > 15) return B2Y_ERR_UNSUPPORTED;
        p.tap_ow[t] = g.tap_ow[t];
        p.tap_oh[t] = g.tap_oh[t];
        p.tap_w_packed |= (unsigned long long)g.tap_ow[t] << (4 * t);
        p.tap_h_packed |= (unsigned long long)g.tap_oh[t] << (4 * t);
    }
    p.out_identity = g.out_identity;
    p.out_OH = g.out_OH;
    p.out_OW = g.out_OW;
    p.out_ys = g.out_ys;
    p.out_xs = g.out_xs;
    p.out_y0 = g.out_y0;
    p.out_x0 = g.out_x0;
    p.bias = e.bias;
    p.act = e.act;
    p.slope = e.slope;
    p.acc_scale = e.acc_scale;
    p.acc_scale_ptr = e.acc_scale_ptr;
    p.ab_bf16 = g.a_bf16 ? 1 : 0;
    p.res_bf16 = e.res_bf16;
    p.res = reinterpret_cast<const __half*>(e.res);
    p.res_pitch = e.res_pitch;
    p.out = e.out;
    p.out_pitch = e.out_pitch;
    p.out_dtype = e.out_dtype;
    p.out_scale = e.out_scale;
    p.out_inv_scale = 1.f / e.out_scale;
    p.out_fakequant = e.out_fakequant;
    p.q_lo = e.q_lo;
    p.q_hi = e.q_hi;
    p.stat_acc = nullptr;
    if (e.stat_sum != nullptr) {
        if (e.stat_sqsum == nullptr || g.Nout > CONV_STAT_MAX) return B2Y_ERR_UNSUPPORTED;
        p.stat_acc = stream_acc(st, 2 * CONV_STAT_MAX);
        if (p.stat_acc == nullptr) return B2Y_ERR_CUDA;
    }
    {
        // the short epilogue: fp16/bf16 output (fp32 only through TMA), everything 16-byte addressable; a clipped last
        // N tile (Cout = 255 heads) needs the TMA store's clipping and has no residual
        auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
        const bool act_ok = e.act == B2Y_ACT_LINEAR || e.act == B2Y_ACT_MISH ||
                            (e.act == B2Y_ACT_LEAKY && e.slope >= 0.f && e.slope <= 1.f);
        const bool out16 = e.out_dtype == OUT_F16 || e.out_dtype == OUT_BF16;
        const bool out32 = e.out_dtype == OUT_F32;
        // the TMA store needs the identity row mapping; the strided dgrad scatters rows through the register stores
        const bool tma_ok = g.out_identity;
        const bool full = g.Nout % block_n == 0;
        // a clipped TMA store still writes whole 16-byte pieces of a row (measured on H100: a 255-wide fp32 output also
        // wrote column 255), so it may clip the last N tile only where the valid width ends on such a piece
        const int out_esize = out32 ? 4 : (e.out_dtype == OUT_I8 ? 1 : 2);
        const bool clip_ok = tma_ok && ((long long)g.Nout * out_esize) % 16 == 0;
        // batch statistics ride on the short path when it stores through TMA and nothing is added to the accumulators
        const bool stats_ok = e.stat_sum == nullptr ||
                              (out16 && tma_ok && e.bias == nullptr && e.res == nullptr);
        p.epi_fast = g.kind == CONV_KIND_F16 && (out16 || (out32 && tma_ok)) && !e.out_fakequant &&
                     stats_ok && act_ok && al16(e.out) && e.out_pitch % (out16 ? 8 : 4) == 0 &&
                     (e.bias == nullptr || al16(e.bias)) && (e.res == nullptr || (al16(e.res) && e.res_pitch % 8 == 0)) &&
                     (full || (clip_ok && e.res == nullptr));
        // int8 graph: int8 codes out, no residual, whole N tiles, and a power-of-two accumulator scale so that
        // fma(acc, s, bias) equals the general path's (acc * s) + bias bit for bit
        int ex = 0;
        const bool pow2 = e.acc_scale > 0.f && frexpf(e.acc_scale, &ex) == 0.5f && e.acc_scale_ptr == nullptr;
        if (g.kind == CONV_KIND_I8 && e.out_dtype == OUT_I8 && !e.out_fakequant && e.stat_sum == nullptr &&
            (e.act == B2Y_ACT_LINEAR || (e.act == B2Y_ACT_LEAKY && e.slope >= 0.f && e.slope <= 1.f)) && pow2 && full &&
            e.res == nullptr && al16(e.out) && e.out_pitch % 16 == 0 && (e.bias == nullptr || al16(e.bias)) &&
            e.q_lo >= -128.f && e.q_hi <= 127.f && e.q_lo == floorf(e.q_lo) && e.q_hi == floorf(e.q_hi))
            p.epi_fast = 1;
        // fake-quantised / linear fp32 rows of the int8 graph (the YOLO heads): through the TMA store where it can clip
        if (g.kind == CONV_KIND_I8 && out32 && tma_ok && (full || clip_ok) && e.stat_sum == nullptr &&
            e.act == B2Y_ACT_LINEAR && pow2 && e.res == nullptr && al16(e.out) && e.out_pitch % 4 == 0 && (e.bias == nullptr || al16(e.bias)) &&
            (!e.out_fakequant || (e.q_lo >= -4194304.f && e.q_hi <= 4194303.f && e.q_lo == floorf(e.q_lo) &&
                                  e.q_hi == floorf(e.q_hi))))
            p.epi_fast = 1;
        if (e.qres != nullptr) {
            auto p2 = [](float v) { int x = 0; return v > 0.f && frexpf(v, &x) == 0.5f; };
            if (!p.epi_fast || e.out_dtype != OUT_I8 || !al16(e.qres) || e.qres_pitch % 16 != 0 || !p2(e.out_scale) ||
                !p2(e.qs_a_in) || !p2(e.qs_x) || !p2(e.qs_a) || !p2(e.qs_sum))
                return B2Y_ERR_UNSUPPORTED;     // the caller runs the stand-alone shortcut kernel instead
            p.qres = reinterpret_cast<const int8_t*>(e.qres);
            p.qres_pitch = e.qres_pitch;
            p.qs_rx = 1.f / e.qs_x;
            p.qs_x = e.qs_x;
            p.qs_a_in = e.qs_a_in;
            p.qs_ra = 1.f / e.qs_a;
            p.qs_a = e.qs_a;
            p.qs_rsum = 1.f / e.qs_sum;
            p.qs_lo = e.qs_lo;
            p.qs_hi = e.qs_hi;
            p.qs_clamp = e.qs_clamp;
            p.qs_cx = e.out_scale / e.qs_sum;
            p.qs_ca = e.qs_a_in / e.qs_sum;
            p.qs_simple = !e.qs_clamp && e.out_scale >= e.qs_x && e.qs_a_in >= e.qs_a && p.qs_cx <= 4096.f && p.qs_ca <= 4096.f &&
                          p.qs_cx >= 1.f / 4096.f && p.qs_ca >= 1.f / 4096.f && e.qs_lo >= -128.f && e.qs_hi <= 127.f;
        }
    }

    CUtensorMap tmA, tmB;
    int rc;
    if (g.pointwise) {
        p.a_mode = A_MODE_TILED2D;
        rc = make_map_2d(&tmA, g.a, esize, M, g.C, g.a_pitch, block_k, 128, kbytes, g.a_bf16);
    } else {
        p.a_mode = A_MODE_IM2COL;
        rc = make_map_im2col(&tmA, g.a, esize, g.N, g.H, g.W, g.C, g.a_pitch, g.lower_w, g.lower_h, g.upper_w,
                             g.upper_h, g.stride, block_k, kbytes, 128, g.a_bf16, p.stride_h);
    }
    if (rc != B2Y_OK) return rc;
    const long long Ktot = (long long)g.ntaps * g.C;
    const int cluster = pick_cluster(block_n, kbytes, p.num_m_tiles);
    rc = make_map_2d(&tmB, g.w, esize, g.Nout, Ktot, Ktot, block_k, block_n / cluster, kbytes, g.b_bf16);
    if (rc != B2Y_OK) return rc;

    {
        // smem ring depth; weight-stationary mode when the whole weight panel of a single N tile fits beside >= 6 A stages
        const long long max_smem = conv_max_stage_smem(block_n);
        const long long a_bytes = 128LL * kbytes, b_bytes = (long long)block_n * kbytes;
        const long long res_bytes = (long long)p.ntaps * p.k_chunks * b_bytes;
        p.b_resident = 0;
        long long ns = max_smem / (a_bytes + b_bytes);
        if (cluster == 1 && p.num_n_tiles == 1 && p.num_m_tiles > g_num_sms && res_bytes + 6 * a_bytes <= max_smem) {
            p.b_resident = 1;
            ns = (max_smem - res_bytes) / a_bytes;
        }
        p.num_stages = (int)(ns > 32 ? 32 : ns);
    }
    // output map for the TMA-store epilogue (16-bit outputs on the short path with identity row mapping)
    CUtensorMap tmC = tmB;
    p.epi_tma = 0;
    if (p.epi_fast && p.out_identity) {
        const bool o32 = e.out_dtype == OUT_F32, o8 = e.out_dtype == OUT_I8;
        rc = make_map_2d(&tmC, e.out, o32 ? 4 : (o8 ? 1 : 2), M, g.Nout, e.out_pitch, 32, 32, o32 ? 128 : (o8 ? 32 : 64),
                         e.out_dtype == OUT_BF16);
        if (rc != B2Y_OK) return rc;
        p.epi_tma = 1;
    }
    rc = g.kind == CONV_KIND_F16 ? dispatch<CONV_KIND_F16>(block_n, kbytes, cluster, tmA, tmB, tmC, p, st)
                                 : dispatch<CONV_KIND_I8>(block_n, kbytes, cluster, tmA, tmB, tmC, p, st);
    if (rc != B2Y_OK || p.stat_acc == nullptr) return rc;
    B2Y_CUDA_CHECK(launch_pdl(stats_finalize_kernel, dim3((g.Nout + 255) / 256), dim3(256), 0, st, p.stat_acc, g.Nout,
                              e.stat_sum, e.stat_sqsum));
    return B2Y_OK;
}

// Forward convolution: x NHWC (fp16 or int8), w [Cout][R][S][Cin].
int conv_tc_launch(int kind, const b2y_conv_desc* d, const void* x, const void* w, const EpilogueArgs& e,
                   cudaStream_t st) {
    if (!d) return B2Y_ERR_INVALID;
    if (d->batch <= 0 || d->in_c <= 0 || d->out_c <= 0 || d->ksize <= 0 || d->stride <= 0) return B2Y_ERR_INVALID;
    if (d->ksize * d->ksize > 16) return B2Y_ERR_UNSUPPORTED;
    const int Ho = (d->in_h + 2 * d->pad - d->ksize) / d->stride + 1;
    const int Wo = (d->in_w + 2 * d->pad - d->ksize) / d->stride + 1;
    if (Ho != d->out_h || Wo != d->out_w) return B2Y_ERR_INVALID;
    GemmConvSpec g;
    g.kind = kind;
    g.a = x;
    g.w = w;
    g.Nout = d->out_c;
    if (d->w_layout == B2Y_WLAYOUT_S2_PAIRS) {
        // pixel-pair view of a narrow stride-2 3x3 layer (include/b200yolo.h): 3 x 2 window, stride 2 x 1, pad top/left 1
        if (d->ksize != 3 || d->stride != 2 || d->pad != 1 || (d->in_w & 1) || d->in_pitch != d->in_c ||
            (d->in_c * (kind == CONV_KIND_F16 ? 2 : 1)) % 32 != 0)
            return B2Y_ERR_UNSUPPORTED;
        g.N = d->batch;
        g.H = d->in_h;
        g.W = d->in_w / 2;
        g.C = 2 * d->in_c;
        g.a_pitch = 2 * d->in_pitch;
        g.MH = Ho;
        g.MW = Wo;
        g.stride = 1;
        g.stride_h = 2;
        g.lower_w = g.lower_h = -1;
        g.upper_w = -1;              // pad_right 0 - (kw - 1)
        g.upper_h = -1;              // pad_bottom 1 - (kh - 1)
        g.ntaps = 6;
        for (int r = 0; r < 3; ++r)
            for (int s = 0; s < 2; ++s) {
                g.tap_oh[r * 2 + s] = (unsigned char)r;
                g.tap_ow[r * 2 + s] = (unsigned char)s;
            }
        return gemm_conv_launch(g, e, st);
    }
    if (d->w_layout != B2Y_WLAYOUT_DENSE) return B2Y_ERR_INVALID;
    g.N = d->batch;
    g.H = d->in_h;
    g.W = d->in_w;
    g.C = d->in_c;
    g.a_pitch = d->in_pitch;
    g.MH = Ho;
    g.MW = Wo;
    g.stride = d->stride;
    g.lower_w = g.lower_h = -d->pad;
    g.upper_w = g.upper_h = d->pad - (d->ksize - 1);
    g.ntaps = d->ksize * d->ksize;
    for (int r = 0; r < d->ksize; ++r)
        for (int s = 0; s < d->ksize; ++s) {
            g.tap_oh[r * d->ksize + s] = (unsigned char)r;
            g.tap_ow[r * d->ksize + s] = (unsigned char)s;
        }
    g.pointwise = (d->ksize == 1 && d->stride == 1 && d->pad == 0);
    g.w = w;
    g.Nout = d->out_c;
    return gemm_conv_launch(g, e, st);
}

// ---- data gradient -------------------------------------------------------------------------------------------
// dx[n, yi, xi, ci] = sum_{r,s} dy[n, (yi+pad-r)/stride, (xi+pad-s)/stride, co] * W[co][ci][r][s]
// decomposed by output phase (yi mod stride, xi mod stride): each phase is a stride-1 implicit GEMM over dy with
// the subset of taps whose parity matches, written to the strided dx positions of that phase.
struct DgradPhase {
    int py, px, nh, nw;       // taps per dimension
    int r[4], dr[4], s[4], ds[4];
    int min_dr, min_ds;
    int MH, MW;
    long long w_offset;       // element offset of this phase's [Cin][ntaps][Cout] slab in the packed buffer
};

static int enumerate_dgrad_phases(const b2y_conv_desc* d, DgradPhase* ph) {
    int n = 0;
    long long off = 0;
    const int k = d->ksize, s = d->stride, pad = d->pad;
    if (k > 4) return -1;
    for (int py = 0; py < s; ++py)
        for (int px = 0; px < s; ++px) {
            DgradPhase& P = ph[n];
            P.py = py;
            P.px = px;
            P.nh = P.nw = 0;
            P.min_dr = P.min_ds = 1 << 20;
            for (int r = 0; r < k; ++r) {
                const int t = py + pad - r;
                if (t % s == 0) {
                    P.r[P.nh] = r;
                    P.dr[P.nh] = t / s;
                    if (t / s < P.min_dr) P.min_dr = t / s;
                    P.nh++;
                }
            }
            for (int c = 0; c < k; ++c) {
                const int t = px + pad - c;
                if (t % s == 0) {
                    P.s[P.nw] = c;
                    P.ds[P.nw] = t / s;
                    if (t / s < P.min_ds) P.min_ds = t / s;
                    P.nw++;
                }
            }
            P.MH = (d->in_h - py + s - 1) / s;
            P.MW = (d->in_w - px + s - 1) / s;
            P.w_offset = off;
            off += (long long)d->in_c * P.nh * P.nw * d->out_c;
            n++;
        }
    return n;
}

}  // namespace b2y

using namespace b2y;

// pack W (OIHW fp32) into the per-phase dgrad layout [phase][Cin][tap][Cout] fp16
template <typename T>
__global__ void pack_dgrad_kernel(const float* __restrict__ w, T* __restrict__ out, int O, int I, int k, int nh,
                                  int nw, int r0, int r1, int r2, int r3, int s0, int s1, int s2, int s3) {
    const int rr[4] = {r0, r1, r2, r3}, ss[4] = {s0, s1, s2, s3};
    const int ntaps = nh * nw;
    const long long total = (long long)I * ntaps * O;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int co = (int)(idx % O);
        long long t = idx / O;
        const int tap = (int)(t % ntaps);
        const int ci = (int)(t / ntaps);
        const int r = rr[tap / nw], s = ss[tap % nw];
        out[idx] = Half8<T>::from_f(w[(((long long)co * I + ci) * k + r) * k + s]);
    }
}

extern "C" int b2y_pack_dgrad_weights(const b2y_conv_desc* d, const float* w_oihw, void* w_packed_t, int grad_dtype,
                                      void* stream) {
    if (!d || !w_oihw || !w_packed_t) return B2Y_ERR_INVALID;
    DgradPhase ph[16];
    if (d->stride > 4) return B2Y_ERR_UNSUPPORTED;
    const int n = enumerate_dgrad_phases(d, ph);
    if (n < 0) return B2Y_ERR_UNSUPPORTED;
    for (int i = 0; i < n; ++i) {
        const DgradPhase& P = ph[i];
        if (P.nh * P.nw == 0) continue;
        const long long total = (long long)d->in_c * P.nh * P.nw * d->out_c;
        int grid = (int)((total + 255) / 256);
        if (grid > 132 * 16) grid = 132 * 16;
        if (grad_dtype == B2Y_DT_BF16)
            pack_dgrad_kernel<__nv_bfloat16><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
                w_oihw, reinterpret_cast<__nv_bfloat16*>(w_packed_t) + P.w_offset, d->out_c, d->in_c, d->ksize, P.nh,
                P.nw, P.r[0], P.r[1], P.r[2], P.r[3], P.s[0], P.s[1], P.s[2], P.s[3]);
        else
            pack_dgrad_kernel<__half><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
                w_oihw, reinterpret_cast<__half*>(w_packed_t) + P.w_offset, d->out_c, d->in_c, d->ksize, P.nh, P.nw,
                P.r[0], P.r[1], P.r[2], P.r[3], P.s[0], P.s[1], P.s[2], P.s[3]);
    }
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_conv2d_bwd_data(const b2y_conv_desc* d, const void* dy, const void* w_packed_t, void* dx,
                                   int accumulate, int operand_dtype, int out_dtype, const float* inv_scale_ptr,
                                   void* stream) {
    const bool gbf = operand_dtype == B2Y_DT_BF16;     // dY and the packed weights (must match: wgmma takes one
                                                       // 16-bit format for both operands)
    const bool obf = out_dtype == B2Y_DT_BF16;         // dX (and the accumulate source)
    if (!d || !dy || !w_packed_t || !dx) return B2Y_ERR_INVALID;
    if (d->stride > 4) return B2Y_ERR_UNSUPPORTED;
    DgradPhase ph[16];
    const int n = enumerate_dgrad_phases(d, ph);
    if (n < 0) return B2Y_ERR_UNSUPPORTED;
    for (int i = 0; i < n; ++i) {
        const DgradPhase& P = ph[i];
        if (P.MH <= 0 || P.MW <= 0) continue;
        if (P.nh * P.nw == 0) {
            if (accumulate) continue;
            return B2Y_ERR_UNSUPPORTED;  // (kernel smaller than the stride: untouched phase would need a zero fill)
        }
        GemmConvSpec g;
        g.kind = CONV_KIND_F16;
        g.a_bf16 = g.b_bf16 = gbf;
        g.a = dy;
        g.N = d->batch;
        g.H = d->out_h;
        g.W = d->out_w;
        g.C = d->out_c;
        g.a_pitch = d->out_pitch;
        g.MH = P.MH;
        g.MW = P.MW;
        g.stride = 1;
        g.lower_w = P.min_ds;
        g.lower_h = P.min_dr;
        g.upper_w = P.min_ds + P.MW - d->out_w;
        g.upper_h = P.min_dr + P.MH - d->out_h;
        g.ntaps = P.nh * P.nw;
        for (int a = 0; a < P.nh; ++a)
            for (int b = 0; b < P.nw; ++b) {
                g.tap_oh[a * P.nw + b] = (unsigned char)(P.dr[a] - P.min_dr);
                g.tap_ow[a * P.nw + b] = (unsigned char)(P.ds[b] - P.min_ds);
            }
        g.pointwise = (d->ksize == 1 && d->stride == 1 && d->pad == 0);
        g.w = reinterpret_cast<const __half*>(w_packed_t) + P.w_offset;
        g.Nout = d->in_c;
        g.out_identity = (d->stride == 1) ? 1 : 0;
        g.out_OH = d->in_h;
        g.out_OW = d->in_w;
        g.out_ys = g.out_xs = d->stride;
        g.out_y0 = P.py;
        g.out_x0 = P.px;
        EpilogueArgs e;
        e.out = dx;
        e.out_pitch = d->in_pitch;
        e.out_dtype = obf ? OUT_BF16 : OUT_F16;
        e.acc_scale_ptr = inv_scale_ptr;
        if (accumulate) {
            e.res = dx;
            e.res_pitch = d->in_pitch;
            e.res_bf16 = obf ? 1 : 0;
        }
        int rc = gemm_conv_launch(g, e, static_cast<cudaStream_t>(stream));
        if (rc != B2Y_OK) return rc;
    }
    return B2Y_OK;
}




// ---- tensor-core stem ------------------------------------------------------------------------------------------
// The first layer (NCHW fp32 image, B2Y_STEM_IM2COL_SHAPES, e.g. 3x3 on RGB = 27 taps): the whole receptive field of
// one output pixel fits one 64-byte GEMM row, so the pack writes the im2col matrix itself,
//   packed[n][yo][xo][(kh*K + kw)*Cin + c] = x[n][c][yo*s + kh - pad][xo*s + kw - pad]   (32 columns, zero padded)
// and the conv is ONE k-step of a plain [M][32] x [32][Cout] GEMM on the wgmma kernel.
template <int CIN, int K>
__global__ void stem_fullpack_kernel(const float* __restrict__ x, __half* __restrict__ out, int B, int H, int W,
                                     int Ho, int Wo, int stride, int pad) {
    const long long total = (long long)B * Ho * Wo;
    const long long plane = (long long)H * W;
    for (long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x; pix < total;
         pix += (long long)gridDim.x * blockDim.x) {
        const int xo = (int)(pix % Wo);
        const long long t = pix / Wo;
        const int yo = (int)(t % Ho);
        const long long n = t / Ho;
        const float* xb = x + n * CIN * plane;
        const int y0 = yo * stride - pad, x0 = xo * stride - pad;
        float v[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = 0.f;
#pragma unroll
        for (int kh = 0; kh < K; ++kh) {
            const int yi = y0 + kh;
            if (yi < 0 || yi >= H) continue;
#pragma unroll
            for (int kw = 0; kw < K; ++kw) {
                const int xi = x0 + kw;
                if (xi >= 0 && xi < W) {
#pragma unroll
                    for (int c = 0; c < CIN; ++c) v[(kh * K + kw) * CIN + c] = __ldg(xb + c * plane + (long long)yi * W + xi);
                }
            }
        }
        uint4 o[4];
        __half2* oh = reinterpret_cast<__half2*>(o);
#pragma unroll
        for (int j = 0; j < 16; ++j) oh[j] = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
        uint4* op = reinterpret_cast<uint4*>(out + pix * 32);
#pragma unroll
        for (int q = 0; q < 4; ++q) op[q] = o[q];
    }
}

// w (OIHW fp32, BN folded) -> [O][32] fp16 with inner index (kh*k + kw)*Cin + c
__global__ void stem_fullpack_weights_kernel(const float* __restrict__ w, __half* __restrict__ out, int O, int Cin,
                                             int k) {
    const int total = O * 32;
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
        const int j = idx % 32;
        const int o = idx / 32;
        float v = 0.f;
        if (j < k * k * Cin) {
            const int c = j % Cin, kw = (j / Cin) % k, kh = j / (Cin * k);
            v = w[(((long long)o * Cin + c) * k + kh) * k + kw];
        }
        out[idx] = __float2half_rn(v);
    }
}

static inline bool stem_im2col_shape(int in_c, int ksize) {
#define B2Y_STEM_IS(CI, KK) if (in_c == CI && ksize == KK) return true;
    B2Y_STEM_IM2COL_SHAPES(B2Y_STEM_IS)
#undef B2Y_STEM_IS
    return false;
}

extern "C" size_t b2y_stem_workspace_bytes(const b2y_conv_desc* d) {
    if (!d || !stem_im2col_shape(d->in_c, d->ksize)) return 0;
    return (size_t)d->batch * d->out_h * d->out_w * 32 * sizeof(__half);
}

extern "C" int b2y_pack_stem_weights(const float* w_oihw_folded, int out_c, int in_c, int ksize, void* w_stem,
                                     void* stream) {
    if (!w_oihw_folded || !w_stem) return B2Y_ERR_INVALID;
    if (!stem_im2col_shape(in_c, ksize)) return B2Y_ERR_UNSUPPORTED;
    stem_fullpack_weights_kernel<<<(out_c * 32 + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        w_oihw_folded, reinterpret_cast<__half*>(w_stem), out_c, in_c, ksize);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_stem_conv_fwd_tc(const b2y_conv_desc* d, const float* x_nchw, const void* w_stem, const float* bias,
                                    void* workspace, void* y, float* stat_sum, float* stat_sqsum, void* stream) {
    if (!d || !x_nchw || !w_stem || !workspace || !y) return B2Y_ERR_INVALID;
    const int Ho = (d->in_h + 2 * d->pad - d->ksize) / d->stride + 1;
    const int Wo = (d->in_w + 2 * d->pad - d->ksize) / d->stride + 1;
    if (Ho != d->out_h || Wo != d->out_w) return B2Y_ERR_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long opix = (long long)d->batch * Ho * Wo;
    int fgrid = (int)((opix + 127) / 128);
    if (fgrid > 132 * 64) fgrid = 132 * 64;
    __half* fws = reinterpret_cast<__half*>(workspace);
#define B2Y_STEM_FULL(CI, KK)                                                                                       \
    if (d->in_c == CI && d->ksize == KK) {                                                                          \
        stem_fullpack_kernel<CI, KK><<<fgrid, 128, 0, st>>>(x_nchw, fws, d->batch, d->in_h, d->in_w, Ho, Wo,        \
                                                            d->stride, d->pad);                                     \
    } else
    B2Y_STEM_IM2COL_SHAPES(B2Y_STEM_FULL) { return B2Y_ERR_UNSUPPORTED; }
#undef B2Y_STEM_FULL
    B2Y_CUDA_CHECK(cudaGetLastError());
    GemmConvSpec g;
    g.kind = CONV_KIND_F16;
    g.a = workspace;
    g.N = d->batch;
    g.H = Ho;
    g.W = Wo;
    g.C = 32;
    g.a_pitch = 32;
    g.MH = Ho;
    g.MW = Wo;
    g.pointwise = true;
    g.ntaps = 1;
    g.w = w_stem;
    g.Nout = d->out_c;
    EpilogueArgs e;
    e.bias = bias;
    e.act = d->act;
    e.slope = d->slope;
    e.out = y;
    e.out_pitch = d->out_pitch;
    e.out_dtype = OUT_F16;
    e.stat_sum = stat_sum;
    e.stat_sqsum = stat_sqsum;
    return gemm_conv_launch(g, e, st);
}

extern "C" int b2y_conv2d_fwd(const b2y_conv_desc* d, const void* x, const void* w_packed, const float* bias,
                              const void* residual, void* y, void* stream) {
    if (!d) return B2Y_ERR_INVALID;
    EpilogueArgs e;
    e.bias = bias;
    e.act = d->act;
    e.slope = d->slope;
    e.res = residual;
    e.res_pitch = d->res_pitch;
    e.out = y;
    e.out_pitch = d->out_pitch;
    e.out_dtype = d->out_dtype == B2Y_OUT_F32 ? OUT_F32 : OUT_F16;
    return conv_tc_launch(CONV_KIND_F16, d, x, w_packed, e, static_cast<cudaStream_t>(stream));
}

extern "C" int b2y_conv2d_fwd_stats(const b2y_conv_desc* d, const void* x, const void* w_packed, const float* bias,
                                    void* y, float* stat_sum, float* stat_sqsum, void* stream) {
    if (!d || !stat_sum || !stat_sqsum) return B2Y_ERR_INVALID;
    EpilogueArgs e;
    e.bias = bias;
    e.act = B2Y_ACT_LINEAR;
    e.out = y;
    e.out_pitch = d->out_pitch;
    e.out_dtype = d->out_dtype == B2Y_OUT_F32 ? OUT_F32 : OUT_F16;
    e.stat_sum = stat_sum;
    e.stat_sqsum = stat_sqsum;
    return conv_tc_launch(CONV_KIND_F16, d, x, w_packed, e, static_cast<cudaStream_t>(stream));
}

extern "C" int b2y_qconv2d_fwd(const b2y_qconv_desc* d, const void* x_i8, const void* w_i8, const float* bias,
                               void* y, void* stream) {
    if (!d) return B2Y_ERR_INVALID;
    EpilogueArgs e;
    e.bias = bias;
    e.act = d->conv.act;
    e.slope = d->conv.slope;
    e.acc_scale = d->acc_scale;
    e.out = y;
    e.out_pitch = d->conv.out_pitch;
    e.out_scale = d->out_scale;
    e.q_lo = d->q_lo;
    e.q_hi = d->q_hi;
    if (d->out_kind == B2Y_OUT_I8) {
        e.out_dtype = OUT_I8;
    } else {
        e.out_dtype = d->out_kind == B2Y_OUT_F32 ? OUT_F32 : OUT_F16;
        e.out_fakequant = d->requant ? 1 : 0;
    }
    return conv_tc_launch(CONV_KIND_I8, &d->conv, x_i8, w_i8, e, static_cast<cudaStream_t>(stream));
}

extern "C" int b2y_qconv2d_shortcut_fwd(const b2y_qconv_desc* d, const void* x_i8, const void* w_i8, const float* bias,
                                        const void* a_i8, long long a_pitch, float sa_in, float scale_x, float scale_a,
                                        float scale_sum, float sum_lo, float sum_hi, void* y, void* stream) {
    if (!d || !a_i8 || d->out_kind != B2Y_OUT_I8) return B2Y_ERR_INVALID;
    EpilogueArgs e;
    e.bias = bias;
    e.act = d->conv.act;
    e.slope = d->conv.slope;
    e.acc_scale = d->acc_scale;
    e.out = y;
    e.out_pitch = d->conv.out_pitch;
    e.out_scale = d->out_scale;
    e.q_lo = d->q_lo;
    e.q_hi = d->q_hi;
    e.out_dtype = OUT_I8;
    e.qres = a_i8;
    e.qres_pitch = a_pitch;
    e.qs_a_in = sa_in;
    e.qs_x = scale_x;
    e.qs_a = scale_a;
    e.qs_sum = scale_sum;
    e.qs_lo = sum_lo;
    e.qs_hi = sum_hi;
    e.qs_clamp = d->clamp_addends ? 1 : 0;
    return conv_tc_launch(CONV_KIND_I8, &d->conv, x_i8, w_i8, e, static_cast<cudaStream_t>(stream));
}
