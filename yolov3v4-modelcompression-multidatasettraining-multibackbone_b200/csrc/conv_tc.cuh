// wgmma implicit-GEMM convolution, sm_90a.
//
//   D[M = B*Ho*Wo pixels][N = Cout] = sum_{tap (r,s)} sum_{c} A_tap[M][c] * W[N][(r,s,c)]
//
// * A (activations, NHWC) is never im2col'ed in memory: the TMA unit gathers each
//   (tap, 64-channel) slab straight from the NHWC tensor in im2col mode (zero fill for the
//   padding halo, traversal stride = conv stride) into a 128B-swizzled K-major smem tile.
// * B (weights, [Cout][R][S][Cin]) comes in through a tiled 2-D TMA map.
// * Two consumer warpgroups issue wgmma.mma_async (M=64 rows each, N=BLOCK_N, K=32 bytes) with the fp32/int32
//   accumulator in registers, then stage it through shared memory for the row-per-thread epilogue.
// * Persistent grid (<= #SMs CTAs), warp-specialised: warp0 = TMA producer (runs up to num_stages k-steps ahead,
//   across tile boundaries), warps 4-11 = MMA + epilogue (bias/act/residual/statistics -> global).
#pragma once
#include <type_traits>

#include "common.cuh"

namespace b2y {

enum { CONV_KIND_F16 = 0, CONV_KIND_I8 = 1 };
enum { A_MODE_IM2COL = 0, A_MODE_TILED2D = 1 };
enum { OUT_F16 = 0, OUT_F32 = 1, OUT_I8 = 2, OUT_BF16 = 3 };
constexpr int CONV_STAT_MAX = 4096;   // channels of a convolution that accumulates batch statistics

struct ConvTcParams {
    int M_total;      // B*Ho*Wo
    int Cout;         // valid output channels
    int num_m_tiles;  // ceil(M_total/128)
    int num_n_tiles;  // ceil(Cout/BLOCK_N)
    int k_chunks;     // Cin*esize / KBYTES
    int Cin;          // elements per tap (GEMM K per tap)
    int ntaps;        // filter taps visited (9 for 3x3; a subset for the stride-2 data-gradient phases)
    int MH, MW;       // GEMM row space = batch x MH x MW "base pixels"
    int stride;       // TMA traversal stride along W (conv stride for fprop, 1 for dgrad)
    int stride_h;     // ... along H (differs from `stride` only for the pixel-pair view of narrow stride-2 layers)
    int lower_w, lower_h;     // coordinate of base pixel (0,0): base = q*stride + lower
    unsigned char tap_ow[16]; // per-tap im2col offsets (>= 0)
    unsigned char tap_oh[16];
    unsigned long long tap_w_packed, tap_h_packed;   // the same offsets, 4 bits per tap (what the producer reads)
    int a_mode;
    // row -> output pixel mapping: pixel(n,p,q) = ((n*out_OH + p*out_ys + out_y0)*out_OW + q*out_xs + out_x0)
    int out_identity;         // 1: output pixel index == GEMM row index
    int out_OH, out_OW, out_ys, out_xs, out_y0, out_x0;
    // epilogue
    const float* bias;  // [Cout] or null
    int act;
    float slope;
    float acc_scale;        // multiplies the accumulator (1 for fp16; s_a*s_w for int8)
    const float* acc_scale_ptr;  // optional device scalar multiplied in as well (per-layer gradient un-scaling)
    int ab_bf16;            // 16-bit operands are bf16 (both: wgmma takes one format for A and B)
    int res_bf16;           // residual / accumulate tensor is bf16 instead of fp16
    const __half* res;      // optional residual (16-bit, NHWC) added after the activation
    long long res_pitch;    // elements per pixel row
    void* out;
    long long out_pitch;    // elements per pixel row
    int out_dtype;          // OUT_*
    float out_inv_scale;    // int8 output: q = clamp(round_half_away(v * out_inv_scale))
    float out_scale;        //              (and v_dequant = q * out_scale when out is fp16/fp32 fake-quant)
    int out_fakequant;      // 1: write the dequantised value q*out_scale in out_dtype (fp16/fp32)
    float q_lo, q_hi;       // clamp range, e.g. -128, 127
    // training extras: per-channel sum / sum of squares of the raw (pre-bias) output, accumulated in double
    // ([0, CONV_STAT_MAX) sums, [CONV_STAT_MAX, 2 CONV_STAT_MAX) squares) so that the result does not depend on the order
    // of the atomics: the variance is E[z^2] - E[z]^2, and that cancellation magnifies fp32 ordering noise, which
    // batch-statistics BatchNorm then carries through every later layer
    double* stat_acc;
    int b_resident;         // 1: the whole weight panel of the (single) N tile stays in smem, loaded once per CTA
    int num_stages;         // smem ring depth for this launch (<= 32)
    int epi_tma;            // the short epilogue stores through smem + TMA (tmC valid); rows / columns clipped by the map
    int epi_fast;           // host-checked: 16-bit out, whole channel tiles, 16-byte aligned bias/residual/output
    // int8 graph: quantised shortcut folded into the epilogue (COSPTQuantizedShortcut eval, ptq_cos.py:876-884 / 931-933):
    //   code = clamp(rha((rha(q*out_scale*qs_rx)*qs_x + rha(a*qs_a_in*qs_ra)*qs_a) * qs_rsum)),  q = this conv's int8 code,
    // all scales powers of two (host-checked), so every product is exact and equals the stand-alone kernel bit for bit
    const int8_t* qres;     // the other addend's int8 codes (NHWC) or null
    long long qres_pitch;
    float qs_rx, qs_x, qs_a_in, qs_ra, qs_a, qs_rsum, qs_lo, qs_hi;
    int qs_clamp;           // the addend codes are clamped to [qs_lo, qs_hi] too (google QuantizedShortcut_max)
    int qs_simple;          // both addend roundings are identities: code = clamp(rha(q*qs_cx + a*qs_ca))
    float qs_cx, qs_ca;     // out_scale / scale_sum, a_in / scale_sum
};

// Opt-in shared memory per block on sm_90 (227 KB); the ring of k-step stages takes what the epilogue leaves.
constexpr int CONV_SMEM_LIMIT = 227 * 1024;
constexpr int conv_max_stage_smem(int block_n) {
    return ((CONV_SMEM_LIMIT - 1024 - 1024 - 8 * 4096 - 128 * block_n * 4) / 1024) * 1024;
}

template <int BLOCK_N, int KBYTES>
struct ConvTcCfg {
    static constexpr int BLOCK_M = 128;
    static constexpr int A_BYTES = BLOCK_M * KBYTES;
    static constexpr int B_BYTES = BLOCK_N * KBYTES;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;  // always a multiple of 1024
    static constexpr int MAX_STAGE_SMEM = conv_max_stage_smem(BLOCK_N);
    static constexpr int AUX_BYTES = 1024;  // barriers, at a fixed offset behind the tile area
    static constexpr int EPI_STAGE_BYTES = 8 * 4096;   // per epilogue warp: 2 x 2 KB output staging for TMA stores
    static constexpr int ACC_BYTES = BLOCK_M * BLOCK_N * 4;   // fp32 / int32 accumulator tile between MMA and epilogue
    static constexpr int SMEM_BYTES = 1024 /*align slack*/ + MAX_STAGE_SMEM + AUX_BYTES + EPI_STAGE_BYTES + ACC_BYTES;
    static_assert(SMEM_BYTES <= CONV_SMEM_LIMIT, "shared memory");
};

__device__ __noinline__ float mish_noinline(float x) { return mish_f(x); }
__device__ __noinline__ float swish_noinline(float x) { return x * sigmoid_f(x); }

__device__ __forceinline__ float round_half_away(float x) {
    // reference utils/quantized/quantized_ptq_cos.py:14-20  sign(x)*floor(|x|+0.5)
    return copysignf(floorf(fabsf(x) + 0.5f), x);
}

// The same rounding for |x| < 2^22 without the conversion pipe (FRND / F2I issue at a quarter of the FP32 rate and bound
// the int8 epilogues): floor(t) = (t + 2^23 rounded DOWN) - 2^23 for 0 <= t < 2^23.
__device__ __forceinline__ float round_half_away_small(float x) {
    const float t = fabsf(x) + 0.5f;
    return copysignf(__fadd_rd(t, 8388608.f) - 8388608.f, x);
}
// four integer-valued floats in [-128, 127] -> packed int8: the low byte of (v + 1.5 * 2^23) is v's two's complement
__device__ __forceinline__ uint32_t pack_i8x4(float a, float b, float c, float d) {
    const uint32_t ua = __float_as_uint(a + 12582912.f), ub = __float_as_uint(b + 12582912.f);
    const uint32_t uc = __float_as_uint(c + 12582912.f), ud = __float_as_uint(d + 12582912.f);
    return __byte_perm(__byte_perm(ua, ub, 0x0040), __byte_perm(uc, ud, 0x0040), 0x5410);
}

struct ConvTcEpi {
    // two consumer warpgroups (warps 4-11): each issues the MMAs of 64 of the 128 tile rows; in the epilogue warp w
    // takes rows 32 (w % 4) .. + 31 (thread = row) and every other 32-column chunk (w / 4 = chunk parity)
    static constexpr int WARPS = 8;
    static constexpr int THREADS = 128 + 32 * WARPS;
};

// General (slow-path) epilogue for one 32-column chunk: every output type, partial channel tiles, batch statistics,
// int8 requantisation.  `v` holds the scaled accumulators on entry.
template <int KIND>
__device__ __forceinline__ void epi_chunk_general(float (&v)[32], const ConvTcParams& p, int n0c0, long long row,
                                               bool row_ok, int lane, uint8_t* stage, bool defer_stats, float& ds1,
                                               float& ds2) {
    ds1 = ds2 = 0.f;
    if (p.stat_acc != nullptr) {
        // per-channel batch statistics of the raw conv output (training BN): the warp's 32x32 chunk goes through its smem
        // staging tile (rotated columns: conflict-free both ways), then lane j sums column j -- 32 STS + 32 LDS instead of
        // 640 shuffles per chunk
        float* tile = reinterpret_cast<float*>(stage);
#pragma unroll
        for (int j = 0; j < 32; ++j) tile[lane * 32 + ((j + lane) & 31)] = row_ok ? v[j] : 0.f;
        __syncwarp();
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const float t = tile[i * 32 + ((lane + i) & 31)];
            s1 += t;
            s2 = fmaf(t, t, s2);
        }
        __syncwarp();
        if (defer_stats) {          // single N tile: the warp keeps per-column partial sums across its tiles
            ds1 = s1;
            ds2 = s2;
        } else if (n0c0 + lane < p.Cout) {
            atomicAdd(p.stat_acc + n0c0 + lane, (double)s1);
            atomicAdd(p.stat_acc + CONV_STAT_MAX + n0c0 + lane, (double)s2);
        }
    }
    const int nvalid = min(32, p.Cout - n0c0);
    if (p.bias != nullptr) {
#pragma unroll
        for (int j = 0; j < 32; ++j)
            if (j < nvalid) v[j] += __ldg(p.bias + n0c0 + j);
    }
    switch (p.act) {
        case B2Y_ACT_LEAKY:
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = v[j] > 0.f ? v[j] : v[j] * p.slope;
            break;
        case B2Y_ACT_MISH:
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = mish_noinline(v[j]);
            break;
        case B2Y_ACT_RELU:
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
            break;
        case B2Y_ACT_RELU6:
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = fminf(fmaxf(v[j], 0.f), 6.f);
            break;
        case B2Y_ACT_HSWISH:
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = v[j] * (fminf(fmaxf(v[j] + 3.f, 0.f), 6.f) / 6.f);
            break;
        case B2Y_ACT_SWISH:
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = swish_noinline(v[j]);
            break;
        default:
            break;
    }
    if (!row_ok) return;
    if (p.res != nullptr) {
        const __half* rp = p.res + row * p.res_pitch + n0c0;
#pragma unroll
        for (int j = 0; j < 32; ++j)
            if (j < nvalid)
                v[j] += p.res_bf16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(rp)[j]) : __half2float(rp[j]);
    }
    if (p.out_fakequant || p.out_dtype == OUT_I8) {
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            float q = round_half_away(v[j] * p.out_inv_scale);
            q = fminf(fmaxf(q, p.q_lo), p.q_hi);
            v[j] = (p.out_dtype == OUT_I8) ? q : q * p.out_scale;
        }
    }
    if (p.out_dtype == OUT_BF16) {
        __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(p.out) + row * p.out_pitch + n0c0;
        if (nvalid == 32 && ((reinterpret_cast<uintptr_t>(op) & 15) == 0)) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                uint4 u;
                __nv_bfloat162* h2 = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
                for (int t = 0; t < 4; ++t) h2[t] = __floats2bfloat162_rn(v[q * 8 + t * 2], v[q * 8 + t * 2 + 1]);
                reinterpret_cast<uint4*>(op)[q] = u;
            }
        } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
                if (j < nvalid) op[j] = __float2bfloat16_rn(v[j]);
        }
    } else if (p.out_dtype == OUT_F16) {
        __half* op = reinterpret_cast<__half*>(p.out) + row * p.out_pitch + n0c0;
        if (nvalid == 32 && ((reinterpret_cast<uintptr_t>(op) & 15) == 0)) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                uint4 u;
                __half2* h2 = reinterpret_cast<__half2*>(&u);
#pragma unroll
                for (int t = 0; t < 4; ++t) h2[t] = __floats2half2_rn(v[q * 8 + t * 2], v[q * 8 + t * 2 + 1]);
                reinterpret_cast<uint4*>(op)[q] = u;
            }
        } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
                if (j < nvalid) op[j] = __float2half_rn(v[j]);
        }
    } else if (p.out_dtype == OUT_F32) {
        float* op = reinterpret_cast<float*>(p.out) + row * p.out_pitch + n0c0;
        if (nvalid == 32 && ((reinterpret_cast<uintptr_t>(op) & 15) == 0)) {
#pragma unroll
            for (int q = 0; q < 8; ++q)
                reinterpret_cast<float4*>(op)[q] = make_float4(v[q * 4], v[q * 4 + 1], v[q * 4 + 2], v[q * 4 + 3]);
        } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
                if (j < nvalid) op[j] = v[j];
        }
    } else {  // OUT_I8
        int8_t* op = reinterpret_cast<int8_t*>(p.out) + row * p.out_pitch + n0c0;
        if (nvalid == 32 && ((reinterpret_cast<uintptr_t>(op) & 15) == 0)) {
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                uint32_t w[4];
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    const int b = q * 16 + t * 4;
                    w[t] = ((uint32_t)(uint8_t)(int8_t)(int)v[b]) | ((uint32_t)(uint8_t)(int8_t)(int)v[b + 1] << 8) |
                           ((uint32_t)(uint8_t)(int8_t)(int)v[b + 2] << 16) |
                           ((uint32_t)(uint8_t)(int8_t)(int)v[b + 3] << 24);
                }
                reinterpret_cast<uint4*>(op)[q] = make_uint4(w[0], w[1], w[2], w[3]);
            }
        } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
                if (j < nvalid) op[j] = (int8_t)(int)v[j];
        }
    }
}

// CLUSTER > 1: the CTAs of a cluster work on CLUSTER consecutive M tiles of the same N tile; each loads 1/CLUSTER of
// the weight tile and TMA-multicasts it to all of them, so the weight re-reads from L2 drop by CLUSTER x.  A stage is
// free again once the consumer warps of every CTA of the cluster have released it.
template <int BLOCK_N, int KBYTES, int KIND, int CLUSTER>
__global__ void __launch_bounds__(ConvTcEpi::THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmC, const __grid_constant__ ConvTcParams p) {
    using Cfg = ConvTcCfg<BLOCK_N, KBYTES>;
    constexpr int MAX_NS = 32;
    constexpr int ESIZE = (KIND == CONV_KIND_F16) ? 2 : 1;
    constexpr int BLOCK_K = KBYTES / ESIZE;  // elements per k-chunk
    constexpr uint32_t LAYOUT = swizzle_layout_type(KBYTES);
    using AccT = typename std::conditional<KIND == CONV_KIND_F16, float, uint32_t>::type;

    // smem: [ns stages of A (+B)] [resident weight panel, if any] ... [aux] [epilogue staging] [accumulator tile]
    const bool b_res = CLUSTER == 1 && p.b_resident != 0;
    const int ns = p.num_stages;
    const uint32_t stage_bytes = b_res ? (uint32_t)Cfg::A_BYTES : (uint32_t)Cfg::STAGE_BYTES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* aux = smem + Cfg::MAX_STAGE_SMEM;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(aux);           // [MAX_NS]
    uint64_t* empty_bar = full_bar + MAX_NS;                         // [MAX_NS]
    uint64_t* bres_bar = empty_bar + MAX_NS;                         // [1] resident weight panel landed
    uint8_t* epi_stage = aux + Cfg::AUX_BYTES;                       // [8 warps][4096] output staging for TMA stores
    uint8_t* acc_stage = epi_stage + Cfg::EPI_STAGE_BYTES;           // [128][BLOCK_N] accumulators

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == 0 && lane == 0) {
        prefetch_tmap(&tmA);
        prefetch_tmap(&tmB);
        prefetch_tmap(&tmC);
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < ns; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], ConvTcEpi::WARPS * CLUSTER);   // every consumer warp of every CTA that reads it
        }
        mbar_init(bres_bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (CLUSTER > 1) cluster_sync_all();   // barriers of every CTA are initialised before any remote arrive / multicast

    // work items: (group of CLUSTER consecutive M tiles, N tile); this CTA takes M tile group*CLUSTER + rank.
    // A "ghost" M tile past the end still runs the pipeline (TMA zero fill) but stores nothing.
    const int cta_rank = CLUSTER > 1 ? (int)cluster_ctarank() : 0;
    const int cluster_id = (int)blockIdx.x / CLUSTER;
    const int num_clusters = (int)gridDim.x / CLUSTER;
    const int num_n_tiles = p.num_n_tiles;
    const int num_mgroups = (p.num_m_tiles + CLUSTER - 1) / CLUSTER;
    const int num_items = num_mgroups * num_n_tiles;
    constexpr uint16_t MC_MASK = (uint16_t)((1u << CLUSTER) - 1u);
    const int taps = p.ntaps;
    const int k_chunks = p.k_chunks;
    const uint32_t smem_base = smem_u32(smem);
    const uint32_t full_base = smem_u32(full_bar);
    const uint32_t empty_base = smem_u32(empty_bar);
    const uint32_t bres_base = smem_base + (uint32_t)ns * stage_bytes;     // resident weight panel (k_steps x B tile)

    // The issue loop is executed by the whole (converged) warp with one elected lane doing the issue: all loop state is
    // then warp-uniform and lives in the uniform datapath.
    if (warp == 0) {
        // ===================== TMA producer =====================
        uint32_t stage = 0, phase = 0;
        const int HoWo = p.MH * p.MW;
        const int MW = p.MW;
        const int cstride = p.stride, lower_w = p.lower_w, lower_h = p.lower_h, Cin = p.Cin;
        const bool im2col = p.a_mode == A_MODE_IM2COL;
        const unsigned long long tw = p.tap_w_packed, th = p.tap_h_packed;
        if (b_res && elect_one()) {
            // weight-stationary: all k-steps of the (only) N tile are fetched once; the ring then carries A alone
            const int k_steps = taps * k_chunks;
            mbar_expect_tx_s(smem_u32(bres_bar), (uint32_t)k_steps * Cfg::B_BYTES);
            for (int ks = 0; ks < k_steps; ++ks)
                tma_load_2d_s(bres_base + ks * Cfg::B_BYTES, &tmB, smem_u32(bres_bar), ks * BLOCK_K, 0);
        }
        __syncwarp();
        // everything above (barriers, the static weights) may overlap the tail of the previous layer's kernel;
        // activations must not be touched before it has completed (programmatic dependent launch)
        pdl_wait();
        pdl_launch_dependents();
        for (int item = cluster_id; item < num_items; item += num_clusters) {
            const int mgroup = item / num_n_tiles;
            const int n_tile = item - mgroup * num_n_tiles;
            const int m0 = (mgroup * CLUSTER + cta_rank) * 128;
            int img = 0, base_w = 0, base_h = 0;
            if (im2col) {
                img = m0 / HoWo;
                const int rem = m0 - img * HoWo;
                const int po = rem / MW;
                base_w = (rem - po * MW) * cstride + lower_w;
                base_h = po * p.stride_h + lower_h;
            }
            const int b_row = n_tile * BLOCK_N + (CLUSTER > 1 ? cta_rank * (BLOCK_N / CLUSTER) : 0);
            int b_k = 0;
            for (int tap = 0; tap < taps; ++tap) {
                const uint16_t s = (uint16_t)((tw >> (4 * tap)) & 15);
                const uint16_t r = (uint16_t)((th >> (4 * tap)) & 15);
                int a_c = 0;
                for (int kc = 0; kc < k_chunks; ++kc) {
                    mbar_wait_s(empty_base + stage * 8, phase ^ 1);
                    if (elect_one()) {
                        const uint32_t a_dst = smem_base + stage * stage_bytes;
                        const uint32_t b_dst = a_dst + Cfg::A_BYTES;
                        const uint32_t fb = full_base + stage * 8;
                        mbar_expect_tx_s(fb, stage_bytes);
                        if (im2col)
                            tma_load_im2col_4d_s(a_dst, &tmA, fb, a_c, base_w, base_h, img, s, r);
                        else
                            tma_load_2d_s(a_dst, &tmA, fb, a_c, m0);
                        if (CLUSTER > 1)
                            tma_load_2d_multicast_s(b_dst + cta_rank * (BLOCK_N / CLUSTER) * KBYTES, &tmB, fb, b_k, b_row,
                                                    MC_MASK);
                        else if (!b_res)
                            tma_load_2d_s(b_dst, &tmB, fb, b_k, b_row);
                    }
                    a_c += BLOCK_K;
                    b_k += BLOCK_K;
                    if (++stage == (uint32_t)ns) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
                b_k += Cin - k_chunks * BLOCK_K;   // == 0 (Cin is a whole number of chunks); keeps the intent explicit
            }
        }
    } else if (warp >= 4) {
        // ===================== MMA (two warpgroups, 64 rows each) + epilogue =====================
        const int wg = (warp - 4) >> 2;
        const int tid_wg = (int)threadIdx.x & 127;
        const int k_steps = taps * k_chunks;
        const uint64_t desc_base = smem_desc_base(16, 8 * KBYTES, LAYOUT);
        const bool ab_bf16 = p.ab_bf16 != 0;
        uint32_t stage = 0, phase = 0;
        pdl_wait();
        const float acc_mul = p.acc_scale * (p.acc_scale_ptr != nullptr ? __ldg(p.acc_scale_ptr) : 1.f);
        const int ew = (warp - 4) & 3;          // row quarter of the tile
        const int cg = (warp - 4) >> 2;         // chunk parity
        const bool fast = p.epi_fast != 0;
        const int act = p.act;
        const float slope = p.slope;
        const int hw = p.MH * p.MW;
        const bool epi_tma = p.epi_tma != 0;
        uint8_t* my_stage = epi_stage + (warp - 4) * 4096;
        const int trow = ew * 32 + lane;        // this thread's row of the tile in the epilogue
        int sbuf = 0;
        // training BN statistics: with a single N tile every tile of this warp covers the same columns, so the channel
        // sums are kept in registers (lane j = column j of chunk q) and flushed with ONE atomic per column per warp at the
        // end -- instead of one per column per 32-row chunk (millions of same-address L2 atomics on the large early layers)
        const bool defer_stats = p.stat_acc != nullptr && num_n_tiles == 1;
        float st1[2] = {0.f, 0.f}, st2[2] = {0.f, 0.f};
        if (b_res) mbar_wait_s(smem_u32(bres_bar), 0);
        for (int item = cluster_id; item < num_items; item += num_clusters) {
            const int mgroup = item / num_n_tiles;
            const int n_tile = item - mgroup * num_n_tiles;
            const int m_tile = mgroup * CLUSTER + cta_rank;
            const int n0 = n_tile * BLOCK_N;

            AccT acc[BLOCK_N / 2];
            uint32_t prev = 0;
            for (int ks = 0; ks < k_steps; ++ks) {
                mbar_wait_s(full_base + stage * 8, phase);
                const uint32_t a_tile = smem_base + stage * stage_bytes;
                const uint32_t a_addr = a_tile + (uint32_t)(wg * 64 * KBYTES);
                const uint32_t b_addr = b_res ? bres_base + ks * Cfg::B_BYTES : a_tile + Cfg::A_BYTES;
                const uint64_t adesc = desc_base | (uint64_t)((a_addr >> 4) & 0x3FFF);
                const uint64_t bdesc = desc_base | (uint64_t)((b_addr >> 4) & 0x3FFF);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < KBYTES / 32; ++k) {
                    const uint32_t sc = (ks > 0 || k > 0) ? 1u : 0u;
                    if constexpr (KIND == CONV_KIND_I8)
                        wgmma_ss<BLOCK_N, 2, 0>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), sc);
                    else if (ab_bf16)
                        wgmma_ss<BLOCK_N, 1, 0>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), sc);
                    else
                        wgmma_ss<BLOCK_N, 0, 0>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), sc);
                }
                wgmma_commit();
                if (ks > 0) {
                    // the MMAs of the previous k-step have retired: its smem slot goes back to the producer(s)
                    wgmma_wait<1>();
                    if (lane == 0) {
                        if (CLUSTER == 1) {
                            mbar_arrive(&empty_bar[prev]);
                        } else {
#pragma unroll
                            for (int r = 0; r < CLUSTER; ++r) mbar_arrive_cluster(mapa_u32(empty_base + prev * 8, r));
                        }
                    }
                }
                prev = stage;
                if (++stage == (uint32_t)ns) {
                    stage = 0;
                    phase ^= 1;
                }
            }
            wgmma_wait<0>();
            wgmma_fence_acc(acc);
            if (lane == 0) {
                if (CLUSTER == 1) {
                    mbar_arrive(&empty_bar[prev]);
                } else {
#pragma unroll
                    for (int r = 0; r < CLUSTER; ++r) mbar_arrive_cluster(mapa_u32(empty_base + prev * 8, r));
                }
            }
            // accumulators -> smem (after every epilogue thread is done with the previous tile's)
            named_bar_sync(1, 256);
            frag_to_stage<BLOCK_N>(acc, acc_stage, wg * 64, tid_wg);
            named_bar_sync(1, 256);

            const long long grow = (long long)m_tile * 128 + trow;              // GEMM row
            const bool row_ok = grow < p.M_total;
            long long row = grow;                                              // output pixel index
            if (!p.out_identity && row_ok) {
                const int n_ = (int)(grow / hw);
                const int r_ = (int)(grow - (long long)n_ * hw);
                const int p_ = r_ / p.MW, q_ = r_ - p_ * p.MW;
                row = ((long long)n_ * p.out_OH + (long long)p_ * p.out_ys + p.out_y0) * p.out_OW +
                      (long long)q_ * p.out_xs + p.out_x0;
            }

#pragma unroll 1
            for (int J = cg; J < BLOCK_N / 32; J += 2) {
                const int cc = J * 32;                                   // column offset of the chunk in the tile
                if (fast) {
                    // short path: 16-bit output (or fp32 through TMA), vector-aligned bias / residual / output (checked on
                    // the host); a clipped last N tile is allowed on TMA-store launches
                    const int cvalid = p.Cout - (n0 + cc);               // < 32 only in the last chunk of a clipped tile
                    if (cvalid <= 0) break;                              // (TMA-store launches only; warp-uniform)
                    uint32_t raw[32];
                    stage_row32<BLOCK_N>(acc_stage, trow, cc, raw);
                    const float* bias_p = p.bias != nullptr ? p.bias + n0 + cc : nullptr;
                    float4 bv[8];
                    if (bias_p != nullptr && cvalid >= 32) {
#pragma unroll
                        for (int q = 0; q < 8; ++q) bv[q] = __ldg(reinterpret_cast<const float4*>(bias_p) + q);
                    } else if (bias_p != nullptr) {
#pragma unroll
                        for (int q = 0; q < 8; ++q) {
                            bv[q].x = 4 * q < cvalid ? __ldg(bias_p + 4 * q) : 0.f;
                            bv[q].y = 4 * q + 1 < cvalid ? __ldg(bias_p + 4 * q + 1) : 0.f;
                            bv[q].z = 4 * q + 2 < cvalid ? __ldg(bias_p + 4 * q + 2) : 0.f;
                            bv[q].w = 4 * q + 3 < cvalid ? __ldg(bias_p + 4 * q + 3) : 0.f;
                        }
                    } else {
#pragma unroll
                        for (int q = 0; q < 8; ++q) bv[q] = make_float4(0.f, 0.f, 0.f, 0.f);
                    }
                    uint4 qa[2] = {make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0)};
                    if (KIND == CONV_KIND_I8 && p.qres != nullptr && row_ok) {
                        const uint4* ap = reinterpret_cast<const uint4*>(p.qres + row * p.qres_pitch + n0 + cc);
                        qa[0] = __ldg(ap);
                        qa[1] = __ldg(ap + 1);
                    }
                    uint4 rcur[4];
                    const bool has_res = p.res != nullptr && row_ok;
                    if (has_res) {
                        const uint4* res_p = reinterpret_cast<const uint4*>(p.res + row * p.res_pitch + n0 + cc);
#pragma unroll
                        for (int q = 0; q < 4; ++q) rcur[q] = __ldg(res_p + q);
                    }
                    float v[32];
#pragma unroll
                    for (int q = 0; q < 8; ++q) {
                        const float a0 = (KIND == CONV_KIND_F16) ? __uint_as_float(raw[4 * q]) : (float)(int)raw[4 * q];
                        const float a1 = (KIND == CONV_KIND_F16) ? __uint_as_float(raw[4 * q + 1]) : (float)(int)raw[4 * q + 1];
                        const float a2 = (KIND == CONV_KIND_F16) ? __uint_as_float(raw[4 * q + 2]) : (float)(int)raw[4 * q + 2];
                        const float a3 = (KIND == CONV_KIND_F16) ? __uint_as_float(raw[4 * q + 3]) : (float)(int)raw[4 * q + 3];
                        v[4 * q] = fmaf(a0, acc_mul, bv[q].x);
                        v[4 * q + 1] = fmaf(a1, acc_mul, bv[q].y);
                        v[4 * q + 2] = fmaf(a2, acc_mul, bv[q].z);
                        v[4 * q + 3] = fmaf(a3, acc_mul, bv[q].w);
                    }
                    if (KIND == CONV_KIND_F16 && p.stat_acc != nullptr) {
                        // training BN statistics on the short path (host: TMA store, no bias, no residual): column sums of
                        // the warp's 32 x 32 chunk through the 2 KB staging buffer the NEXT TMA store will use, 16 columns
                        // at a time (rotated columns; lane L sums column L & 15 over rows 16 (L >> 4) .. + 15)
                        float* tile = reinterpret_cast<float*>(my_stage + sbuf * 2048);
                        if (lane == 0) bulk_wait_read<1>();      // the store that last read this buffer is done with it
                        __syncwarp();
                        float s1 = 0.f, s2 = 0.f;
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
#pragma unroll
                            for (int j = 0; j < 16; ++j) tile[lane * 16 + ((j + lane) & 15)] = row_ok ? v[h * 16 + j] : 0.f;
                            __syncwarp();
                            const int col = lane & 15, r0 = (lane >> 4) * 16;
                            float t1 = 0.f, t2 = 0.f;
#pragma unroll
                            for (int i = 0; i < 16; ++i) {
                                const float t = tile[(r0 + i) * 16 + ((col + r0 + i) & 15)];
                                t1 += t;
                                t2 = fmaf(t, t, t2);
                            }
                            t1 += __shfl_xor_sync(0xffffffffu, t1, 16);
                            t2 += __shfl_xor_sync(0xffffffffu, t2, 16);
                            if ((lane >> 4) == h) {
                                s1 = t1;
                                s2 = t2;
                            }
                            __syncwarp();
                        }
                        if (defer_stats) {
#pragma unroll
                            for (int q = 0; q < 2; ++q)
                                if ((J >> 1) == q) {
                                    st1[q] += s1;
                                    st2[q] += s2;
                                }
                        } else if (n0 + cc + lane < p.Cout) {
                            atomicAdd(p.stat_acc + n0 + cc + lane, (double)s1);
                            atomicAdd(p.stat_acc + CONV_STAT_MAX + n0 + cc + lane, (double)s2);
                        }
                    }
                    if (act == B2Y_ACT_LEAKY) {       // 0 <= slope <= 1 on this path: max(v, slope*v)
#pragma unroll
                        for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], v[j] * slope);
                    } else if (act == B2Y_ACT_MISH) {
                        // inlined closed form (one ex2, one rcp per element): 32 independent dependency chains the
                        // scheduler can interleave
#pragma unroll
                        for (int j = 0; j < 32; ++j) v[j] = mish_f(v[j]);
                    }
                    if (has_res) {
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            const uint4 u = rcur[q];
                            if (p.res_bf16) {
                                const __nv_bfloat162* b2 = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
                                for (int t = 0; t < 4; ++t) {
                                    const float2 f = __bfloat1622float2(b2[t]);
                                    v[q * 8 + t * 2] += f.x;
                                    v[q * 8 + t * 2 + 1] += f.y;
                                }
                            } else {
                                const __half2* h2 = reinterpret_cast<const __half2*>(&u);
#pragma unroll
                                for (int t = 0; t < 4; ++t) {
                                    const float2 f = __half22float2(h2[t]);
                                    v[q * 8 + t * 2] += f.x;
                                    v[q * 8 + t * 2 + 1] += f.y;
                                }
                            }
                        }
                    }
                    if (KIND == CONV_KIND_I8 && (p.out_dtype == OUT_I8 || p.out_fakequant)) {
                        // int8 graph: requantise exactly like the general path (round half away, clamp); values are
                        // identical because acc_mul is a power of two there
                        // clamp first: the bounds are integers and the rounding is monotone, so the result is the same
                        // and the rounding operand is small
#pragma unroll
                        for (int j = 0; j < 32; ++j)
                            v[j] = round_half_away_small(fminf(fmaxf(v[j] * p.out_inv_scale, p.q_lo), p.q_hi));
                        if (p.qres != nullptr && p.qs_simple) {
                            // both addends already sit on the common grid (scale_x <= out_scale, scale_a <= sa_in: what the
                            // _min / _max shortcuts vote): their roundings are identities, the sum is exact in fp32
                            const uint32_t* aw = reinterpret_cast<const uint32_t*>(qa);
#pragma unroll
                            for (int t = 0; t < 8; ++t) {
                                const uint32_t ax = aw[t] ^ 0x80808080u;
#pragma unroll
                                for (int e = 0; e < 4; ++e) {
                                    const float af = __uint_as_float(__byte_perm(ax, 0x4B400000u, 0x7650u | e)) - 12583040.f;
                                    const float tt = fmaf(af, p.qs_ca, v[t * 4 + e] * p.qs_cx);
                                    v[t * 4 + e] = round_half_away_small(fminf(fmaxf(tt, p.qs_lo), p.qs_hi));
                                }
                            }
                        } else if (p.qres != nullptr) {
                            const int8_t* ab = reinterpret_cast<const int8_t*>(qa);
#pragma unroll
                            for (int j = 0; j < 32; ++j) {
                                float xr = round_half_away(v[j] * p.out_scale * p.qs_rx);   // rounded, clamped in
                                float ar = round_half_away((float)ab[j] * p.qs_a_in * p.qs_ra);  // qs_clamp mode only
                                if (p.qs_clamp) {
                                    xr = fminf(fmaxf(xr, p.qs_lo), p.qs_hi);
                                    ar = fminf(fmaxf(ar, p.qs_lo), p.qs_hi);
                                }
                                const float xf = xr * p.qs_x, af = ar * p.qs_a;
                                const float q = round_half_away((xf + af) * p.qs_rsum);
                                v[j] = fminf(fmaxf(q, p.qs_lo), p.qs_hi);
                            }
                        } else if (p.out_fakequant) {
#pragma unroll
                            for (int j = 0; j < 32; ++j) v[j] *= p.out_scale;
                        }
                    }
                    if (p.out_dtype == OUT_I8) {
                        uint32_t w[8];
#pragma unroll
                        for (int t = 0; t < 8; ++t) w[t] = pack_i8x4(v[t * 4], v[t * 4 + 1], v[t * 4 + 2], v[t * 4 + 3]);
                        if (epi_tma) {
                            // 32 rows x 32 B through smem (SWIZZLE_32B image) and one TMA store: whole 32-byte sectors per
                            // row reach L2 in one request instead of 2 x 32 scattered 16-byte pieces
                            uint8_t* buf = my_stage + sbuf * 2048;
                            if (lane == 0) bulk_wait_read<1>();
                            __syncwarp();
                            const int sw = (lane >> 2) & 1;
                            *reinterpret_cast<uint4*>(buf + lane * 32 + ((0 ^ sw) << 4)) = make_uint4(w[0], w[1], w[2], w[3]);
                            *reinterpret_cast<uint4*>(buf + lane * 32 + ((1 ^ sw) << 4)) = make_uint4(w[4], w[5], w[6], w[7]);
                            fence_proxy_async_cta();
                            __syncwarp();
                            if (lane == 0) {
                                tma_store_2d(&tmC, smem_u32(buf), n0 + cc, m_tile * 128 + ew * 32);
                                bulk_commit();
                            }
                            sbuf ^= 1;
                        } else if (row_ok) {
                            uint4* op8 = reinterpret_cast<uint4*>(reinterpret_cast<int8_t*>(p.out) + row * p.out_pitch + n0 + cc);
                            op8[0] = make_uint4(w[0], w[1], w[2], w[3]);
                            op8[1] = make_uint4(w[4], w[5], w[6], w[7]);
                        }
                        continue;
                    }
                    if (p.out_dtype == OUT_F32) {
                        // fp32 rows (YOLO head): 32 rows x 128 B, SWIZZLE_128B image, one TMA store; the map clips column 255
                        uint8_t* buf = my_stage;
                        if (lane == 0) bulk_wait_read<0>();
                        __syncwarp();
#pragma unroll
                        for (int q = 0; q < 8; ++q)
                            *reinterpret_cast<float4*>(buf + lane * 128 + ((q ^ (lane & 7)) << 4)) =
                                make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
                        fence_proxy_async_cta();
                        __syncwarp();
                        if (lane == 0) {
                            tma_store_2d(&tmC, smem_u32(buf), n0 + cc, m_tile * 128 + ew * 32);
                            bulk_commit();
                        }
                        continue;
                    }
                    uint4 ou[4];
                    if (p.out_dtype == OUT_BF16) {
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            __nv_bfloat162* h2 = reinterpret_cast<__nv_bfloat162*>(&ou[q]);
#pragma unroll
                            for (int t = 0; t < 4; ++t) h2[t] = __floats2bfloat162_rn(v[q * 8 + t * 2], v[q * 8 + t * 2 + 1]);
                        }
                    } else {
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            __half2* h2 = reinterpret_cast<__half2*>(&ou[q]);
#pragma unroll
                            for (int t = 0; t < 4; ++t) h2[t] = __floats2half2_rn(v[q * 8 + t * 2], v[q * 8 + t * 2 + 1]);
                        }
                    }
                    if (epi_tma) {
                        // 32 rows x 64 B through smem (SWIZZLE_64B image) and one TMA store: full 64-byte row segments reach
                        // L2 instead of 32 scattered 16-byte pieces per store instruction; the map clips the M / Cout tails
                        uint8_t* buf = my_stage + sbuf * 2048;
                        if (lane == 0) bulk_wait_read<1>();      // the store that last read this buffer is done with it
                        __syncwarp();
#pragma unroll
                        for (int q = 0; q < 4; ++q)
                            *reinterpret_cast<uint4*>(buf + lane * 64 + ((q ^ ((lane >> 1) & 3)) << 4)) = ou[q];
                        fence_proxy_async_cta();
                        __syncwarp();
                        if (lane == 0) {
                            tma_store_2d(&tmC, smem_u32(buf), n0 + cc, m_tile * 128 + ew * 32);
                            bulk_commit();
                        }
                        sbuf ^= 1;
                    } else if (row_ok) {
                        uint4* out_p = reinterpret_cast<uint4*>(reinterpret_cast<__half*>(p.out) + row * p.out_pitch + n0 + cc);
#pragma unroll
                        for (int q = 0; q < 4; ++q) out_p[q] = ou[q];
                    }
                } else {
                    if (n0 + cc >= p.Cout) continue;  // warp-uniform
                    uint32_t raw[32];
                    stage_row32<BLOCK_N>(acc_stage, trow, cc, raw);
                    float v[32];
#pragma unroll
                    for (int j = 0; j < 32; ++j)
                        v[j] = ((KIND == CONV_KIND_F16) ? __uint_as_float(raw[j]) : (float)(int)raw[j]) * acc_mul;
                    float ds1, ds2;
                    epi_chunk_general<KIND>(v, p, n0 + cc, row, row_ok, lane, my_stage, defer_stats, ds1, ds2);
#pragma unroll
                    for (int q = 0; q < 2; ++q)
                        if ((J >> 1) == q) {
                            st1[q] += ds1;
                            st2[q] += ds2;
                        }
                }
            }
        }
        if (defer_stats) {
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                const int col = (2 * q + cg) * 32 + lane;
                if ((2 * q + cg) * 32 < BLOCK_N && col < p.Cout && (st1[q] != 0.f || st2[q] != 0.f)) {
                    atomicAdd(p.stat_acc + col, (double)st1[q]);
                    atomicAdd(p.stat_acc + CONV_STAT_MAX + col, (double)st2[q]);
                }
            }
        }
        if (epi_tma && lane == 0) bulk_wait_all();   // outstanding TMA stores complete before the CTA exits
    }

    __syncthreads();
    if (CLUSTER > 1) cluster_sync_all();   // nobody leaves while a peer may still multicast / arrive into its smem
}

}  // namespace b2y
