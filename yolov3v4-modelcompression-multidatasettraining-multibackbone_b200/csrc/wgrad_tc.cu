// Weight gradient of a dense convolution as a wgmma GEMM with the *pixel* dimension as K:
//
//   dW[co][tap][ci] = sum_{pixel m} dY[m][co] * X[m @ tap][ci]
//
// Both operands are pixel-major in HBM (NHWC), i.e. "MN-major" for the tensor core: the TMA boxes
// [64 pixels][64 channels] land in smem exactly as a 128B-swizzled MN-major wgmma operand, so neither
// tensor is ever transposed or im2col'ed in memory.  dY comes through a tiled 2-D map, X through the im2col
// map (tap offset + zero fill for the halo).  Work = (Cout/128) x (Cin/BLOCK_N) x taps x split-K slices.
// With one slice the fp32 accumulator tile is added straight into dW (each element has one owner).  With S > 1 slices
// every CTA stores its tile into slice `split` of a per-stream workspace, and wgrad_reduce_kernel then sums the S
// partials of each element in double in a fixed order and adds the rounded total into dW: the result does not depend
// on which CTA finishes first.
#include "common.cuh"

#include <mutex>

namespace b2y {

struct WgradParams {
    int Cout, Cin;
    int ntaps, ksize;
    int K_total;              // B*Ho*Wo output pixels
    int MH, MW;               // Ho, Wo
    int stride, pad;
    int m_tiles, n_tiles, ksplits;
    int ksteps_total;         // ceil(K_total / BK)
    int ksteps_per_split;
    float scale;              // multiplies the accumulator (1 / loss-scale)
    int ab_bf16;              // both operands bf16 (else fp16; wgmma takes one 16-bit format for A and B)
    const float* scale_ptr;   // optional device scalar multiplied into `scale` (per-layer gradient un-scaling)
    float* out;               // ksplits == 1: dw (+=); else the workspace (stream_ws), slice s at out + s * slice
    long long slice;          // Cout * k * k * Cin: one slice, laid out as dw [Cout][k][k][Cin]
};

template <int BLOCK_N, int NB_ROW_BYTES>
struct WgradCfg {
    static constexpr int BK = 64;                                   // pixels per pipeline stage
    static constexpr int A_ATOMS = 2;                               // 2 x 64 output channels = M 128
    static constexpr int A_ATOM_BYTES = BK * 128;
    static constexpr int B_ATOM_CH = NB_ROW_BYTES / 2;              // channels per B atom
    static constexpr int B_ATOMS = BLOCK_N / B_ATOM_CH;
    static constexpr int B_ATOM_BYTES = BK * NB_ROW_BYTES;
    static constexpr int A_BYTES = A_ATOMS * A_ATOM_BYTES;          // 16 KB
    static constexpr int B_BYTES = B_ATOMS * B_ATOM_BYTES;
    static constexpr int STAGE_BYTES = A_BYTES + ((B_BYTES + 1023) / 1024) * 1024;
    static constexpr int NUM_STAGES_RAW = (225 * 1024) / STAGE_BYTES;
    static constexpr int NUM_STAGES = NUM_STAGES_RAW > 6 ? 6 : NUM_STAGES_RAW;
    static constexpr int SMEM_BYTES = 1024 + NUM_STAGES * STAGE_BYTES + 1024;
};

// warp 0: TMA producer; warps 4-11: two consumer warpgroups, warpgroup g owns output channels 64 g .. 64 g + 63 of the
// tile (A atom g) and writes its accumulator fragment straight from registers (into dW or its workspace slice).
template <int BLOCK_N, int NB_ROW_BYTES>
__global__ void __launch_bounds__(384, 1)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap tmDy, const __grid_constant__ CUtensorMap tmX,
                const WgradParams p) {
    using Cfg = WgradCfg<BLOCK_N, NB_ROW_BYTES>;
    constexpr int NS = Cfg::NUM_STAGES;
    constexpr int BK = Cfg::BK;
    constexpr int CONSUMER_WARPS = 8;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* aux = smem + NS * Cfg::STAGE_BYTES;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(aux);
    uint64_t* empty_bar = full_bar + NS;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == 0 && lane == 0) {
        prefetch_tmap(&tmDy);
        prefetch_tmap(&tmX);
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < NS; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], CONSUMER_WARPS);
        }
        fence_barrier_init();
    }
    __syncthreads();

    const int num_tiles = p.m_tiles * p.n_tiles * p.ntaps * p.ksplits;

    // tile -> (m_tile, n_tile, tap, split); split fastest so CTAs working on the same dW tile run concurrently
    auto decode = [&](int tile, int& m_tile, int& n_tile, int& tap, int& split) {
        split = tile % p.ksplits;
        int t = tile / p.ksplits;
        tap = t % p.ntaps;
        t /= p.ntaps;
        n_tile = t % p.n_tiles;
        m_tile = t / p.n_tiles;
    };

    // The issue loop runs warp-uniform with one elected lane issuing (same reason as in conv_tc.cuh).
    if (warp == 0) {
        uint32_t stage = 0;
        uint32_t phase = 0;
        const int HoWo = p.MH * p.MW;
        const uint32_t smem_base = smem_u32(smem), full_base = smem_u32(full_bar), empty_base = smem_u32(empty_bar);
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            int m_tile, n_tile, tap, split;
            decode(tile, m_tile, n_tile, tap, split);
            const int r = tap / p.ksize, s = tap - r * p.ksize;
            const int ks0 = split * p.ksteps_per_split;
            const int ks1 = min(ks0 + p.ksteps_per_split, p.ksteps_total);
            // pixel coordinates of the k-step, advanced incrementally (BK pixels per step)
            int k0 = ks0 * BK;
            int img = k0 / HoWo;
            int rem = k0 - img * HoWo;
            for (int ks = ks0; ks < ks1; ++ks) {
                const int po = rem / p.MW, qo = rem - po * p.MW;
                mbar_wait_s(empty_base + stage * 8, phase ^ 1);
                if (elect_one()) {
                    const uint32_t a_dst = smem_base + stage * Cfg::STAGE_BYTES;
                    const uint32_t b_dst = a_dst + Cfg::A_BYTES;
                    const uint32_t fb = full_base + stage * 8;
                    mbar_expect_tx_s(fb, Cfg::A_BYTES + Cfg::B_BYTES);
#pragma unroll
                    for (int at = 0; at < Cfg::A_ATOMS; ++at)
                        tma_load_2d_s(a_dst + at * Cfg::A_ATOM_BYTES, &tmDy, fb, m_tile * 128 + at * 64, k0);
#pragma unroll
                    for (int at = 0; at < Cfg::B_ATOMS; ++at)
                        tma_load_im2col_4d_s(b_dst + at * Cfg::B_ATOM_BYTES, &tmX, fb,
                                             n_tile * BLOCK_N + at * Cfg::B_ATOM_CH, qo * p.stride - p.pad,
                                             po * p.stride - p.pad, img, (uint16_t)s, (uint16_t)r);
                }
                k0 += BK;
                rem += BK;
                if (rem >= HoWo) {      // BK <= HoWo is not guaranteed for tiny maps: general wrap
                    img += rem / HoWo;
                    rem = rem % HoWo;
                }
                if (++stage == NS) {
                    stage = 0;
                    phase ^= 1;
                }
            }
        }
    } else if (warp >= 4) {
        const int wg = (warp - 4) >> 2;
        const int tid_wg = (int)threadIdx.x & 127;
        const bool bf16 = p.ab_bf16 != 0;
        uint32_t stage = 0, phase = 0;
        // MN-major canonical layouts: LBO = distance between MN atoms, SBO = 8 K-rows
        const uint64_t adesc_base = smem_desc_base(Cfg::A_ATOM_BYTES, 8 * 128, swizzle_layout_type(128));
        const uint64_t bdesc_base =
            smem_desc_base(Cfg::B_ATOM_BYTES, 8 * NB_ROW_BYTES, swizzle_layout_type(NB_ROW_BYTES));
        const float wscale = p.scale * (p.scale_ptr != nullptr ? __ldg(p.scale_ptr) : 1.f);
        const uint32_t full_base = smem_u32(full_bar), empty_base = smem_u32(empty_bar);
        // this thread's fragment coordinates (see wgmma.cuh)
        const int frow = 64 * wg + 16 * (tid_wg >> 5) + ((tid_wg & 31) >> 2);
        const int fcol = 2 * (tid_wg & 3);
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            int m_tile, n_tile, tap, split;
            decode(tile, m_tile, n_tile, tap, split);
            const int ks0 = split * p.ksteps_per_split;
            const int ks1 = min(ks0 + p.ksteps_per_split, p.ksteps_total);
            if (ks0 >= ks1) continue;
            float acc[BLOCK_N / 2];
            uint32_t prev = 0;
            for (int ks = ks0; ks < ks1; ++ks) {
                mbar_wait_s(full_base + stage * 8, phase);
                const uint32_t a_addr = smem_u32(smem + stage * Cfg::STAGE_BYTES) + wg * Cfg::A_ATOM_BYTES;
                const uint32_t b_addr = smem_u32(smem + stage * Cfg::STAGE_BYTES) + Cfg::A_BYTES;
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / 16; ++k) {
                    const uint64_t adesc = smem_desc_at(adesc_base, a_addr + k * 16 * 128);
                    const uint64_t bdesc = smem_desc_at(bdesc_base, b_addr + k * 16 * NB_ROW_BYTES);
                    const uint32_t sc = (ks > ks0 || k > 0) ? 1u : 0u;
                    if (bf16)
                        wgmma_ss<BLOCK_N, 1, 1>(acc, adesc, bdesc, sc);
                    else
                        wgmma_ss<BLOCK_N, 0, 1>(acc, adesc, bdesc, sc);
                }
                wgmma_commit();
                if (ks > ks0) {
                    wgmma_wait<1>();
                    if (lane == 0) mbar_arrive(&empty_bar[prev]);
                }
                prev = stage;
                if (++stage == NS) {
                    stage = 0;
                    phase ^= 1;
                }
            }
            wgmma_wait<0>();
            wgmma_fence_acc(acc);
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
            // fp32 partial sums -> [co][tap][ci] of dW or of the slice, two adjacent channels per thread (__fmul_rn: the
            // product is rounded before it is added, whichever path takes it)
            float* const out = p.out + split * p.slice;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int co = m_tile * 128 + frow + 8 * h;
                if (co >= p.Cout) continue;
                float* orow = out + ((long long)co * p.ntaps + tap) * p.Cin;
#pragma unroll
                for (int i = 0; i < BLOCK_N / 8; ++i) {
                    const int ci = n_tile * BLOCK_N + 8 * i + fcol;
                    if (ci < p.Cin) {
                        const float v0 = __fmul_rn(acc[4 * i + 2 * h], wscale);
                        const float v1 = __fmul_rn(acc[4 * i + 2 * h + 1], wscale);
                        if (p.ksplits == 1) {
                            orow[ci] += v0;
                            orow[ci + 1] += v1;
                        } else {
                            *reinterpret_cast<float2*>(orow + ci) = make_float2(v0, v1);
                        }
                    }
                }
            }
        }
    }
}

// ---- narrow-input 3x3 layers (Cin = 32 / 64) -----------------------------------------------------------------
// The kernel above re-reads dY once per filter tap and feeds the tensor core N = Cin <= 64 columns.  Here the GEMM is
// transposed:
//
//   dW^T[(tap, ci)][co] = sum_{pixel m} X[m @ tap][ci] * dY[m][co]
//
// A = X: the nine im2col boxes [64 pixels][Cin] of one k-step sit back to back in smem; 128 / Cin consecutive boxes
//        are one MN-major M = 128 operand (LBO = box size), so the 9 taps are GROUPS = 3 (Cin 32) or 5 (Cin 64) groups;
// B = dY: one [64 pixels][BLOCK_N] tile per k-step, loaded ONCE and shared by all taps.
// Warpgroup w of the two consumer warpgroups owns rows 64 w .. 64 w + 63 of every group, with one register accumulator
// per group (BLOCK_N = 64 for Cin 32, 32 for Cin 64: 96 / 80 accumulator registers per thread).  The last group's
// missing taps read whatever follows in smem (the allocation is padded): garbage rows of D that are never stored.
// Work = n_tiles x split-K slices (~ one per SM); D rows are (tap, ci), columns co.
template <int ROW_BYTES, int BLOCK_N>
struct WgradTCfg {
    static constexpr int BK = 64;
    static constexpr int CIN = ROW_BYTES / 2;
    static constexpr int NTAPS = 9;
    static constexpr int TPG = 128 / CIN;
    static constexpr int GROUPS = (NTAPS + TPG - 1) / TPG;
    static constexpr int X_ATOM_BYTES = BK * ROW_BYTES;
    static constexpr int DY_ROW = BLOCK_N >= 64 ? 128 : BLOCK_N * 2;   // swizzle span of the dY tile
    static constexpr int DY_ATOM_CO = DY_ROW / 2;
    static constexpr int DY_ATOMS = BLOCK_N / DY_ATOM_CO;
    static constexpr int DY_BYTES = DY_ATOMS * BK * DY_ROW;
    static constexpr int STAGE_BYTES = DY_BYTES + NTAPS * X_ATOM_BYTES;
    static constexpr int PAD_BYTES = (GROUPS * TPG - NTAPS) * X_ATOM_BYTES;
    static constexpr int NUM_STAGES_RAW = (223 * 1024 - PAD_BYTES) / STAGE_BYTES;
    static constexpr int NUM_STAGES = NUM_STAGES_RAW > 6 ? 6 : NUM_STAGES_RAW;
    static constexpr int SMEM_BYTES = 1024 + NUM_STAGES * STAGE_BYTES + PAD_BYTES + 1024;
    static_assert(STAGE_BYTES % 1024 == 0, "stage alignment");
    static_assert(NUM_STAGES >= 2, "pipeline depth");
};

template <int ROW_BYTES, int BLOCK_N, int BF16>
__global__ void __launch_bounds__(384, 1)
wgrad_taps_kernel(const __grid_constant__ CUtensorMap tmDy, const __grid_constant__ CUtensorMap tmX,
                  const WgradParams p) {
    using Cfg = WgradTCfg<ROW_BYTES, BLOCK_N>;
    constexpr int NS = Cfg::NUM_STAGES;
    constexpr int BK = Cfg::BK;
    constexpr int CONSUMER_WARPS = 8;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* aux = smem + NS * Cfg::STAGE_BYTES + Cfg::PAD_BYTES;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(aux);
    uint64_t* empty_bar = full_bar + NS;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == 0 && lane == 0) {
        prefetch_tmap(&tmDy);
        prefetch_tmap(&tmX);
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < NS; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], CONSUMER_WARPS);
        }
        fence_barrier_init();
    }
    __syncthreads();

    const int num_items = p.n_tiles * p.ksplits;      // item -> (n_tile, split), split fastest
    const uint32_t smem_base = smem_u32(smem), full_base = smem_u32(full_bar), empty_base = smem_u32(empty_bar);

    if (warp == 0) {
        uint32_t stage = 0, phase = 0;
        const int HoWo = p.MH * p.MW;
        for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
            const int split = item % p.ksplits, n_tile = item / p.ksplits;
            const int ks0 = split * p.ksteps_per_split;
            const int ks1 = min(ks0 + p.ksteps_per_split, p.ksteps_total);
            int k0 = ks0 * BK;
            int img = k0 / HoWo;
            int rem = k0 - img * HoWo;
            for (int ks = ks0; ks < ks1; ++ks) {
                const int po = rem / p.MW, qo = rem - po * p.MW;
                mbar_wait_s(empty_base + stage * 8, phase ^ 1);
                if (elect_one()) {
                    const uint32_t dy_dst = smem_base + stage * Cfg::STAGE_BYTES;
                    const uint32_t x_dst = dy_dst + Cfg::DY_BYTES;
                    const uint32_t fb = full_base + stage * 8;
                    mbar_expect_tx_s(fb, Cfg::STAGE_BYTES);
#pragma unroll
                    for (int at = 0; at < Cfg::DY_ATOMS; ++at)
                        tma_load_2d_s(dy_dst + at * (BK * Cfg::DY_ROW), &tmDy, fb, n_tile * BLOCK_N + at * Cfg::DY_ATOM_CO,
                                      k0);
#pragma unroll
                    for (int tap = 0; tap < Cfg::NTAPS; ++tap)
                        tma_load_im2col_4d_s(x_dst + tap * Cfg::X_ATOM_BYTES, &tmX, fb, 0, qo * p.stride - p.pad,
                                             po * p.stride - p.pad, img, (uint16_t)(tap % 3), (uint16_t)(tap / 3));
                }
                k0 += BK;
                rem += BK;
                if (rem >= HoWo) {
                    img += rem / HoWo;
                    rem = rem % HoWo;
                }
                if (++stage == NS) {
                    stage = 0;
                    phase ^= 1;
                }
            }
        }
    } else if (warp >= 4) {
        const int wg = (warp - 4) >> 2;
        const int tid_wg = (int)threadIdx.x & 127;
        uint32_t stage = 0, phase = 0;
        const uint64_t adesc_base =
            smem_desc_base(Cfg::X_ATOM_BYTES, 8 * ROW_BYTES, swizzle_layout_type(ROW_BYTES));
        const uint64_t bdesc_base = smem_desc_base(BK * Cfg::DY_ROW, 8 * Cfg::DY_ROW, swizzle_layout_type(Cfg::DY_ROW));
        const float wscale = p.scale * (p.scale_ptr != nullptr ? __ldg(p.scale_ptr) : 1.f);
        // this thread's fragment rows (see wgmma.cuh): M index 64 wg + frow (+ 8), columns fcol (+ 1) + 8 i
        const int frow = 16 * (tid_wg >> 5) + ((tid_wg & 31) >> 2);
        const int fcol = 2 * (tid_wg & 3);
        for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
            const int split = item % p.ksplits, n_tile = item / p.ksplits;
            const int ks0 = split * p.ksteps_per_split;
            const int ks1 = min(ks0 + p.ksteps_per_split, p.ksteps_total);
            if (ks0 >= ks1) continue;
            float acc[Cfg::GROUPS][BLOCK_N / 2];
            uint32_t prev = 0;
            for (int ks = ks0; ks < ks1; ++ks) {
                mbar_wait_s(full_base + stage * 8, phase);
                const uint32_t dy_addr = smem_base + stage * Cfg::STAGE_BYTES;
                const uint32_t x_addr = dy_addr + Cfg::DY_BYTES + (uint32_t)(wg * (64 / Cfg::CIN) * Cfg::X_ATOM_BYTES);
                wgmma_fence();
#pragma unroll
                for (int g = 0; g < Cfg::GROUPS; ++g) {
#pragma unroll
                    for (int k = 0; k < BK / 16; ++k) {
                        const uint64_t adesc = smem_desc_at(
                            adesc_base, x_addr + g * Cfg::TPG * Cfg::X_ATOM_BYTES + k * 16 * ROW_BYTES);
                        const uint64_t bdesc = smem_desc_at(bdesc_base, dy_addr + k * 16 * Cfg::DY_ROW);
                        const uint32_t sc = (ks > ks0 || k > 0) ? 1u : 0u;
                        wgmma_ss<BLOCK_N, BF16, 1>(acc[g], adesc, bdesc, sc);
                    }
                }
                wgmma_commit();
                if (ks > ks0) {
                    wgmma_wait<1>();
                    if (lane == 0) mbar_arrive(&empty_bar[prev]);
                }
                prev = stage;
                if (++stage == NS) {
                    stage = 0;
                    phase ^= 1;
                }
            }
            wgmma_wait<0>();
#pragma unroll
            for (int g = 0; g < Cfg::GROUPS; ++g) wgmma_fence_acc(acc[g]);
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
            // D[(tap, ci)][co] -> [co][tap][ci] of dW or of the slice: the 8 lanes of a fragment row hold 8 consecutive
            // ci, so every store instruction writes whole 32-byte sectors
            float* const out = p.out + split * p.slice;
#pragma unroll
            for (int g = 0; g < Cfg::GROUPS; ++g) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int m = 64 * wg + frow + 8 * h;
                    const int tap = g * Cfg::TPG + m / Cfg::CIN, ci = m % Cfg::CIN;
                    if (tap >= Cfg::NTAPS) continue;
#pragma unroll
                    for (int i = 0; i < BLOCK_N / 8; ++i) {
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int co = n_tile * BLOCK_N + 8 * i + fcol + e;
                            if (co >= p.Cout) continue;
                            float* o = out + ((long long)co * Cfg::NTAPS + tap) * p.Cin + ci;
                            const float v = __fmul_rn(acc[g][4 * i + 2 * h + e], wscale);
                            if (p.ksplits == 1)
                                *o += v;
                            else
                                *o = v;
                        }
                    }
                }
            }
        }
    }
}

// ---- fixed-order split-K reduction -----------------------------------------------------------------------------
// dw[i] += (float) sum_{s < S} (double) ws[s * n + i].  A block is VB = 256 / G float4 columns x G groups of slices:
// group g sums its contiguous slice range in ascending order, then group 0 adds the G partial sums in ascending g.  The
// order is fixed by (S, G) alone, and while the double sum is exact (common.cuh) the result equals that of any other
// order.  G > 1 keeps the serial chain per thread short for the layers with hundreds of slices but few dW elements.
__global__ void __launch_bounds__(256)
wgrad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ dw, long long n, int S, int G, int dw_vec) {
    __shared__ double part[256][4];
    pdl_wait();
    const int VB = 256 / G;
    const int v = (int)threadIdx.x % VB, g = (int)threadIdx.x / VB;
    const long long i = ((long long)blockIdx.x * VB + v) * 4;
    const int per = (S + G - 1) / G;
    const int s0 = g * per, s1 = min(S, s0 + per);
    double a[4] = {0.0, 0.0, 0.0, 0.0};
    if (i < n) {
        const float* src = ws + i;
#pragma unroll 4
        for (int s = s0; s < s1; ++s) {
            const float4 t = *reinterpret_cast<const float4*>(src + s * n);
            a[0] += t.x;
            a[1] += t.y;
            a[2] += t.z;
            a[3] += t.w;
        }
    }
    if (G > 1) {
#pragma unroll
        for (int k = 0; k < 4; ++k) part[threadIdx.x][k] = a[k];
        __syncthreads();
        if (g != 0) return;
        for (int q = 1; q < G; ++q)
#pragma unroll
            for (int k = 0; k < 4; ++k) a[k] += part[q * VB + v][k];
    }
    if (i >= n) return;
    if (dw_vec) {
        float4* d = reinterpret_cast<float4*>(dw + i);
        float4 t = *d;
        t.x += (float)a[0];
        t.y += (float)a[1];
        t.z += (float)a[2];
        t.w += (float)a[3];
        *d = t;
    } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) dw[i + k] += (float)a[k];
    }
}

// n % 4 == 0 (Cin is a multiple of 16), so every slice starts 16-byte aligned
static int wgrad_reduce(const float* ws, float* dw, long long n, int S, cudaStream_t st) {
    int G = 1;
    while (G < 32 && (S + G - 1) / G > 16) G *= 2;
    const long long cols = 256 / G;
    const long long grid = (n / 4 + cols - 1) / cols;
    const int dw_vec = (reinterpret_cast<uintptr_t>(dw) & 15) == 0 ? 1 : 0;
    B2Y_CUDA_CHECK(launch_pdl(wgrad_reduce_kernel, dim3((unsigned)grid), dim3(256), 0, st, ws, dw, n, S, G, dw_vec));
    return B2Y_OK;
}

// ---- host ------------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*PFN_encodeIm2col)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t,
                                     const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                     CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled w_encodeTiled = nullptr;
static PFN_encodeIm2col w_encodeIm2col = nullptr;
static int w_driver_version = 0;
static int w_num_sms = 132;
static std::once_flag w_once;

static void w_resolve() {
    cudaDriverEntryPointQueryResult q;
    void* fn = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
        w_encodeTiled = reinterpret_cast<PFN_encodeTiled>(fn);
    fn = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
        w_encodeIm2col = reinterpret_cast<PFN_encodeIm2col>(fn);
    cudaDriverGetVersion(&w_driver_version);
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) ==
                                                  cudaSuccess && n > 0)
        w_num_sms = n;
}

template <int BLOCK_N, int NB_ROW_BYTES>
static int wgrad_launch_cfg(const CUtensorMap& a, const CUtensorMap& b, const WgradParams& p, cudaStream_t st) {
    using Cfg = WgradCfg<BLOCK_N, NB_ROW_BYTES>;
    auto kern = wgrad_tc_kernel<BLOCK_N, NB_ROW_BYTES>;
    static unsigned long long attr_set = 0;      // one bit per device: the attribute is per (function, device)
    if (b2y_first_use_on_device(attr_set)) {
        B2Y_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    }
    const int tiles = p.m_tiles * p.n_tiles * p.ntaps * p.ksplits;
    const int grid = tiles < w_num_sms ? tiles : w_num_sms;
    kern<<<grid, 384, Cfg::SMEM_BYTES, st>>>(a, b, p);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

template <int ROW_BYTES, int BLOCK_N>
static int wgrad_taps_launch(const CUtensorMap& a, const CUtensorMap& b, const WgradParams& p, cudaStream_t st) {
    using Cfg = WgradTCfg<ROW_BYTES, BLOCK_N>;
    auto kern = p.ab_bf16 ? wgrad_taps_kernel<ROW_BYTES, BLOCK_N, 1> : wgrad_taps_kernel<ROW_BYTES, BLOCK_N, 0>;
    static unsigned long long attr_set[2] = {0, 0};
    if (b2y_first_use_on_device(attr_set[p.ab_bf16 ? 1 : 0])) {
        B2Y_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    }
    const int items = p.n_tiles * p.ksplits;
    const int grid = items < w_num_sms ? items : w_num_sms;
    kern<<<grid, 384, Cfg::SMEM_BYTES, st>>>(a, b, p);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

}  // namespace b2y

using namespace b2y;

extern "C" int b2y_conv2d_bwd_weight(const b2y_conv_desc* d, const void* x, const void* dy, float* dw, float scale,
                                     int operand_dtype, const float* inv_scale_ptr, void* stream) {
    const int grad_dtype = operand_dtype;   // X and dY share one 16-bit format
    std::call_once(w_once, w_resolve);
    if (!d || !x || !dy || !dw) return B2Y_ERR_INVALID;
    if (!w_encodeTiled || !w_encodeIm2col) return B2Y_ERR_DRIVER;
    if (d->ksize * d->ksize > 16 || d->in_c % 16 != 0) return B2Y_ERR_UNSUPPORTED;
    if ((d->in_pitch * 2) % 16 != 0 || (d->out_pitch * 2) % 16 != 0) return B2Y_ERR_INVALID;
    const int Ho = (d->in_h + 2 * d->pad - d->ksize) / d->stride + 1;
    const int Wo = (d->in_w + 2 * d->pad - d->ksize) / d->stride + 1;
    if (Ho != d->out_h || Wo != d->out_w) return B2Y_ERR_INVALID;
    const long long K = (long long)d->batch * Ho * Wo;
    if (K > 0x7fffff00LL) return B2Y_ERR_UNSUPPORTED;

    int block_n, row_bytes;
    if (d->in_c % 64 == 0) {
        row_bytes = 128;
        // at most 128 columns: the fp32 fragment of a 64 x 128 wgmma is 64 registers per thread
        block_n = d->in_c >= 128 ? 128 : 64;
        if (d->in_c % block_n != 0 && d->in_c > block_n) block_n = 64;  // e.g. Cin = 192/320: 64-wide tiles
    } else if (d->in_c % 32 == 0) {
        row_bytes = 64;
        block_n = 32;
    } else {
        row_bytes = 32;
        block_n = 16;
    }

    WgradParams p{};
    p.Cout = d->out_c;
    p.Cin = d->in_c;
    p.ksize = d->ksize;
    p.ntaps = d->ksize * d->ksize;
    p.K_total = (int)K;
    p.MH = Ho;
    p.MW = Wo;
    p.stride = d->stride;
    p.pad = d->pad;
    p.m_tiles = (d->out_c + 127) / 128;
    p.n_tiles = (d->in_c + block_n - 1) / block_n;
    p.ksteps_total = (int)((K + 63) / 64);
    const int base_tiles = p.m_tiles * p.n_tiles * p.ntaps;
    int splits = (2 * w_num_sms + base_tiles - 1) / base_tiles;     // aim for ~2 waves of CTAs
    int max_splits = p.ksteps_total / 8;                             // keep >= 8 k-steps per slice
    if (max_splits < 1) max_splits = 1;
    if (splits > max_splits) splits = max_splits;
    if (splits < 1) splits = 1;
    p.ksteps_per_split = (p.ksteps_total + splits - 1) / splits;
    p.ksplits = (p.ksteps_total + p.ksteps_per_split - 1) / p.ksteps_per_split;
    p.scale = scale;
    p.slice = (long long)d->out_c * p.ntaps * d->in_c;
    p.ab_bf16 = grad_dtype == B2Y_DT_BF16 ? 1 : 0;
    p.scale_ptr = inv_scale_ptr;

    CUtensorMap tmDy, tmX;
    {
        cuuint64_t gdim[2] = {(cuuint64_t)d->out_c, (cuuint64_t)K};
        cuuint64_t gstride[1] = {(cuuint64_t)(d->out_pitch * 2)};
        cuuint32_t box[2] = {64, 64};
        cuuint32_t estr[2] = {1, 1};
        if (w_encodeTiled(&tmDy, grad_dtype == B2Y_DT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                           : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(dy), gdim, gstride, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
            return B2Y_ERR_DRIVER;
    }
    {
        cuuint64_t gdim[4] = {(cuuint64_t)d->in_c, (cuuint64_t)d->in_w, (cuuint64_t)d->in_h, (cuuint64_t)d->batch};
        cuuint64_t gstride[3] = {(cuuint64_t)(d->in_pitch * 2), (cuuint64_t)(d->in_pitch * 2 * d->in_w),
                                 (cuuint64_t)(d->in_pitch * 2 * d->in_w * (long long)d->in_h)};
        int lower[2] = {-d->pad, -d->pad};
        int upper[2] = {d->pad - (d->ksize - 1), d->pad - (d->ksize - 1)};
        cuuint32_t estr[4] = {1, (cuuint32_t)d->stride, (cuuint32_t)d->stride, 1};
        CUtensorMapSwizzle sw = row_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                                 : (row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                                    : CU_TENSOR_MAP_SWIZZLE_32B);
        if (w_encodeIm2col(&tmX, grad_dtype == B2Y_DT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                            : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(x), gdim, gstride, lower, upper,
                           (cuuint32_t)(row_bytes / 2), 64, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
            return B2Y_ERR_DRIVER;
        if (w_driver_version <= 13010) {
            long long bytes = (long long)d->batch * d->in_h * d->in_w * d->in_pitch * 2;
            if (bytes < 131072) reinterpret_cast<uint64_t*>(&tmX)[1] &= ~(1ull << 21);
        }
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc;
    const bool taps = d->ksize == 3 && (d->in_c == 32 || d->in_c == 64);
    CUtensorMap tmDyT = tmDy;
    if (taps) {
        const int bn = d->in_c == 32 ? 64 : 32;
        if (bn < 64) {
            // a [64 pixels][32 channels] dY box, SWIZZLE_64B: the MN-major B operand of the N = 32 tiles
            cuuint64_t gdim[2] = {(cuuint64_t)d->out_c, (cuuint64_t)K};
            cuuint64_t gstride[1] = {(cuuint64_t)(d->out_pitch * 2)};
            cuuint32_t box[2] = {(cuuint32_t)bn, 64};
            cuuint32_t estr[2] = {1, 1};
            if (w_encodeTiled(&tmDyT, grad_dtype == B2Y_DT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                                : CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                              2, const_cast<void*>(dy), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                              CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
                return B2Y_ERR_DRIVER;
        }
        p.n_tiles = (d->out_c + bn - 1) / bn;
        int sp = w_num_sms / p.n_tiles;
        if (sp < 1) sp = 1;
        if (sp > p.ksteps_total) sp = p.ksteps_total;
        p.ksteps_per_split = (p.ksteps_total + sp - 1) / sp;
        p.ksplits = (p.ksteps_total + p.ksteps_per_split - 1) / p.ksteps_per_split;
    }
    p.out = p.ksplits == 1 ? dw : stream_ws(st, p.ksplits * p.slice);
    if (p.out == nullptr) return B2Y_ERR_CUDA;
    if (taps)
        rc = d->in_c == 32 ? wgrad_taps_launch<64, 64>(tmDyT, tmX, p, st) : wgrad_taps_launch<128, 32>(tmDyT, tmX, p, st);
    else if (row_bytes == 128)
        rc = block_n == 128 ? wgrad_launch_cfg<128, 128>(tmDy, tmX, p, st) : wgrad_launch_cfg<64, 128>(tmDy, tmX, p, st);
    else
        rc = row_bytes == 64 ? wgrad_launch_cfg<32, 64>(tmDy, tmX, p, st) : wgrad_launch_cfg<16, 32>(tmDy, tmX, p, st);
    if (rc != B2Y_OK) return rc;
    return p.ksplits == 1 ? B2Y_OK : wgrad_reduce(p.out, dw, p.slice, p.ksplits, st);
}

// [O][kh][kw][I] fp32 -> OIHW fp32: dst = alpha*src (+ dst when accumulate)
__global__ void unpack_wgrad_kernel(const float* __restrict__ src, float* __restrict__ dst, int O, int I, int k,
                                    float alpha, int accumulate) {
    const long long total = (long long)O * I * k * k;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        // idx enumerates the OIHW destination
        const int kw = (int)(idx % k);
        long long t = idx / k;
        const int kh = (int)(t % k);
        t /= k;
        const int i = (int)(t % I);
        const int o = (int)(t / I);
        const float v = alpha * src[(((long long)o * k + kh) * k + kw) * I + i];
        dst[idx] = accumulate ? dst[idx] + v : v;
    }
}

extern "C" int b2y_unpack_wgrad(const float* dw_packed, float* dw_oihw, int out_c, int in_c, int ksize, float alpha,
                                int accumulate, void* stream) {
    if (!dw_packed || !dw_oihw || out_c <= 0 || in_c <= 0 || ksize <= 0) return B2Y_ERR_INVALID;
    const long long total = (long long)out_c * in_c * ksize * ksize;
    int grid = (int)((total + 255) / 256);
    if (grid > 132 * 16) grid = 132 * 16;
    unpack_wgrad_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(dw_packed, dw_oihw, out_c, in_c, ksize,
                                                                               alpha, accumulate);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// dst = alpha*src + beta*dst (fp32), used to move scaled BN/bias gradients into parameter .grad buffers
__global__ void axpby_kernel(const float* __restrict__ src, float* __restrict__ dst, long long n, float alpha,
                             float beta) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x)
        dst[i] = alpha * src[i] + (beta != 0.f ? beta * dst[i] : 0.f);
}
extern "C" int b2y_axpby_f32(const float* src, float* dst, long long n, float alpha, float beta, void* stream) {
    if (!src || !dst || n < 0) return B2Y_ERR_INVALID;
    int grid = (int)((n + 255) / 256);
    if (grid < 1) grid = 1;
    if (grid > 132 * 16) grid = 132 * 16;
    axpby_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(src, dst, n, alpha, beta);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}
