// Table-driven ("multi-tensor") layout kernels of the training step: ONE launch re-packs the fp32 master weights of
// every convolution into the two fp16 operand layouts of the tensor-core kernels, ONE launch turns all packed fp32
// weight gradients back into the OIHW parameter layout.  Round 1 issued 4 small launches per layer and step for this
// (pack_weights / pack_dgrad / unpack_wgrad / axpby: ~10 % of the step, launch bound).
//
//   master   W  fp32 [O][I][k][k]                       (nn.Conv2d.weight, checkpoint layout, models.py:92-99)
//   forward  Wf fp16 [Opad][k][k][Ipad]                 (K-major B operand of the implicit GEMM, conv_tc.cuh; columns
//                                                        >= I are never written: the caller zero-fills them once)
//   dgrad    Wd fp16 [phase][I][tap][Opad]              (per output-phase slabs, conv_tc.cu enumerate_dgrad_phases)
//   wgrad    dW fp32 [Opad][k][k][Ipad] -> OIHW fp32    (wgrad_tc.cu writes the packed form with red.global.add)
//
// Work unit = a tile of 32 output channels x TI input channels x all taps, staged through shared memory so that both
// the global reads and the global writes are contiguous runs (>= 64 bytes).  b2y_layout_tile_i(k) gives TI.
#include "b200yolo.h"
#include "common.cuh"

using namespace b2y;

namespace {

constexpr int TO = 32;          // output channels per tile
constexpr int ROW = 289;        // floats per smem row (k*k*TI <= 288, +1 -> conflict-free column reads)

__host__ __device__ inline int tile_i(int k) {
    int t = 288 / (k * k);
    t -= t % 8;
    return t > 256 ? 256 : (t < 8 ? 8 : t);
}

template <typename Item>
__device__ __forceinline__ int find_item(const Item* __restrict__ items, int n, int tile) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {            // last item with tile_begin <= tile
        const int mid = (lo + hi + 1) >> 1;
        if (items[mid].tile_begin <= tile) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(256)
pack_multi_kernel(const b2y_pack_item* __restrict__ items, int n_items) {
    __shared__ float tile[TO][ROW];
    __shared__ long long tap_base[16];     // dgrad: element offset of (phase slab + tap index * Opad) per source tap
    __shared__ int tap_ntaps[16];          // dgrad: taps of that phase
    const b2y_pack_item it = items[find_item(items, n_items, blockIdx.x)];
    const int k2 = it.k * it.k, TI = tile_i(it.k);
    const int t = blockIdx.x - it.tile_begin;
    const int tiles_i = (it.I + TI - 1) / TI;
    const int o0 = (t / tiles_i) * TO, i0 = (t % tiles_i) * TI;
    const int ni = min(TI, it.I - i0);
    if (threadIdx.x < k2) {
        // phase of tap (r, s): the output phase py with (py + pad - r) % stride == 0; inside the phase taps are
        // ordered by ascending (r, s) -- same enumeration as enumerate_dgrad_phases (conv_tc.cu)
        const int st = it.stride, pad = it.pad, k = it.k;
        const int r = threadIdx.x / k, s = threadIdx.x % k;
        const int py = ((r - pad) % st + st) % st, px = ((s - pad) % st + st) % st;
        long long off = 0;
        int my_nh = 0, my_nw = 0, r_idx = 0, s_idx = 0;
        for (int qy = 0; qy < st; ++qy)
            for (int qx = 0; qx < st; ++qx) {
                const int rmin = (qy + pad) % st, smin = (qx + pad) % st;
                const int nh = rmin < k ? (k - 1 - rmin) / st + 1 : 0;
                const int nw = smin < k ? (k - 1 - smin) / st + 1 : 0;
                if (qy == py && qx == px) {
                    my_nh = nh;
                    my_nw = nw;
                    r_idx = (r - rmin) / st;
                    s_idx = (s - smin) / st;
                } else if (qy < py || (qy == py && qx < px)) {
                    off += (long long)it.I * nh * nw * it.Opad;
                }
            }
        tap_base[threadIdx.x] = off + (long long)(r_idx * my_nw + s_idx) * it.Opad;
        tap_ntaps[threadIdx.x] = my_nh * my_nw;
    }
    // Every phase below gives a WARP one tile row (or one tile column) and strides the lanes along the contiguous
    // direction of the global tensor, so there is no per-element index division (the first version of this kernel
    // spent its time on idx / run, idx % ni: ~0.38 ms per step for 64 M weights; the traffic is worth ~0.08 ms).
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // ---- load: per output channel one contiguous run of ni*k2 floats ----
    // all (<= 4 rows x 9) loads of a thread are issued before the first shared-memory store: with 4 scalar loads in flight
    // per thread the kernel was latency bound (25 KB in flight per SM)
    const int run = ni * k2;
    {
        float v[TO / 8][9];
#pragma unroll
        for (int r = 0; r < TO / 8; ++r) {
            const int o = o0 + warp + 8 * r;
            const float* src = it.w + ((long long)o * it.I + i0) * k2;
#pragma unroll
            for (int t = 0; t < 9; ++t) {
                const int j = lane + 32 * t;
                v[r][t] = (o < it.O && j < run) ? __ldg(src + j) : 0.f;
            }
        }
#pragma unroll
        for (int r = 0; r < TO / 8; ++r)
#pragma unroll
            for (int t = 0; t < 9; ++t) {
                const int j = lane + 32 * t;
                if (j < run) tile[warp + 8 * r][j] = v[r][t];
            }
    }
    __syncthreads();
    // ---- forward layout [o][tap][i]: runs of ni halves, two per lane ----
    if (it.w_fwd != nullptr) {
        __half* wf = reinterpret_cast<__half*>(it.w_fwd);
        if (it.col_map != nullptr) {
            // input column i goes to physical column col_map[i] (a channel-pruned source: its pad channels and the gaps
            // of a concat keep the zeros the caller filled the buffer with)
            for (int ol = warp; ol < TO; ol += 8) {
                const int o = o0 + ol;
                if (o >= it.Opad) break;
                for (int j = lane; j < k2 * ni; j += 32) {
                    const int tap = j / ni, il = j - tap * ni;
                    wf[((long long)o * k2 + tap) * it.Ipad + __ldg(it.col_map + i0 + il)] =
                        __float2half_rn(tile[ol][il * k2 + tap]);
                }
            }
        } else if ((ni & 1) == 0) {
            const int npair = ni >> 1;
            const int sh = (npair & (npair - 1)) == 0 ? 31 - __clz(npair) : -1;
            for (int ol = warp; ol < TO; ol += 8) {
                const int o = o0 + ol;
                if (o >= it.Opad) break;
                __half* dst = wf + (long long)o * k2 * it.Ipad + i0;
                const float* row = tile[ol];
#pragma unroll 2
                for (int j = lane; j < k2 * npair; j += 32) {
                    const int tap = sh >= 0 ? (j >> sh) : (j / npair);
                    const int il = (j - tap * npair) * 2;
                    *reinterpret_cast<__half2*>(dst + (long long)tap * it.Ipad + il) =
                        __floats2half2_rn(row[il * k2 + tap], row[(il + 1) * k2 + tap]);
                }
            }
        } else {
            for (int ol = warp; ol < TO; ol += 8) {
                const int o = o0 + ol;
                if (o >= it.Opad) break;
                for (int j = lane; j < k2 * ni; j += 32) {
                    const int tap = j / ni, il = j - tap * ni;
                    wf[((long long)o * k2 + tap) * it.Ipad + i0 + il] = __float2half_rn(tile[ol][il * k2 + tap]);
                }
            }
        }
    }
    // ---- data-gradient layout [phase][i][tap][o]: one (i, tap) column of the tile = a run of 32 output channels ----
    if (it.w_dgrad != nullptr) {
        __half* wd = reinterpret_cast<__half*>(it.w_dgrad);
        const int o = o0 + lane;
        if (o < it.Opad) {
#pragma unroll 4
            for (int q = warp; q < run; q += 8) {
                const int il = q / k2, tap = q - il * k2;           // warp-uniform
                wd[tap_base[tap] + (long long)(i0 + il) * tap_ntaps[tap] * it.Opad + o] = __float2half_rn(tile[lane][q]);
            }
        }
    }
}

__global__ void __launch_bounds__(256)
unpack_multi_kernel(const b2y_unpack_item* __restrict__ items, int n_items) {
    __shared__ float tile[TO][ROW];
    const b2y_unpack_item it = items[find_item(items, n_items, blockIdx.x)];
    const int k2 = it.k * it.k, TI = tile_i(it.k);
    const int t = blockIdx.x - it.tile_begin;
    const int tiles_i = (it.I + TI - 1) / TI;
    const int o0 = (t / tiles_i) * TO, i0 = (t % tiles_i) * TI;
    const int ni = min(TI, it.I - i0);
    const int no = min(TO, it.O - o0);
    if (no <= 0) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int sh = (ni & (ni - 1)) == 0 ? 31 - __clz(ni) : -1;
    // packed [o][tap][i]: runs of ni floats (a warp per output channel, lanes along i)
    for (int ol = warp; ol < no; ol += 8) {
        const float* src = it.src + (long long)(o0 + ol) * k2 * it.Ipad + i0;
        float* row = tile[ol];
#pragma unroll 4
        for (int j = lane; j < k2 * ni; j += 32) {
            const int tap = sh >= 0 ? (j >> sh) : (j / ni);
            const int il = j - tap * ni;
            row[il * k2 + tap] = __ldg(src + (long long)tap * it.Ipad + il);
        }
    }
    __syncthreads();
    const int run = ni * k2;
    for (int ol = warp; ol < no; ol += 8) {
        float* d = it.dst + ((long long)(o0 + ol) * it.I + i0) * k2;
        const float* row = tile[ol];
        if (it.accumulate) {
#pragma unroll 4
            for (int j = lane; j < run; j += 32) d[j] += row[j];
        } else {
#pragma unroll 4
            for (int j = lane; j < run; j += 32) d[j] = row[j];
        }
    }
}

}  // namespace

extern "C" int b2y_layout_tile_i(int ksize) { return ksize >= 1 && ksize <= 4 ? tile_i(ksize) : 0; }

extern "C" int b2y_pack_conv_weights_multi(const b2y_pack_item* items_dev, int n_items, int total_tiles, void* stream) {
    if (!items_dev || n_items <= 0 || total_tiles <= 0) return B2Y_ERR_INVALID;
    pack_multi_kernel<<<total_tiles, 256, 0, static_cast<cudaStream_t>(stream)>>>(items_dev, n_items);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_unpack_wgrad_multi(const b2y_unpack_item* items_dev, int n_items, int total_tiles, void* stream) {
    if (!items_dev || n_items <= 0 || total_tiles <= 0) return B2Y_ERR_INVALID;
    unpack_multi_kernel<<<total_tiles, 256, 0, static_cast<cudaStream_t>(stream)>>>(items_dev, n_items);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}
