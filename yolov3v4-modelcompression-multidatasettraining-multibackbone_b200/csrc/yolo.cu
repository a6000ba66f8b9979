// YOLO head: grid/anchor decode (models.py:350-437) and the detection loss with its gradient
// (utils/utils.py:254-297 bbox_iou, 368-432 compute_loss, 725-779 build_targets), all fp32, no host syncs.
#include "b200yolo.h"
#include "common.cuh"

using namespace b2y;

static inline int grid_for(long long n, int block) {
    long long g = (n + block - 1) / block;
    if (g < 1) g = 1;
    if (g > 132LL * 32) g = 132LL * 32;
    return (int)g;
}

// ------------------------------------------------------------------------------------------------
// decode: one warp per (image, pixel, anchor) = one contiguous run of `no` floats in raw, p and io; lanes stride the run,
// so every load / store instruction is one contiguous 128-byte segment and all index arithmetic is per warp.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) yolo_decode_kernel(const float* __restrict__ raw, long long raw_pitch,
                                                          float* __restrict__ p, float* __restrict__ io,
                                                          long long total_rows, long long row_offset, int B, int na,
                                                          int no, int ny, int nx, const float* __restrict__ anchors_px,
                                                          float stride) {
    const int lane = threadIdx.x & 31;
    const unsigned plane = (unsigned)(ny * nx);
    const unsigned runs = (unsigned)B * plane * (unsigned)na;          // host checks < 2^31
    const unsigned warps = (gridDim.x * blockDim.x) >> 5;
    for (unsigned run = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; run < runs; run += warps) {
        // run order = raw memory order: (b, y, x, a)
        const unsigned a = run % (unsigned)na;
        const unsigned pix = run / (unsigned)na;                        // b*plane + y*nx + x
        const unsigned b = pix / plane;
        const unsigned yx = pix - b * plane;
        const unsigned y = yx / (unsigned)nx, x = yx - y * (unsigned)nx;
        const float* src = raw + (long long)pix * raw_pitch + a * no;
        const long long prow = ((long long)b * na + a) * plane + yx;
        float* pd = p != nullptr ? p + prow * no : nullptr;
        float* iod = io != nullptr ? io + ((long long)b * total_rows + row_offset + (long long)a * plane + yx) * no : nullptr;
        const float aw = __ldg(anchors_px + a * 2) / stride, ah = __ldg(anchors_px + a * 2 + 1) / stride;   // anchor_vec
        for (int o = lane; o < no; o += 32) {
            const float v = __ldg(src + o);
            if (pd != nullptr) pd[o] = v;
            if (iod != nullptr) {
                float r;
                if (o < 2) {
                    const float g = (o == 0) ? (float)x : (float)y;  // grid[...,0]=x, grid[...,1]=y (models.py:373-374)
                    r = (sigmoid_f(v) + g) * stride;
                } else if (o < 4) {
                    r = (expf(v) * (o == 2 ? aw : ah)) * stride;     // (models.py:362, 416-417)
                } else {
                    r = sigmoid_f(v);
                }
                iod[o] = r;
            }
        }
    }
}

// Same decode, one warp per PIXEL: the na*no <= 256 raw floats of a pixel are one contiguous run, so a lane issues all of
// its (<= 8) loads before the first use -- 1 KB in flight per warp instead of 340 B -- and the (anchor, output) split of
// every element is computed once per thread instead of once per run.  Values are computed by the same expressions.
__global__ void __launch_bounds__(256) yolo_decode_pixel_kernel(const float* __restrict__ raw, long long raw_pitch,
                                                                float* __restrict__ p, float* __restrict__ io,
                                                                long long total_rows, long long row_offset, int B,
                                                                int na, int no, int ny, int nx,
                                                                const float* __restrict__ anchors_px, float stride) {
    const int lane = threadIdx.x & 31;
    const unsigned plane = (unsigned)(ny * nx);
    const unsigned pixels = (unsigned)B * plane;
    const unsigned warps = (gridDim.x * blockDim.x) >> 5;
    const int nel = na * no;
    int ea[8], eo[8];
    float ew[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int e = lane + 32 * i;
        ea[i] = e < nel ? e / no : 0;
        eo[i] = e < nel ? e - ea[i] * no : -1;
        ew[i] = 0.f;
        if (eo[i] == 2) ew[i] = __ldg(anchors_px + ea[i] * 2) / stride;          // anchor_vec
        if (eo[i] == 3) ew[i] = __ldg(anchors_px + ea[i] * 2 + 1) / stride;
    }
    for (unsigned pix = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; pix < pixels; pix += warps) {
        const unsigned b = pix / plane;
        const unsigned yx = pix - b * plane;
        const unsigned y = yx / (unsigned)nx, x = yx - y * (unsigned)nx;
        const float* src = raw + (long long)pix * raw_pitch;
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = eo[i] >= 0 ? __ldg(src + lane + 32 * i) : 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int o = eo[i];
            if (o < 0) continue;
            const long long prow = ((long long)b * na + ea[i]) * plane + yx;
            if (p != nullptr) p[prow * no + o] = v[i];
            if (io != nullptr) {
                float r;
                if (o < 2) {
                    const float g = (o == 0) ? (float)x : (float)y;
                    r = (sigmoid_f(v[i]) + g) * stride;
                } else if (o < 4) {
                    r = (expf(v[i]) * ew[i]) * stride;
                } else {
                    r = sigmoid_f(v[i]);
                }
                io[((long long)b * total_rows + row_offset + (long long)ea[i] * plane + yx) * no + o] = r;
            }
        }
    }
}

extern "C" int b2y_yolo_decode(const float* raw, long long raw_pitch, float* p, float* io, long long total_rows,
                               long long row_offset, int batch, int na, int no, int ny, int nx,
                               const float* anchors_px, float stride, void* stream) {
    if (!raw || !anchors_px || batch <= 0 || na <= 0 || no < 5 || ny <= 0 || nx <= 0) return B2Y_ERR_INVALID;
    if (raw_pitch < (long long)na * no) return B2Y_ERR_INVALID;
    const long long runs = (long long)batch * na * ny * nx;
    if (runs > 0x7fffffffLL) return B2Y_ERR_UNSUPPORTED;
    if (na * no <= 256) {
        const long long pixels = (long long)batch * ny * nx;
        long long pb = (pixels + 7) / 8;
        if (pb > 132 * 8) pb = 132 * 8;
        yolo_decode_pixel_kernel<<<(int)pb, 256, 0, static_cast<cudaStream_t>(stream)>>>(
            raw, raw_pitch, p, io, total_rows, row_offset, batch, na, no, ny, nx, anchors_px, stride);
        B2Y_CUDA_CHECK(cudaGetLastError());
        return B2Y_OK;
    }
    long long blocks = (runs + 7) / 8;                 // 8 warps per block
    if (blocks > 132 * 16) blocks = 132 * 16;
    yolo_decode_kernel<<<(int)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        raw, raw_pitch, p, io, total_rows, row_offset, batch, na, no, ny, nx, anchors_px, stride);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// ------------------------------------------------------------------------------------------------
// target assignment helpers
// ------------------------------------------------------------------------------------------------
struct Match {
    int ok;
    int b, c, gi, gj;
    float tx, ty, tw, th;  // tbox: (frac x, frac y, w, h) in grid units
};

// A candidate whose image index b lies outside [0, B) or whose cell (gi, gj) lies off the grid (x or y == 1.0 after
// the .long() truncation, a negative image index) is dropped, by the loss and by build_targets alike: the reference
// would raise an IndexError at pi[b, a, gj, gi], and writing or reading such a cell here would go out of bounds.
__device__ __forceinline__ Match match_candidate(const float* __restrict__ targets, const float* __restrict__ anchors,
                                                 int a, int j, int B, int nx, int ny, float iou_t) {
    Match m;
    const float* t = targets + (long long)j * 6;
    // t = targets * gain, gain = (1,1,nx,ny,nx,ny)  (utils.py:742-743)
    const float gx = t[2] * (float)nx, gy = t[3] * (float)ny;
    const float gw = t[4] * (float)nx, gh = t[5] * (float)ny;
    const float aw = anchors[a * 2], ah = anchors[a * 2 + 1];
    // wh_iou (utils.py:325-330): each prod(2) rounded on its own, as torch does.  Contracting aw*ah + gw*gh into one FMA
    // moves the denominator by an ulp, which flips the `> iou_t` decision of a candidate whose IoU sits at the threshold.
    const float inter = __fmul_rn(fminf(aw, gw), fminf(ah, gh));
    const float iou = inter / __fsub_rn(__fadd_rn(__fmul_rn(aw, ah), __fmul_rn(gw, gh)), inter);
    m.b = (int)t[0];  // .long() truncation (utils.py:761,764)
    m.c = (int)t[1];
    m.gi = (int)gx;
    m.gj = (int)gy;
    m.ok = iou > iou_t && m.b >= 0 && m.b < B && m.gi >= 0 && m.gi < nx && m.gj >= 0 && m.gj < ny;
    m.tx = gx - floorf(gx);
    m.ty = gy - floorf(gy);
    m.tw = gw;
    m.th = gh;
    return m;
}

// GIoU of predicted box (from logits) vs target box, plus d(giou)/d(logits[0..3]).
__device__ __forceinline__ float giou_fwd_bwd(const float* __restrict__ ps, float aw, float ah, const Match& m,
                                              float* dgi /*[4] or null*/) {
    const float sx = sigmoid_f(ps[0]), sy = sigmoid_f(ps[1]);
    const float ew = expf(ps[2]), eh = expf(ps[3]);
    const float cwv = fminf(ew, 1e3f), chv = fminf(eh, 1e3f);  // .clamp(max=1E3) (utils.py:400)
    const float pw = cwv * aw, ph = chv * ah;
    // xywh -> xyxy (utils.py:263-266)
    const float b1x1 = sx - pw / 2, b1x2 = sx + pw / 2, b1y1 = sy - ph / 2, b1y2 = sy + ph / 2;
    const float b2x1 = m.tx - m.tw / 2, b2x2 = m.tx + m.tw / 2, b2y1 = m.ty - m.th / 2, b2y2 = m.ty + m.th / 2;
    const float iw_raw = fminf(b1x2, b2x2) - fmaxf(b1x1, b2x1);
    const float ih_raw = fminf(b1y2, b2y2) - fmaxf(b1y1, b2y1);
    const float iw = fmaxf(iw_raw, 0.f), ih = fmaxf(ih_raw, 0.f);
    const float inter = iw * ih;
    const float w1 = b1x2 - b1x1, h1 = b1y2 - b1y1, w2 = b2x2 - b2x1, h2 = b2y2 - b2y1;
    const float uni = (w1 * h1 + 1e-16f) + w2 * h2 - inter;
    const float iou = inter / uni;
    const float cw = fmaxf(b1x2, b2x2) - fminf(b1x1, b2x1);
    const float ch = fmaxf(b1y2, b2y2) - fminf(b1y1, b2y1);
    const float c_area = cw * ch + 1e-16f;
    const float giou = iou - (c_area - uni) / c_area;
    if (dgi != nullptr) {
        // selector derivatives of min/max (ties split 1/2, as torch.minimum/maximum do)
        auto sel_lt = [](float a, float b) { return a < b ? 1.f : (a == b ? 0.5f : 0.f); };
        const float miw = iw_raw >= 0.f ? 1.f : 0.f, mih = ih_raw >= 0.f ? 1.f : 0.f;
        // d inter / d(b1 corners)
        const float di_x2 = ih * miw * sel_lt(b1x2, b2x2);
        const float di_x1 = -ih * miw * sel_lt(b2x1, b1x1);
        const float di_y2 = iw * mih * sel_lt(b1y2, b2y2);
        const float di_y1 = -iw * mih * sel_lt(b2y1, b1y1);
        // d union
        const float du_x2 = h1 - di_x2, du_x1 = -h1 - di_x1, du_y2 = w1 - di_y2, du_y1 = -w1 - di_y1;
        // d c_area
        const float dc_x2 = sel_lt(b2x2, b1x2) * ch, dc_x1 = -sel_lt(b1x1, b2x1) * ch;
        const float dc_y2 = sel_lt(b2y2, b1y2) * cw, dc_y1 = -sel_lt(b1y1, b2y1) * cw;
        const float inv_u2 = 1.f / (uni * uni), inv_c2 = 1.f / (c_area * c_area);
        auto dg = [&](float di, float du, float dc) {
            return (di * uni - inter * du) * inv_u2 + (du * c_area - uni * dc) * inv_c2;
        };
        const float g_x1 = dg(di_x1, du_x1, dc_x1), g_x2 = dg(di_x2, du_x2, dc_x2);
        const float g_y1 = dg(di_y1, du_y1, dc_y1), g_y2 = dg(di_y2, du_y2, dc_y2);
        const float g_px = g_x1 + g_x2, g_py = g_y1 + g_y2;
        const float g_pw = 0.5f * (g_x2 - g_x1), g_ph = 0.5f * (g_y2 - g_y1);
        dgi[0] = g_px * sx * (1.f - sx);
        dgi[1] = g_py * sy * (1.f - sy);
        dgi[2] = (ew <= 1e3f) ? g_pw * aw * ew : 0.f;
        dgi[3] = (eh <= 1e3f) ? g_ph * ah * eh : 0.f;
    }
    return giou;
}

// BCEWithLogits element with pos_weight, torch's stable form:
//   (1-y)*x + (1+(pw-1)*y) * (log1p(exp(-|x|)) + max(-x,0))
__device__ __forceinline__ float bce_logits(float x, float y, float pw, float* dx) {
    const float lw = (pw - 1.f) * y + 1.f;
    const float sp = log1pf(expf(-fabsf(x))) + fmaxf(-x, 0.f);
    if (dx != nullptr) *dx = (1.f - y) - lw * (1.f - sigmoid_f(x));
    return (1.f - y) * x + lw * sp;
}

// Focal modulation of one BCE element (FocalLoss, utils/utils.py:333-360, alpha = 0.25), applied only when gamma > 0:
//   l = bce * af * m,   af = y*a + (1-y)*(1-a),   m = (1-p_t)^gamma,   p_t = y*s + (1-y)*(1-s),   s = sigmoid(x)
// The reference differentiates this with autograd; here in closed form.  With d p_t/dx = (2y-1) * s*(1-s):
//   dl/dx = af * [ bce' * m + bce * gamma * (1-p_t)^(gamma-1) * (-(2y-1) * s*(1-s)) ]
// `bce` is the element's BCE value and *dx holds bce' on entry and dl/dx on return.  y may be fractional (objectness).
// Saturated logits (s rounds to exactly 0 or 1, so 1-p_t = 0): the second term is taken as 0, its limit for x -> +-inf.
// That equals the reference's gradient for gamma >= 1; for gamma < 1 the reference's autograd gives 0 * inf = NaN there.
__device__ __forceinline__ float focal_modulate(float x, float y, float gamma, float bce, float* dx) {
    const float s = sigmoid_f(x);
    const float omp = 1.f - (y * s + (1.f - y) * (1.f - s));
    const float af = y * 0.25f + (1.f - y) * 0.75f;
    const float m = powf(omp, gamma);
    if (dx != nullptr) {
        const float dm = omp > 0.f ? gamma * powf(omp, gamma - 1.f) * (-(2.f * y - 1.f) * (s * (1.f - s))) : 0.f;
        *dx = af * (*dx * m + bce * dm);
    }
    return bce * (af * m);
}

__device__ __forceinline__ float block_sum(float v, float* sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) sh[w] = v;
    __syncthreads();
    float r = 0.f;
    if (w == 0) {
        r = (l < (int)(blockDim.x >> 5)) ? sh[l] : 0.f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
    }
    return r;  // valid in thread 0
}

// workspace layout: [0] int nb | [1..3] pad | winner int32[cells]
// K1: count matches and resolve duplicate cells ("highest list position wins" == CPU index_put order)
__global__ void loss_assign_kernel(const float* __restrict__ targets, int nt, const float* __restrict__ anchors,
                                   int B, int na, int ny, int nx, float iou_t, int* __restrict__ nb,
                                   int* __restrict__ winner) {
    const int total = na * nt;
    int local = 0;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < total; k += gridDim.x * blockDim.x) {
        const int a = k / nt, j = k - a * nt;
        const Match m = match_candidate(targets, anchors, a, j, B, nx, ny, iou_t);
        if (m.ok) {
            local++;
            const long long cell = (((long long)m.b * na + a) * ny + m.gj) * nx + m.gi;
            atomicMax(winner + cell, k);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(nb, local);
}

// K2: per-match box + class loss and their gradients (atomicAdd into dp: duplicates accumulate)
__global__ void loss_match_kernel(const float* __restrict__ p, const float* __restrict__ targets, int nt,
                                  const float* __restrict__ anchors, int B, int na, int no, int ny, int nx,
                                  float iou_t, float cls_pw, float w_box, float w_cls, float fl_gamma,
                                  const int* __restrict__ nb_ptr, float* __restrict__ out4, float* __restrict__ dp) {
    __shared__ float sh[32];
    const int total = na * nt;
    const int nb = *nb_ptr;
    const int nc = no - 5;
    float s_box = 0.f, s_cls = 0.f;
    const float inv_nb = nb > 0 ? 1.f / (float)nb : 0.f;
    const float inv_cls = (nb > 0 && nc > 0) ? 1.f / ((float)nb * (float)nc) : 0.f;
    // one WARP per (anchor, target) candidate: lane 0 does the box term, the lanes stride the class logits (a thread per
    // candidate walked its 80 classes through 80 dependent global loads: 40 us per head for ~150 candidates)
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    for (int k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; k < total; k += warps) {
        const int a = k / nt, j = k - a * nt;
        const Match m = match_candidate(targets, anchors, a, j, B, nx, ny, iou_t);
        if (!m.ok) continue;   // warp-uniform
        const long long cell = (((long long)m.b * na + a) * ny + m.gj) * nx + m.gi;
        const float* ps = p + cell * no;
        if (lane == 0) {
            float dgi[4];
            const float giou = giou_fwd_bwd(ps, anchors[a * 2], anchors[a * 2 + 1], m, dp ? dgi : nullptr);
            s_box += 1.f - giou;
            if (dp != nullptr) {
                // lbox = w_box * mean(1 - giou)
                const float g = -w_box * inv_nb;
#pragma unroll
                for (int q = 0; q < 4; ++q) atomicAdd(dp + cell * no + q, g * dgi[q]);
            }
        }
        if (nc > 1) {
            for (int c = lane; c < nc; c += 32) {
                const float y = (c == m.c) ? 1.f : 0.f;  // cp=1, cn=0 (utils.py:380)
                float dx;
                float l = bce_logits(ps[5 + c], y, cls_pw, dp ? &dx : nullptr);
                if (fl_gamma > 0.f) l = focal_modulate(ps[5 + c], y, fl_gamma, l, dp ? &dx : nullptr);
                s_cls += l;
                if (dp != nullptr) atomicAdd(dp + cell * no + 5 + c, w_cls * inv_cls * dx);
            }
        }
    }
    float r = block_sum(s_box, sh);
    if (threadIdx.x == 0 && r != 0.f) atomicAdd(out4 + 0, r);
    r = block_sum(s_cls, sh);
    if (threadIdx.x == 0 && r != 0.f) atomicAdd(out4 + 2, r);
    if (blockIdx.x == 0 && threadIdx.x == 0) out4[1] = (float)nb;
}

// K3: objectness BCE over every cell; tobj of a matched cell is recomputed from the winning candidate
__global__ void loss_obj_kernel(const float* __restrict__ p, const float* __restrict__ targets, int nt,
                                const float* __restrict__ anchors, int B, int na, int no, int ny, int nx, float iou_t,
                                float gr, float obj_pw, float w_obj, float fl_gamma, const int* __restrict__ winner,
                                float* __restrict__ out4, float* __restrict__ dp) {
    __shared__ float sh[32];
    const long long cells = (long long)B * na * ny * nx;
    const float inv_cells = 1.f / (float)cells;
    float s = 0.f;
    for (long long cell = (long long)blockIdx.x * blockDim.x + threadIdx.x; cell < cells;
         cell += (long long)gridDim.x * blockDim.x) {
        const int k = winner[cell];
        float tobj = 0.f;
        if (k >= 0) {
            const int a = k / nt, j = k - a * nt;
            const Match m = match_candidate(targets, anchors, a, j, B, nx, ny, iou_t);
            const float giou = giou_fwd_bwd(p + cell * no, anchors[a * 2], anchors[a * 2 + 1], m, nullptr);
            tobj = (1.f - gr) + gr * fmaxf(giou, 0.f);  // utils.py:407
        }
        float dx;
        float l = bce_logits(p[cell * no + 4], tobj, obj_pw, dp ? &dx : nullptr);
        if (fl_gamma > 0.f) l = focal_modulate(p[cell * no + 4], tobj, fl_gamma, l, dp ? &dx : nullptr);
        s += l;
        if (dp != nullptr) dp[cell * no + 4] = w_obj * inv_cells * dx;
    }
    const float r = block_sum(s, sh);
    if (threadIdx.x == 0) atomicAdd(out4 + 3, r);
}

extern "C" size_t b2y_yolo_loss_workspace_bytes(int batch, int na, int ny, int nx, int nt) {
    (void)nt;
    return 16 + sizeof(int) * (size_t)batch * na * ny * nx;
}

extern "C" int b2y_yolo_loss(const float* p, const float* targets, int nt, const float* anchors, int batch, int na,
                             int no, int ny, int nx, float iou_t, float gr, float cls_pw, float obj_pw, float w_box,
                             float w_obj, float w_cls, float fl_gamma, float* out4, float* dp, void* workspace,
                             void* stream) {
    if (!p || !anchors || !out4 || !workspace || batch <= 0 || na <= 0 || no < 5 || nt < 0) return B2Y_ERR_INVALID;
    if (nt > 0 && !targets) return B2Y_ERR_INVALID;
    if (!(fl_gamma >= 0.f)) return B2Y_ERR_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long cells = (long long)batch * na * ny * nx;
    int* nb = reinterpret_cast<int*>(workspace);
    int* winner = nb + 4;
    B2Y_CUDA_CHECK(cudaMemsetAsync(nb, 0, 16, st));
    B2Y_CUDA_CHECK(cudaMemsetAsync(winner, 0xFF, sizeof(int) * cells, st));
    B2Y_CUDA_CHECK(cudaMemsetAsync(out4, 0, 4 * sizeof(float), st));
    if (dp != nullptr) B2Y_CUDA_CHECK(cudaMemsetAsync(dp, 0, sizeof(float) * cells * no, st));
    if (nt > 0) {
        const int total = na * nt;
        loss_assign_kernel<<<grid_for(total, 256), 256, 0, st>>>(targets, nt, anchors, batch, na, ny, nx, iou_t, nb,
                                                                 winner);
        loss_match_kernel<<<grid_for((long long)total * 32, 128), 128, 0, st>>>(p, targets, nt, anchors, batch, na, no, ny, nx, iou_t,
                                                                cls_pw, w_box, w_cls, fl_gamma, nb, out4, dp);
    }
    loss_obj_kernel<<<grid_for(cells, 256), 256, 0, st>>>(p, targets, nt, anchors, batch, na, no, ny, nx, iou_t, gr,
                                                          obj_pw, w_obj, fl_gamma, winner, out4, dp);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

// ------------------------------------------------------------------------------------------------
// build_targets as a standalone op: ordered (anchor-major, target-minor) compaction in one CTA
// ------------------------------------------------------------------------------------------------
__global__ void build_targets_kernel(const float* __restrict__ targets, int nt, const float* __restrict__ anchors,
                                     int B, int na, int ny, int nx, float iou_t, long long* __restrict__ idx,
                                     float* __restrict__ tbox, long long* __restrict__ tcls,
                                     int* __restrict__ count) {
    __shared__ int warp_tot[32];
    __shared__ int base;
    const int total = na * nt;
    if (threadIdx.x == 0) base = 0;
    __syncthreads();
    for (int k0 = 0; k0 < total; k0 += blockDim.x) {
        const int k = k0 + threadIdx.x;
        Match m;
        m.ok = 0;
        int a = 0;
        if (k < total) {
            a = k / nt;
            m = match_candidate(targets, anchors, a, k - a * nt, B, nx, ny, iou_t);
        }
        const unsigned bal = __ballot_sync(0xffffffffu, m.ok);
        const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
        const int before = __popc(bal & ((1u << lane) - 1));
        if (lane == 0) warp_tot[w] = __popc(bal);
        __syncthreads();
        int woff = 0;
        for (int i = 0; i < w; ++i) woff += warp_tot[i];
        const int pos = base + woff + before;
        if (m.ok) {
            const long long cap = total;
            idx[0 * cap + pos] = m.b;
            idx[1 * cap + pos] = a;
            idx[2 * cap + pos] = m.gj;
            idx[3 * cap + pos] = m.gi;
            tbox[pos * 4 + 0] = m.tx;
            tbox[pos * 4 + 1] = m.ty;
            tbox[pos * 4 + 2] = m.tw;
            tbox[pos * 4 + 3] = m.th;
            tcls[pos] = m.c;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int t = 0;
            for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += warp_tot[i];
            base += t;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) *count = base;
}

extern "C" int b2y_build_targets(const float* targets, int nt, const float* anchors, int batch, int na, int ny,
                                 int nx, float iou_t, long long* idx, float* tbox, long long* tcls, int* count,
                                 void* stream) {
    if (!anchors || !idx || !tbox || !tcls || !count || nt < 0 || batch <= 0 || na <= 0) return B2Y_ERR_INVALID;
    if (nt > 0 && !targets) return B2Y_ERR_INVALID;
    build_targets_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(targets, nt, anchors, batch, na, ny, nx,
                                                                            iou_t, idx, tbox, tcls, count);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}
