// Knowledge-distillation losses of the YOLO head (SURVEY section 8 f4; utils/utils.py:435-520: compute_lost_KD, KD2, KD3),
// forward value and gradient w.r.t. the student's raw predictions in one pass each.  HBM bound: every head cell is read
// once from the student and once from the teacher, the gradient is written once.
//
//   kd_soft_rows_kernel : sum over rows of KL( softmax(t/T) || softmax(s/T) ) on `width` columns starting at `col0` of
//                         rows of `row_len` floats (KD1: the whole 5 + nc row; KD2..5: columns 4.. = objectness + classes),
//                         gradient (p - q) * grad_scale / T.  One warp per row.
//   kd_box_kernel       : the matched cells of build_targets: squared distance between the student's decoded box and the
//                         target (KD2, counted only where the student is further from the target than the teacher) or
//                         the teacher's box (KD3..5), gradient scattered into the same buffer.
#include "b200yolo.h"
#include "common.cuh"

using namespace b2y;

namespace {

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(~0u, v, o));
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(~0u, v, o);
    return v;
}

__global__ void __launch_bounds__(256) kd_soft_rows_kernel(const float* __restrict__ s, const float* __restrict__ t,
                                                           long long rows, int row_len, int col0, int width,
                                                           float inv_T, float grad_scale, double* __restrict__ loss,
                                                           float* __restrict__ ds) {
    const int lane = threadIdx.x & 31;
    const long long warps = ((long long)gridDim.x * blockDim.x) >> 5;
    double acc = 0.0;
    for (long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += warps) {
        const float* sr = s + row * row_len + col0;
        const float* tr = t + row * row_len + col0;
        float ms = -INFINITY, mt = -INFINITY;
        for (int c = lane; c < width; c += 32) {
            ms = fmaxf(ms, __ldg(sr + c) * inv_T);
            mt = fmaxf(mt, __ldg(tr + c) * inv_T);
        }
        ms = warp_max(ms);
        mt = warp_max(mt);
        float es = 0.f, et = 0.f;
        for (int c = lane; c < width; c += 32) {
            es += expf(__ldg(sr + c) * inv_T - ms);
            et += expf(__ldg(tr + c) * inv_T - mt);
        }
        es = warp_sum(es);
        et = warp_sum(et);
        const float ls = logf(es), lt = logf(et), ies = 1.f / es, iet = 1.f / et;
        float kl = 0.f;
        for (int c = lane; c < width; c += 32) {
            const float zs = __ldg(sr + c) * inv_T - ms, zt = __ldg(tr + c) * inv_T - mt;
            const float logp = zs - ls, logq = zt - lt;
            const float q = expf(zt) * iet;
            if (q > 0.f) kl += q * (logq - logp);               // KLDivLoss: xlogy(q, q) - q * input, 0 where q == 0
            if (ds != nullptr) ds[row * row_len + col0 + c] = (expf(zs) * ies - q) * grad_scale;
        }
        kl = warp_sum(kl);
        if (lane == 0) acc += (double)kl;
    }
    // one atomic per warp (double: the order of the adds does not show in the fp32 result)
    if (lane == 0 && acc != 0.0) atomicAdd(loss, acc);
}

__global__ void kd_box_kernel(const float* __restrict__ ps, const float* __restrict__ pt,
                              const long long* __restrict__ idx, const float* __restrict__ tbox,
                              const float* __restrict__ anchors, int n, int na, int ny, int nx, int no, int mode,
                              float reg_m, float grad_scale, double* __restrict__ loss, int* __restrict__ reg_num,
                              float* __restrict__ ds) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long b = idx[i], a = idx[(long long)n + i], gj = idx[2LL * n + i], gi = idx[3LL * n + i];
    const long long off = (((b * na + a) * ny + gj) * nx + gi) * no;
    const float aw = anchors[a * 2], ah = anchors[a * 2 + 1];
    const float s0 = ps[off], s1 = ps[off + 1], s2 = ps[off + 2], s3 = ps[off + 3];
    const float sx = sigmoid_f(s0), sy = sigmoid_f(s1), sw = expf(s2) * aw, sh = expf(s3) * ah;
    const float tx = sigmoid_f(pt[off]), ty = sigmoid_f(pt[off + 1]), tw = expf(pt[off + 2]) * aw,
                th = expf(pt[off + 3]) * ah;
    float rx, ry, rw, rh;                 // what the student is pulled towards
    bool on = true;
    if (mode == 2) {
        rx = tbox[i * 4]; ry = tbox[i * 4 + 1]; rw = tbox[i * 4 + 2]; rh = tbox[i * 4 + 3];
        const float l2s = (sx - rx) * (sx - rx) + (sy - ry) * (sy - ry) + (sw - rw) * (sw - rw) + (sh - rh) * (sh - rh);
        const float l2t = (tx - rx) * (tx - rx) + (ty - ry) * (ty - ry) + (tw - rw) * (tw - rw) + (th - rh) * (th - rh);
        on = (l2s + reg_m) > l2t;         // utils.py:471-474
        if (on) {
            atomicAdd(loss, (double)l2s);
            atomicAdd(reg_num, 1);
        }
    } else {
        rx = tx; ry = ty; rw = tw; rh = th;
        const float l2 = (sx - rx) * (sx - rx) + (sy - ry) * (sy - ry) + (sw - rw) * (sw - rw) + (sh - rh) * (sh - rh);
        atomicAdd(loss, (double)l2);
    }
    if (ds != nullptr && on) {            // duplicates of a cell accumulate like autograd's index backward
        atomicAdd(ds + off, 2.f * (sx - rx) * sx * (1.f - sx) * grad_scale);
        atomicAdd(ds + off + 1, 2.f * (sy - ry) * sy * (1.f - sy) * grad_scale);
        atomicAdd(ds + off + 2, 2.f * (sw - rw) * sw * grad_scale);
        atomicAdd(ds + off + 3, 2.f * (sh - rh) * sh * grad_scale);
    }
}

}  // namespace

extern "C" int b2y_kd_soft_rows(const float* student, const float* teacher, long long rows, int row_len, int col0,
                                int width, float temperature, float grad_scale, double* loss_acc, float* dstudent,
                                void* stream) {
    if (!student || !teacher || !loss_acc || rows < 0 || row_len <= 0 || col0 < 0 || width <= 0 ||
        col0 + width > row_len || !(temperature > 0.f))
        return B2Y_ERR_INVALID;
    if (rows == 0) return B2Y_OK;
    long long blocks = (rows + 7) / 8;
    if (blocks > 132LL * 16) blocks = 132LL * 16;
    kd_soft_rows_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        student, teacher, rows, row_len, col0, width, 1.f / temperature, grad_scale / temperature, loss_acc, dstudent);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_kd_box(const float* student, const float* teacher, const long long* idx, const float* tbox,
                          const float* anchor_vec, int n, int na, int ny, int nx, int no, int mode, float reg_m,
                          float grad_scale, double* loss_acc, int* reg_num, float* dstudent, void* stream) {
    if (n < 0 || na <= 0 || ny <= 0 || nx <= 0 || no < 5 || (mode != 2 && mode != 3) || !loss_acc)
        return B2Y_ERR_INVALID;
    if (n == 0) return B2Y_OK;
    if (!student || !teacher || !idx || !anchor_vec || (mode == 2 && (!tbox || !reg_num))) return B2Y_ERR_INVALID;
    kd_box_kernel<<<(n + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(
        student, teacher, idx, tbox, anchor_vec, n, na, ny, nx, no, mode, reg_m, grad_scale, loss_acc, reg_num, dstudent);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}
