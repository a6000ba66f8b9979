// Input pipeline on the device, inference slice (SURVEY section 8 f2): the reference's letterbox (utils/datasets.py:611-646:
// cv2.resize INTER_LINEAR + cv2.copyMakeBorder with colour 114) fused with the BGR -> RGB / HWC -> CHW shuffle of
// LoadImages.__next__ (datasets.py:108-118), writing straight into the uint8 NCHW batch slot that the stem kernel
// consumes (it applies the "/ 256").  The arithmetic is OpenCV's (third-party dependency of the reference, not vendored;
// this container: 4.13.0) -- restated in csrc/preprocess_core.h / oracle/preprocess_oracle.py and pinned against cv2's
// own outputs; bit-exact.  HBM / gather bound: 4 source pixels read per output pixel, one byte written per channel.
//
// b2y_load_batch_u8 builds a whole evaluation batch of LoadImagesAndLabels(rect=True) (utils/datasets.py:419-475,
// 511-531) in one table-driven launch: load_image's INTER_AREA downscale, the letterbox border (its own resize is not
// reached: the rect batch shape always holds the resized image) and the channel shuffle.  Gather bound: an output byte
// reads its source cell (about scale_x * scale_y bytes, each once from HBM and the rest from L1/L2) and does a few
// float operations per source byte; the border bytes read nothing.
//
// b2y_mosaic_u8 and b2y_affine_hsv_u8 build a training batch of LoadImagesAndLabels(augment=True) (utils/datasets.py:
// 419-501, 534-608, 649-715) in two table-driven launches: load_mosaic's 2s x 2s canvases, then per output pixel
// random_affine's warpAffine, augment_hsv, the flip and the channel shuffle.  Gather bound, like the loaders above.
#include <cmath>

#include "b200yolo.h"
#include "common.cuh"
#include "preprocess_core.h"

namespace {

__global__ void __launch_bounds__(256) letterbox_u8_kernel(const unsigned char* __restrict__ src,
                                                           unsigned char* __restrict__ dst, b2y_lb_params p) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= p.dst_w) return;
    b2y_lb_pixel(src, dst, p, x, (int)blockIdx.y);
}

// One launch for a whole evaluation batch: blockIdx.z = item, blockIdx.y = output row, threads along the row.  Each
// output byte is the border colour or the INTER_AREA value computed straight from the source (copy when the source
// already has the resized size), written to channel c of slot item.slot of the planar [B][C][H][W] batch.
__global__ void __launch_bounds__(128) load_batch_u8_kernel(const b2y_load_item* __restrict__ items,
                                                            unsigned char* __restrict__ dst, int C, int H, int W,
                                                            int swap_rb, unsigned char color) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= W) return;
    const b2y_load_item it = items[blockIdx.z];
    const long long plane = (long long)H * W;
    b2y_area_params p;
    p.src_h = it.src_h; p.src_w = it.src_w; p.channels = C; p.src_pitch = it.src_pitch;
    p.rs_h = it.rs_h; p.rs_w = it.rs_w; p.kx = it.area_kx; p.ky = it.area_ky;
    p.scale_x = it.scale_x; p.scale_y = it.scale_y;
    b2y_load_pixel(it.src, p, it.top, it.left, x, y, swap_rb, color,
                   dst + (long long)it.slot * C * plane + (long long)y * W + x, plane);
}

// Mosaic canvases: blockIdx.z = item, blockIdx.y = canvas row, threads along the row; each thread writes every channel
// of one canvas pixel (HWC).  Gather bound: a tile pixel reads 1 (copy) or 4 (INTER_LINEAR) source bytes per channel,
// the 114 fill reads nothing; the canvas bytes are written once.
__global__ void __launch_bounds__(128) mosaic_u8_kernel(const b2y_mosaic_item* __restrict__ items,
                                                        unsigned char* __restrict__ canvas, int C, int s2) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= s2) return;
    const b2y_mosaic_item& it = items[blockIdx.z];
    unsigned char* out = canvas + (((long long)it.slot * s2 + y) * s2 + x) * C;
    int k = 3;
    for (; k >= 0; --k) {
        const b2y_mosaic_tile& t = it.tiles[k];
        if (x >= t.x1a && x < t.x2a && y >= t.y1a && y < t.y2a) break;
    }
    if (k < 0) {
        for (int c = 0; c < C; ++c) out[c] = 114;
        return;
    }
    const b2y_mosaic_tile& t = it.tiles[k];
    b2y_lb_params p;
    p.src_h = t.src_h; p.src_w = t.src_w; p.channels = C; p.src_pitch = t.src_pitch;
    p.rs_h = t.rs_h; p.rs_w = t.rs_w; p.scale_x = t.scale_x; p.scale_y = t.scale_y;
    const int tx = x + t.dx, ty = y + t.dy;
    if (t.rs_w == t.src_w && t.rs_h == t.src_h) {
        const unsigned char* sp = t.src + (long long)ty * t.src_pitch + (long long)tx * C;
        for (int c = 0; c < C; ++c) out[c] = sp[c];
        return;
    }
    const b2y_lb_taps taps = b2y_lb_pixel_taps(p, tx, ty);
    for (int c = 0; c < C; ++c) out[c] = (unsigned char)b2y_lb_value(t.src, p, taps, c);
}

// Training batch from the canvases: blockIdx.z = item, blockIdx.y = output row, threads along the row.  The item's
// 768-byte HSV table is staged in shared memory.  Gather bound: 4 canvas pixels per output pixel (mostly L1/L2 hits:
// neighbouring threads read neighbouring taps), integer and a few float operations per pixel, C bytes written.
__global__ void __launch_bounds__(128) affine_hsv_u8_kernel(const b2y_affine_item* __restrict__ items,
                                                            const unsigned char* __restrict__ canvas,
                                                            unsigned char* __restrict__ dst, int C, int s) {
    __shared__ unsigned char lut[768];
    const b2y_affine_item& it = items[blockIdx.z];
    const int hsv = it.hsv;
    if (hsv)
        for (int i = threadIdx.x; i < 768; i += blockDim.x) lut[i] = it.lut[i];
    __syncthreads();
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= s) return;
    double im[6];
    for (int i = 0; i < 6; ++i) im[i] = it.im[i];
    const long long plane = (long long)s * s;
    const int s2 = 2 * s;
    b2y_augment_pixel(canvas + (long long)it.slot * s2 * s2 * C, s2, s2, C, im, hsv ? lut : nullptr, x, y,
                      dst + (long long)it.slot * C * plane + (long long)y * s + (it.flip ? s - 1 - x : x), plane);
}

bool exact_factor(double scale, int k) {            // cv::resize: |scale - saturate_cast<int>(scale)| < DBL_EPSILON
    return k > 0 && std::fabs(scale - (double)k) < 2.220446049250313e-16;
}

}  // namespace

extern "C" int b2y_load_batch_u8(const b2y_load_item* items, const b2y_load_item* items_dev, int n_items,
                                 unsigned char* dst, int batch, int channels, int dst_h, int dst_w, int swap_rb,
                                 int color, void* stream) {
    if (!items || !items_dev || !dst || n_items <= 0 || batch <= 0 || channels < 1 || channels > 4 || dst_h <= 0 ||
        dst_w <= 0 || color < 0 || color > 255)
        return B2Y_ERR_INVALID;
    if (n_items > 65535 || dst_h > 65535) return B2Y_ERR_UNSUPPORTED;
    for (int i = 0; i < n_items; ++i) {
        const b2y_load_item& it = items[i];
        if (!it.src || it.src_h <= 0 || it.src_w <= 0 || it.src_pitch < (long long)it.src_w * channels ||
            it.rs_h <= 0 || it.rs_w <= 0 || it.rs_h > it.src_h || it.rs_w > it.src_w || it.top < 0 || it.left < 0 ||
            it.top + it.rs_h > dst_h || it.left + it.rs_w > dst_w || it.slot < 0 || it.slot >= batch)
            return B2Y_ERR_INVALID;
        if (it.rs_h == it.src_h && it.rs_w == it.src_w) continue;            // copy: no resize
        // INTER_AREA downscale: the scales cv::resize derives from the two sizes, and the integer factors exactly when
        // it takes the block-mean path (which reads kx * rs_w columns and ky * rs_h rows)
        const double sx = 1.0 / ((double)it.rs_w / it.src_w), sy = 1.0 / ((double)it.rs_h / it.src_h);
        if (it.scale_x != sx || it.scale_y != sy) return B2Y_ERR_INVALID;
        const int kx = (int)std::nearbyint(sx), ky = (int)std::nearbyint(sy);
        if (exact_factor(sx, kx) && exact_factor(sy, ky)) {
            if (it.area_kx != kx || it.area_ky != ky || kx * it.rs_w != it.src_w || ky * it.rs_h != it.src_h)
                return B2Y_ERR_INVALID;
        } else if (it.area_kx != 0 || it.area_ky != 0) {
            return B2Y_ERR_INVALID;
        }
    }
    const dim3 grid((dst_w + 127) / 128, dst_h, n_items);
    load_batch_u8_kernel<<<grid, 128, 0, static_cast<cudaStream_t>(stream)>>>(items_dev, dst, channels, dst_h, dst_w,
                                                                              swap_rb ? 1 : 0, (unsigned char)color);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_mosaic_u8(const b2y_mosaic_item* items, const b2y_mosaic_item* items_dev, int n_items,
                             unsigned char* canvas, int batch, int channels, int s, void* stream) {
    if (!items || !items_dev || !canvas || n_items <= 0 || batch <= 0 || channels < 1 || channels > 4 || s <= 0)
        return B2Y_ERR_INVALID;
    if (n_items > 65535 || 2 * s > 65535) return B2Y_ERR_UNSUPPORTED;
    const int s2 = 2 * s;
    for (int i = 0; i < n_items; ++i) {
        if (items[i].slot < 0 || items[i].slot >= batch) return B2Y_ERR_INVALID;
        for (int k = 0; k < 4; ++k) {
            const b2y_mosaic_tile& t = items[i].tiles[k];
            if (!t.src || t.src_h <= 0 || t.src_w <= 0 || t.src_pitch < (long long)t.src_w * channels || t.rs_h <= 0 ||
                t.rs_w <= 0 || t.x1a < 0 || t.y1a < 0 || t.x1a > t.x2a || t.y1a > t.y2a || t.x2a > s2 || t.y2a > s2)
                return B2Y_ERR_INVALID;
            if (t.x2a > t.x1a && t.y2a > t.y1a &&                            // a non-empty rectangle reads its tile
                (t.x1a + t.dx < 0 || t.y1a + t.dy < 0 || t.x2a + t.dx > t.rs_w || t.y2a + t.dy > t.rs_h))
                return B2Y_ERR_INVALID;
            if (t.rs_h == t.src_h && t.rs_w == t.src_w) continue;            // copy: no resize
            if (t.scale_x != 1.0 / ((double)t.rs_w / t.src_w) || t.scale_y != 1.0 / ((double)t.rs_h / t.src_h))
                return B2Y_ERR_INVALID;
        }
    }
    const dim3 grid((s2 + 127) / 128, s2, n_items);
    mosaic_u8_kernel<<<grid, 128, 0, static_cast<cudaStream_t>(stream)>>>(items_dev, canvas, channels, s2);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_affine_hsv_u8(const b2y_affine_item* items, const b2y_affine_item* items_dev, int n_items,
                                 const unsigned char* canvas, unsigned char* dst, int batch, int channels, int s,
                                 void* stream) {
    if (!items || !items_dev || !canvas || !dst || n_items <= 0 || batch <= 0 || channels < 1 || channels > 4 || s <= 0)
        return B2Y_ERR_INVALID;
    if (n_items > 65535 || s > 65535) return B2Y_ERR_UNSUPPORTED;
    for (int i = 0; i < n_items; ++i) {
        const b2y_affine_item& it = items[i];
        if (it.slot < 0 || it.slot >= batch || (it.hsv != 0 && it.hsv != 1) || (it.hsv && channels != 3) ||
            (it.flip != 0 && it.flip != 1))
            return B2Y_ERR_INVALID;
        // the fixed-point coordinates (source position * 1024) of every output pixel must fit an int: the map is
        // affine, so its extremes are at the corners
        for (int r = 0; r < 2; ++r)
            for (int cy = 0; cy < 2; ++cy)
                for (int cx = 0; cx < 2; ++cx) {
                    const double v = (it.im[3 * r] * (cx * (s - 1)) + it.im[3 * r + 1] * (cy * (s - 1)) + it.im[3 * r + 2]);
                    if (!(std::fabs(v) < 1.0e6)) return B2Y_ERR_INVALID;            // also rejects NaN
                }
    }
    const dim3 grid((s + 127) / 128, s, n_items);
    affine_hsv_u8_kernel<<<grid, 128, 0, static_cast<cudaStream_t>(stream)>>>(items_dev, canvas, dst, channels, s);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}

extern "C" int b2y_letterbox_u8(const unsigned char* src, int src_h, int src_w, int channels, long long src_pitch,
                                int resized_h, int resized_w, int top, int left, unsigned char* dst, int dst_h, int dst_w,
                                int swap_rb, int color, void* stream) {
    if (!src || !dst || src_h <= 0 || src_w <= 0 || channels < 1 || channels > 4 || resized_h <= 0 || resized_w <= 0 ||
        dst_h <= 0 || dst_w <= 0 || top < 0 || left < 0 || src_pitch < (long long)src_w * channels || color < 0 ||
        color > 255)
        return B2Y_ERR_INVALID;
    if (top + resized_h > dst_h || left + resized_w > dst_w) return B2Y_ERR_INVALID;
    if (dst_h > 65535) return B2Y_ERR_UNSUPPORTED;
    b2y_lb_params p;
    p.src_h = src_h; p.src_w = src_w; p.channels = channels; p.src_pitch = src_pitch;
    p.rs_h = resized_h; p.rs_w = resized_w; p.top = top; p.left = left; p.dst_h = dst_h; p.dst_w = dst_w;
    p.swap_rb = swap_rb ? 1 : 0; p.color = (unsigned char)color;
    b2y_lb_set_scales(p);
    const dim3 grid((dst_w + 255) / 256, dst_h);
    letterbox_u8_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(src, dst, p);
    B2Y_CUDA_CHECK(cudaGetLastError());
    return B2Y_OK;
}
