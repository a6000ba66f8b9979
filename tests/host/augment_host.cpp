// Host harness of the CPU tests: runs csrc/preprocess_core.h's training-augmentation per-pixel code (shared with the
// device training loader, csrc/preprocess.cu) over whole images, in the layouts of the cv2 calls it restates.
#include "preprocess_core.h"

// cv2.cvtColor(COLOR_BGR2HSV) / (COLOR_HSV2BGR) of n pixels, interleaved triples.
extern "C" void b2y_bgr2hsv_host(const unsigned char* src, unsigned char* dst, long long n) {
    for (long long i = 0; i < n; ++i) {
        int h, s, v;
        b2y_bgr2hsv(src[3 * i], src[3 * i + 1], src[3 * i + 2], h, s, v);
        dst[3 * i] = (unsigned char)h; dst[3 * i + 1] = (unsigned char)s; dst[3 * i + 2] = (unsigned char)v;
    }
}

extern "C" void b2y_hsv2bgr_host(const unsigned char* src, unsigned char* dst, long long n) {
    for (long long i = 0; i < n; ++i) {
        int b, g, r;
        b2y_hsv2bgr(src[3 * i], src[3 * i + 1], src[3 * i + 2], b, g, r);
        dst[3 * i] = (unsigned char)b; dst[3 * i + 1] = (unsigned char)g; dst[3 * i + 2] = (unsigned char)r;
    }
}

// cv2.warpAffine(src, M, (dst_w, dst_h), INTER_LINEAR, borderValue=border) with im = invertAffineTransform(M);
// src and dst HWC.
extern "C" void b2y_warp_host(const unsigned char* src, int h, int w, int C, const double* im, unsigned char* dst,
                              int dst_h, int dst_w, int border) {
    for (int y = 0; y < dst_h; ++y)
        for (int x = 0; x < dst_w; ++x) {
            const b2y_warp_taps t = b2y_warp_pixel_taps(im, x, y);
            for (int c = 0; c < C; ++c)
                dst[((long long)y * dst_w + x) * C + c] =
                    (unsigned char)b2y_warp_value(src, h, w, C, (long long)w * C, t, c, border);
        }
}

// load_image's cv2.resize(INTER_LINEAR) of an HWC source to rs_w x rs_h, through the mosaic's tile code.
extern "C" void b2y_tile_host(const unsigned char* src, int src_h, int src_w, int C, int rs_h, int rs_w,
                              unsigned char* dst) {
    b2y_lb_params p = {};
    p.src_h = src_h; p.src_w = src_w; p.channels = C; p.src_pitch = (long long)src_w * C;
    p.rs_h = rs_h; p.rs_w = rs_w;
    b2y_lb_set_scales(p);
    for (int y = 0; y < rs_h; ++y)
        for (int x = 0; x < rs_w; ++x)
            for (int c = 0; c < C; ++c) dst[((long long)y * rs_w + x) * C + c] = (unsigned char)b2y_tile_value(src, p, x, y, c);
}

// One batch slot after the canvas: warp, HSV (lut = 3 x 256 bytes, or null), flip, channel reversal; dst planar
// [C][s][s].
extern "C" void b2y_augment_slot_host(const unsigned char* canvas, int ch, int cw, int C, const double* im,
                                      const unsigned char* lut, int flip, unsigned char* dst, int s) {
    const long long plane = (long long)s * s;
    for (int y = 0; y < s; ++y)
        for (int x = 0; x < s; ++x)
            b2y_augment_pixel(canvas, ch, cw, C, im, lut, x, y, dst + (long long)y * s + (flip ? s - 1 - x : x), plane);
}
