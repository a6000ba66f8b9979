// Per-pixel arithmetic of the device letterbox, evaluation and training batch loaders (csrc/preprocess.cu), shared with
// the host harnesses of the CPU tests (tests/host/letterbox_host.cpp, area_host.cpp, augment_host.cpp) so that the very
// same code is checked against cv2's outputs without a GPU.
//
// OpenCV 4.x modules/imgproc/src/resize.cpp, 8-bit INTER_LINEAR (fixed point, INTER_RESIZE_COEF_BITS = 11):
//   fx = (float)((dx + 0.5) * scale_x - 0.5), sx = floor(fx), fx -= sx; columns clamp (sx < 0 -> fx = 0, sx = 0;
//   sx >= w - 1 -> fx = 0, sx = w - 1); rows clamp the ROW INDICES only, not the weights;
//   coefficients = cvRound(c * 2048) (int16); horizontal pass S[sx] * a0 + S[sx + 1] * a1 (int32);
//   vertical pass (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2.
#ifndef B2Y_PREPROCESS_CORE_H_
#define B2Y_PREPROCESS_CORE_H_

#if defined(__CUDACC__)
#define B2Y_HD __host__ __device__ __forceinline__
#else
#include <cmath>
#define B2Y_HD inline
#endif

struct b2y_lb_params {
    int src_h, src_w, channels;       // source image, HWC uint8
    long long src_pitch;              // bytes per source row
    int rs_h, rs_w;                   // size after cv2.resize (== source size: plain copy)
    int top, left;                    // border
    int dst_h, dst_w;                 // output plane size
    int swap_rb;                      // 1: output channel c = source channel (channels - 1 - c)   (BGR -> RGB)
    unsigned char color;
    double scale_x, scale_y;          // resize.cpp: scale_x = 1. / ((double)dsize.width / ssize.width)
};

// OpenCV's scalar set-up code runs without FMA: (dx + 0.5) * scale - 0.5 rounds twice.  Device code must not contract it.
B2Y_HD float b2y_lb_src_coord(int d, double scale) {
#if defined(__CUDA_ARCH__)
    return (float)__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5);
#else
    volatile double t = ((double)d + 0.5) * scale;      // volatile: no contraction on the host either
    return (float)(t - 0.5);
#endif
}

B2Y_HD int b2y_lb_round(float v) {                       // saturate_cast<short>(float) = cvRound: nearest, ties to even
#if defined(__CUDA_ARCH__)
    return __float2int_rn(v);
#else
    return (int)std::nearbyint(v);
#endif
}

B2Y_HD void b2y_lb_coeff(int d, double scale, int src, bool clamp, int& s, int& a0, int& a1) {
    float f = b2y_lb_src_coord(d, scale);
    int si = (int)floorf(f);
#if defined(__CUDA_ARCH__)
    f = __fsub_rn(f, (float)si);
    const float g = __fsub_rn(1.f, f);
#else
    f = f - (float)si;
    const float g = 1.f - f;
#endif
    float f1 = f, f0 = g;
    if (clamp) {
        if (si < 0) { f1 = 0.f; f0 = 1.f; si = 0; }
        if (si >= src - 1) { f1 = 0.f; f0 = 1.f; si = src - 1; }
    }
#if defined(__CUDA_ARCH__)
    a0 = b2y_lb_round(__fmul_rn(f0, 2048.f));
    a1 = b2y_lb_round(__fmul_rn(f1, 2048.f));
#else
    a0 = b2y_lb_round(f0 * 2048.f);
    a1 = b2y_lb_round(f1 * 2048.f);
#endif
    s = si;
}

// The taps of resized pixel (rx, ry): source columns sx, x1 with weights a0, a1; rows y0, y1 with weights b0, b1.
struct b2y_lb_taps {
    int sx, x1, y0, y1, a0, a1, b0, b1;
};

B2Y_HD b2y_lb_taps b2y_lb_pixel_taps(const b2y_lb_params& p, int rx, int ry) {
    b2y_lb_taps t;
    int sy;
    b2y_lb_coeff(rx, p.scale_x, p.src_w, true, t.sx, t.a0, t.a1);
    b2y_lb_coeff(ry, p.scale_y, p.src_h, false, sy, t.b0, t.b1);
    t.x1 = t.sx + 1 < p.src_w ? t.sx + 1 : p.src_w - 1;
    int y0 = sy < 0 ? 0 : sy, y1 = sy + 1 < 0 ? 0 : sy + 1;
    t.y0 = y0 < p.src_h ? y0 : p.src_h - 1;
    t.y1 = y1 < p.src_h ? y1 : p.src_h - 1;
    return t;
}

// Channel sc of the resized pixel whose taps are t.
B2Y_HD int b2y_lb_value(const unsigned char* src, const b2y_lb_params& p, const b2y_lb_taps& t, int sc) {
    const int C = p.channels;
    const unsigned char* r0 = src + (long long)t.y0 * p.src_pitch;
    const unsigned char* r1 = src + (long long)t.y1 * p.src_pitch;
    const int h0 = (int)r0[t.sx * C + sc] * t.a0 + (int)r0[t.x1 * C + sc] * t.a1;
    const int h1 = (int)r1[t.sx * C + sc] * t.a0 + (int)r1[t.x1 * C + sc] * t.a1;
    const int v = (((t.b0 * (h0 >> 4)) >> 16) + ((t.b1 * (h1 >> 4)) >> 16) + 2) >> 2;
    return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// One output pixel (all channels): dst is planar [channels][dst_h][dst_w].
B2Y_HD void b2y_lb_pixel(const unsigned char* src, unsigned char* dst, const b2y_lb_params& p, int x, int y) {
    const int C = p.channels;
    const int rx = x - p.left, ry = y - p.top;
    const long long plane = (long long)p.dst_h * p.dst_w;
    unsigned char* out = dst + (long long)y * p.dst_w + x;
    if (rx < 0 || ry < 0 || rx >= p.rs_w || ry >= p.rs_h) {                 // copyMakeBorder(..., value = color)
        for (int c = 0; c < C; ++c) out[c * plane] = p.color;
        return;
    }
    if (p.rs_w == p.src_w && p.rs_h == p.src_h) {                            // shape[::-1] == new_unpad: no resize
        const unsigned char* s = src + (long long)ry * p.src_pitch + (long long)rx * C;
        for (int c = 0; c < C; ++c) out[c * plane] = s[p.swap_rb ? C - 1 - c : c];
        return;
    }
    const b2y_lb_taps t = b2y_lb_pixel_taps(p, rx, ry);
    for (int c = 0; c < C; ++c) out[c * plane] = (unsigned char)b2y_lb_value(src, p, t, p.swap_rb ? C - 1 - c : c);
}

B2Y_HD void b2y_lb_set_scales(b2y_lb_params& p) {
    p.scale_x = 1.0 / ((double)p.rs_w / (double)p.src_w);
    p.scale_y = 1.0 / ((double)p.rs_h / (double)p.src_h);
}

// ---- 8-bit INTER_AREA downscale (load_image of the reference's LoadImagesAndLabels, utils/datasets.py:511-531) ----
// OpenCV 4.x resize.cpp, both scales >= 1 (scale = 1. / ((double)dsize / ssize)), restated and pinned against cv2:
//   * integer factors (|scale - cvRound(scale)| < DBL_EPSILON on both axes): mean of the kx x ky block, integer sum;
//     2 x 2 rounds (sum + 2) >> 2, every other block cvRound((float)sum * (1.f / (kx * ky)));
//   * otherwise per axis and output index d (computeResizeAreaTab, in double): f1 = d * scale, f2 = f1 + scale,
//     cell = min(scale, size - f1), s1 = ceil(f1), s2 = min(floor(f2), size - 1), s1 = min(s1, s2); the taps are
//     s1 - 1 with (float)((s1 - f1) / cell) if s1 - f1 > 1e-3, s1 .. s2 - 1 with (float)(1. / cell), and s2 with
//     (float)(min(min(f2 - s2, 1.), cell) / cell) if f2 - s2 > 1e-3 -- consecutive source indices.  Per source row of
//     the y taps, a float row buf = buf + src * alpha over the x taps; then sum = beta0 * buf0, sum = sum + beta * buf
//     (float, no FMA anywhere); the byte is saturate_cast<uchar>(sum) = cvRound, ties to even.
struct b2y_area_params {
    int src_h, src_w, channels;
    long long src_pitch;              // bytes per source row
    int rs_h, rs_w;                   // INTER_AREA output size
    int kx, ky;                       // both > 0: integer factors (block mean); 0: the fractional path
    double scale_x, scale_y;          // src / rs as cv::resize computes it
};

B2Y_HD double b2y_dmul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    volatile double t = a * b;
    return t;
#endif
}

B2Y_HD float b2y_fmul(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    volatile float t = a * b;
    return t;
#endif
}

B2Y_HD float b2y_fadd(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    volatile float t = a + b;
    return t;
#endif
}

B2Y_HD int b2y_area_round(float v) {                     // saturate_cast<uchar>(float)
    const int i = b2y_lb_round(v);
    return i < 0 ? 0 : (i > 255 ? 255 : i);
}

// The taps of output index d along one axis: n consecutive source indices from first; weight k is w_lo for k == 0
// when has_lo, w_hi for k == n - 1 when has_hi, w_mid otherwise.
struct b2y_area_taps {
    int first, n;
    bool has_lo, has_hi;
    float w_lo, w_mid, w_hi;
    B2Y_HD float weight(int k) const { return (k == 0 && has_lo) ? w_lo : ((k == n - 1 && has_hi) ? w_hi : w_mid); }
};

B2Y_HD b2y_area_taps b2y_area_axis(int d, int size, double scale) {
    const double f1 = b2y_dmul((double)d, scale);
#if defined(__CUDA_ARCH__)
    const double f2 = __dadd_rn(f1, scale);
    const double rest = __dsub_rn((double)size, f1);
#else
    volatile double f2v = f1 + scale, restv = (double)size - f1;
    const double f2 = f2v, rest = restv;
#endif
    const double cell = scale < rest ? scale : rest;
    int s1 = (int)ceil(f1), s2 = (int)floor(f2);
    s2 = s2 < size - 1 ? s2 : size - 1;
    s1 = s1 < s2 ? s1 : s2;
    b2y_area_taps t;
#if defined(__CUDA_ARCH__)
    const double lo = __dsub_rn((double)s1, f1), hi = __dsub_rn(f2, (double)s2);
    t.w_lo = (float)__ddiv_rn(lo, cell);
    t.w_mid = (float)__ddiv_rn(1.0, cell);
    double h = hi < 1.0 ? hi : 1.0;
    h = h < cell ? h : cell;
    t.w_hi = (float)__ddiv_rn(h, cell);
#else
    volatile double lov = (double)s1 - f1, hiv = f2 - (double)s2;
    const double lo = lov, hi = hiv;
    t.w_lo = (float)(lo / cell);
    t.w_mid = (float)(1.0 / cell);
    double h = hi < 1.0 ? hi : 1.0;
    h = h < cell ? h : cell;
    t.w_hi = (float)(h / cell);
#endif
    t.has_lo = lo > 1e-3;
    t.has_hi = hi > 1e-3;
    t.first = t.has_lo ? s1 - 1 : s1;
    t.n = (s2 - s1) + (t.has_lo ? 1 : 0) + (t.has_hi ? 1 : 0);
    return t;
}

// Output pixel (x, y) of the resized image, channel sc of the source, as a byte.
B2Y_HD int b2y_area_value(const unsigned char* src, const b2y_area_params& p, int x, int y, int sc) {
    const int C = p.channels;
    if (p.kx > 0 && p.ky > 0) {
        const unsigned char* s = src + (long long)y * p.ky * p.src_pitch + (long long)x * p.kx * C + sc;
        int sum = 0;
        for (int j = 0; j < p.ky; ++j)
            for (int i = 0; i < p.kx; ++i) sum += s[(long long)j * p.src_pitch + i * C];
        if (p.kx == 2 && p.ky == 2) return (sum + 2) >> 2;
#if defined(__CUDA_ARCH__)
        const float inv = __fdiv_rn(1.f, (float)(p.kx * p.ky));
#else
        volatile float inv = 1.f / (float)(p.kx * p.ky);
#endif
        return b2y_area_round(b2y_fmul((float)sum, inv));
    }
    const b2y_area_taps tx = b2y_area_axis(x, p.src_w, p.scale_x);
    const b2y_area_taps ty = b2y_area_axis(y, p.src_h, p.scale_y);
    float sum = 0.f;
    for (int j = 0; j < ty.n; ++j) {
        const unsigned char* row = src + (long long)(ty.first + j) * p.src_pitch + (long long)tx.first * C + sc;
        float buf = 0.f;
        for (int i = 0; i < tx.n; ++i) buf = b2y_fadd(buf, b2y_fmul((float)row[i * C], tx.weight(i)));
        const float v = b2y_fmul(ty.weight(j), buf);
        sum = j == 0 ? v : b2y_fadd(sum, v);
    }
    return b2y_area_round(sum);
}

// One output pixel (all channels) of an evaluation batch slot: border `color` outside the resized image at (top, left),
// else the INTER_AREA value (a plain copy when the source already has the resized size), channels reversed when swap_rb.
// out points at channel 0 of the pixel in a planar [C][H][W] slot.
B2Y_HD void b2y_load_pixel(const unsigned char* src, const b2y_area_params& p, int top, int left, int x, int y,
                           int swap_rb, unsigned char color, unsigned char* out, long long plane) {
    const int C = p.channels;
    const int rx = x - left, ry = y - top;
    if (rx < 0 || ry < 0 || rx >= p.rs_w || ry >= p.rs_h) {
        for (int c = 0; c < C; ++c) out[c * plane] = color;
        return;
    }
    if (p.rs_w == p.src_w && p.rs_h == p.src_h) {
        const unsigned char* s = src + (long long)ry * p.src_pitch + (long long)rx * C;
        for (int c = 0; c < C; ++c) out[c * plane] = s[swap_rb ? C - 1 - c : c];
        return;
    }
    for (int c = 0; c < C; ++c) out[c * plane] = (unsigned char)b2y_area_value(src, p, rx, ry, swap_rb ? C - 1 - c : c);
}

// ---- training-time augmentation (LoadImagesAndLabels(augment=True).__getitem__, utils/datasets.py:419-501) ----
// Mosaic tiles (load_mosaic, :553-608): a canvas pixel inside a tile's rectangle is the tile pixel at (x + dx, y + dy);
// an uncached tile is load_image's cv2.resize(INTER_LINEAR) of its source, i.e. b2y_lb_value.  cv::resize takes the
// INTER_AREA 2 x 2 block mean for an exact 2x downscale; the bilinear weights there are 1024 / 1024 on both axes and
// give the same (a + b + c + d + 2) >> 2, so this one path covers it.
B2Y_HD int b2y_tile_value(const unsigned char* src, const b2y_lb_params& p, int tx, int ty, int sc) {
    if (p.rs_w == p.src_w && p.rs_h == p.src_h) return src[(long long)ty * p.src_pitch + (long long)tx * p.channels + sc];
    const b2y_lb_taps t = b2y_lb_pixel_taps(p, tx, ty);
    return b2y_lb_value(src, p, t, sc);
}

// cv2.warpAffine(src, M, dsize, INTER_LINEAR, BORDER_CONSTANT) for 8-bit images, OpenCV 4.x imgwarp.cpp: im = the
// inverse of M (invertAffineTransform, in double, computed by the caller).  Per output pixel, with AB_BITS = 10 and
// INTER_BITS = 5: X = (cvRound((im1 * y + im2) * 1024) + 16 + cvRound(im0 * x * 1024)) >> 5 (and Y with im3..im5);
// the top-left tap is (X >> 5, Y >> 5), the fraction (X & 31, Y & 31).  The 32 x 32 fixed-point table of
// initInterTab2D holds (1 - fy)(1 - fx), (1 - fy) fx, fy (1 - fx), fy fx times 32768 for fx, fy = k / 32: exact
// products that sum to 32768, so OpenCV's rounding correction never fires.  The byte is (sum w * S + (1 << 14)) >> 15;
// a tap outside the source reads the border value.
struct b2y_warp_taps {
    int sx, sy, w[4];
};

B2Y_HD int b2y_dround(double v) {                        // cvRound(double): nearest, ties to even
#if defined(__CUDA_ARCH__)
    return __double2int_rn(v);
#else
    return (int)std::nearbyint(v);
#endif
}

B2Y_HD double b2y_dadd(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    volatile double t = a + b;
    return t;
#endif
}

B2Y_HD b2y_warp_taps b2y_warp_pixel_taps(const double* im, int x, int y) {
    const int X0 = b2y_dround(b2y_dmul(b2y_dadd(b2y_dmul(im[1], (double)y), im[2]), 1024.0)) + 16;
    const int Y0 = b2y_dround(b2y_dmul(b2y_dadd(b2y_dmul(im[4], (double)y), im[5]), 1024.0)) + 16;
    const int X = (X0 + b2y_dround(b2y_dmul(b2y_dmul(im[0], (double)x), 1024.0))) >> 5;
    const int Y = (Y0 + b2y_dround(b2y_dmul(b2y_dmul(im[3], (double)x), 1024.0))) >> 5;
    b2y_warp_taps t;
    t.sx = X >> 5;
    t.sy = Y >> 5;
    const int fx = X & 31, fy = Y & 31;
    t.w[0] = (32 - fy) * (32 - fx) * 32;
    t.w[1] = (32 - fy) * fx * 32;
    t.w[2] = fy * (32 - fx) * 32;
    t.w[3] = fy * fx * 32;
    return t;
}

// Channel c of the warped pixel: src HWC [h][w][C] with row pitch `pitch` bytes.
B2Y_HD int b2y_warp_value(const unsigned char* src, int h, int w, int C, long long pitch, const b2y_warp_taps& t, int c,
                          int border) {
    const bool x0 = t.sx >= 0 && t.sx < w, x1 = t.sx + 1 >= 0 && t.sx + 1 < w;
    const bool y0 = t.sy >= 0 && t.sy < h, y1 = t.sy + 1 >= 0 && t.sy + 1 < h;
    const unsigned char* p = src + (long long)t.sy * pitch + (long long)t.sx * C + c;
    const int sum = t.w[0] * (y0 && x0 ? (int)p[0] : border) + t.w[1] * (y0 && x1 ? (int)p[C] : border) +
                    t.w[2] * (y1 && x0 ? (int)p[pitch] : border) + t.w[3] * (y1 && x1 ? (int)p[pitch + C] : border);
    const int v = (sum + (1 << 14)) >> 15;
    return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// cv2.cvtColor(COLOR_BGR2HSV) for 8-bit images (OpenCV 4.x color_hsv: integer tables, hsv_shift = 12, H in 0..179):
// sdiv(v) = cvRound((255 << 12) / (double)v), hdiv(d) = cvRound((180 << 12) / (6. * d)), both 0 at 0.
B2Y_HD void b2y_bgr2hsv(int b, int g, int r, int& h, int& s, int& v) {
    v = b > g ? b : g;
    v = v > r ? v : r;
    int vmin = b < g ? b : g;
    vmin = vmin < r ? vmin : r;
    const int diff = v - vmin;
    const int vr = v == r ? -1 : 0, vg = v == g ? -1 : 0;
#if defined(__CUDA_ARCH__)
    const int sdiv = v ? __double2int_rn(__ddiv_rn((double)(255 << 12), (double)v)) : 0;
    const int hdiv = diff ? __double2int_rn(__ddiv_rn((double)(180 << 12), 6.0 * diff)) : 0;
#else
    const int sdiv = v ? (int)std::nearbyint((double)(255 << 12) / (double)v) : 0;
    const int hdiv = diff ? (int)std::nearbyint((double)(180 << 12) / (6.0 * diff)) : 0;
#endif
    s = (diff * sdiv + (1 << 11)) >> 12;
    int hh = (vr & (g - b)) + (~vr & ((vg & (b - r + 2 * diff)) + (~vg & (r - g + 4 * diff))));
    hh = (hh * hdiv + (1 << 11)) >> 12;
    hh += hh < 0 ? 180 : 0;
    h = hh < 0 ? 0 : (hh > 255 ? 255 : hh);
}

B2Y_HD float b2y_ffma(float a, float b, float c) {
#if defined(__CUDA_ARCH__)
    return __fmaf_rn(a, b, c);
#else
    return std::fmaf(a, b, c);
#endif
}

B2Y_HD float b2y_fsub(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fsub_rn(a, b);
#else
    volatile float t = a - b;
    return t;
#endif
}

// cv2.cvtColor(COLOR_HSV2BGR) for 8-bit images as OpenCV 4.x's default (vectorised, AVX2) dispatch computes it, in
// float: h = H * (6.f / 180), s = S * (1.f / 255), v = V * (1.f / 255); sector = trunc(h) mod 6, f = h - trunc(h);
// tab = {v, v * (1 - s), v * fma(-s, f, 1), v * fma(-s, 1 - f, 1)} -- the two inner products FUSED with the
// subtraction, as the optimised build contracts them (the scalar path, cv2.setUseOptimized(False), rounds them
// separately and differs in the last bit on about 1 in 7000 bytes); each output byte is trunc(tab[k] * 255.f).
// The vector loop covers whole blocks of 32 pixels of a row; every row width the training loader uses (img_size is a
// multiple of 32) runs it end to end.
B2Y_HD void b2y_hsv2bgr(int H, int S, int V, int& b, int& g, int& r) {
    const float hh = b2y_fmul((float)H, 6.0f / 180), s = b2y_fmul((float)S, 1.0f / 255), v = b2y_fmul((float)V, 1.0f / 255);
    const float pre = truncf(hh), f = b2y_fsub(hh, pre);
    const float t1 = b2y_fmul(v, b2y_fsub(1.f, s));
    const float t2 = b2y_fmul(v, b2y_ffma(-s, f, 1.f));
    const float t3 = b2y_fmul(v, b2y_ffma(-s, b2y_fsub(1.f, f), 1.f));
    const int sh = 4 * ((int)pre % 6);
    // sector_data of color_hsv ({1,3,0}, {1,0,2}, {3,0,1}, {0,2,1}, {0,1,3}, {2,1,0}): the tab index of b, g and r
    // per sector, one nibble per sector
    const int kb = (0x200311 >> sh) & 15, kg = (0x112003 >> sh) & 15, kr = (0x031120 >> sh) & 15;
    b = (int)b2y_fmul(kb == 0 ? v : (kb == 1 ? t1 : (kb == 2 ? t2 : t3)), 255.f);
    g = (int)b2y_fmul(kg == 0 ? v : (kg == 1 ? t1 : (kg == 2 ? t2 : t3)), 255.f);
    r = (int)b2y_fmul(kr == 0 ? v : (kr == 1 ? t1 : (kr == 2 ? t2 : t3)), 255.f);
}

// One output pixel of a training batch after the mosaic canvas: warp (border 114), augment_hsv's BGR2HSV -> LUT ->
// HSV2BGR when lut != nullptr (colour only), then written reversed (BGR -> RGB) into channel planes out[c * plane].
// (x, y) is the position in the warped image; the caller applies the left-right flip by choosing where out points.
B2Y_HD void b2y_augment_pixel(const unsigned char* canvas, int ch, int cw, int C, const double* im,
                              const unsigned char* lut, int x, int y, unsigned char* out, long long plane) {
    const b2y_warp_taps t = b2y_warp_pixel_taps(im, x, y);
    const long long pitch = (long long)cw * C;
    if (C == 3) {
        int b = b2y_warp_value(canvas, ch, cw, 3, pitch, t, 0, 114);
        int g = b2y_warp_value(canvas, ch, cw, 3, pitch, t, 1, 114);
        int r = b2y_warp_value(canvas, ch, cw, 3, pitch, t, 2, 114);
        if (lut) {
            int h, s, v;
            b2y_bgr2hsv(b, g, r, h, s, v);
            b2y_hsv2bgr(lut[h], lut[256 + s], lut[512 + v], b, g, r);
        }
        out[0] = (unsigned char)r;
        out[plane] = (unsigned char)g;
        out[2 * plane] = (unsigned char)b;
        return;
    }
    for (int c = 0; c < C; ++c) out[c * plane] = (unsigned char)b2y_warp_value(canvas, ch, cw, C, pitch, t, c, 114);
}

#endif  // B2Y_PREPROCESS_CORE_H_
