// Host harness of the CPU tests: runs csrc/preprocess_core.h's INTER_AREA per-pixel code (shared with the device
// loader, csrc/preprocess.cu) over a whole image.  dst is HWC [rs_h][rs_w][channels], like cv2.resize's output.
#include "preprocess_core.h"

extern "C" int b2y_area_resize_host(const unsigned char* src, int src_h, int src_w, int channels, long long src_pitch,
                                    int rs_h, int rs_w, int kx, int ky, double scale_x, double scale_y,
                                    unsigned char* dst) {
    b2y_area_params p;
    p.src_h = src_h; p.src_w = src_w; p.channels = channels; p.src_pitch = src_pitch;
    p.rs_h = rs_h; p.rs_w = rs_w; p.kx = kx; p.ky = ky; p.scale_x = scale_x; p.scale_y = scale_y;
    for (int y = 0; y < rs_h; ++y)
        for (int x = 0; x < rs_w; ++x)
            for (int c = 0; c < channels; ++c)
                dst[((long long)y * rs_w + x) * channels + c] = (unsigned char)b2y_area_value(src, p, x, y, c);
    return 0;
}

// One slot of an evaluation batch, pixel by pixel as b2y_load_batch_u8's kernel writes it: dst planar [channels][H][W].
extern "C" int b2y_load_slot_host(const unsigned char* src, int src_h, int src_w, int channels, long long src_pitch,
                                  int rs_h, int rs_w, int kx, int ky, double scale_x, double scale_y, int top, int left,
                                  unsigned char* dst, int H, int W, int swap_rb, int color) {
    b2y_area_params p;
    p.src_h = src_h; p.src_w = src_w; p.channels = channels; p.src_pitch = src_pitch;
    p.rs_h = rs_h; p.rs_w = rs_w; p.kx = kx; p.ky = ky; p.scale_x = scale_x; p.scale_y = scale_y;
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x)
            b2y_load_pixel(src, p, top, left, x, y, swap_rb, (unsigned char)color, dst + (long long)y * W + x,
                           (long long)H * W);
    return 0;
}
