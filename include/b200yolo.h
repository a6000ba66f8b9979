/*
 * b200yolo.h -- C ABI of libb200yolo.so (sm_90a kernels for the Darknet YOLOv3/v4 hot path).
 *
 * The reference (SpursLipu/YOLOv3v4-ModelCompression-MultidatasetTraining-Multibackbone) is pure
 * Python on top of torch ATen; it has no FFI of its own.  The drop-in boundary is therefore the
 * Python module API (models.Darknet, utils.utils.compute_loss, utils/quantized/...), and this
 * header is the native boundary *underneath* it (SURVEY.md section 8b): every entry point replaces
 * the ATen/cuDNN call(s) issued at the cited reference file:line.
 *
 * Conventions
 *   - plain C, device pointers + explicit shapes, no allocation inside, no exceptions;
 *   - every function returns 0 on success, <0 on error (b2y_strerror);
 *   - `stream` is a cudaStream_t passed as void*; kernels are enqueued, never synchronised;
 *   - activations are NHWC ("pixel-major"): element (n,y,x,c) at ((n*H+y)*W+x)*pitch + c, where
 *     `pitch` >= C lets a tensor live as a channel slice of a wider (route/concat) buffer;
 *   - fp16 activations/weights for the dense path, fp32 for the YOLO head, loss and statistics.
 */
#ifndef B200YOLO_H_
#define B200YOLO_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2Y_ABI_VERSION 3

/* status codes */
#define B2Y_OK 0
#define B2Y_ERR_INVALID (-1)
#define B2Y_ERR_CUDA (-2)
#define B2Y_ERR_UNSUPPORTED (-3)
#define B2Y_ERR_DRIVER (-4)

/* activation ids -- models.py:102-113 (leaky/relu6/h_swish/relu/mish), utils/layers.py:141-173 */
#define B2Y_ACT_LINEAR 0
#define B2Y_ACT_LEAKY 1
#define B2Y_ACT_MISH 2
#define B2Y_ACT_RELU 3
#define B2Y_ACT_RELU6 4
#define B2Y_ACT_HSWISH 5
#define B2Y_ACT_SWISH 6

/* 16-bit tensor dtypes.  Training: activation gradients (dY) are stored in bf16 (fp16 over/underflows across the ~100
 * BatchNorm layers of a Darknet); the conv data gradient dZ that feeds the tensor-core GEMMs is fp16 times a per-layer
 * power-of-two scale picked on the device (wgmma takes one 16-bit format for both operands) */
#define B2Y_DT_F16 0
#define B2Y_DT_BF16 1

/* output dtypes of the conv epilogue */
#define B2Y_OUT_F16 0
#define B2Y_OUT_F32 1
#define B2Y_OUT_I8 2

int b2y_abi_version(void);
const char* b2y_strerror(int status);
int b2y_last_cuda_error(void);   /* raw cudaError_t of the last B2Y_ERR_CUDA on this thread */
int b2y_device_sm_count(void);   /* -1 without a CUDA device */

/* ------------------------------------------------------------------------------------------------
 * Dense convolution block: Conv2d (+ folded BatchNorm) + activation (+ residual add)
 * replaces nn.Conv2d / nn.BatchNorm2d(eval) / activation / Shortcut  (models.py:92-113,
 * utils/layers.py:43-72, utils/torch_utils.py:65-89).
 * ------------------------------------------------------------------------------------------------ */
typedef struct b2y_conv_desc {
    int batch, in_h, in_w, in_c; /* logical NHWC input */
    long long in_pitch;          /* elements between consecutive input pixels (>= in_c, multiple of 8) */
    int out_c, ksize, stride, pad;
    int out_h, out_w;
    long long out_pitch; /* elements between consecutive output pixels */
    int act;             /* B2Y_ACT_* */
    float slope;         /* leaky slope (0.1; 0.25 with maxabsscaler, models.py:103) */
    int out_dtype;       /* B2Y_OUT_F16 or B2Y_OUT_F32 */
    long long res_pitch; /* pitch of the residual tensor (ignored when residual == NULL) */
    int w_layout;        /* B2Y_WLAYOUT_*: how w_packed is laid out (0 = [out_c][k][k][in_c]) */
} b2y_conv_desc;

/* Weight layouts of the forward convolutions (b2y_conv2d_fwd / _fwd_stats / b2y_qconv2d_fwd).
 * B2Y_WLAYOUT_S2_PAIRS: 3x3 / stride 2 / pad 1 layers with a narrow, dense input (in_c = 32, in_pitch == in_c, even
 * in_w): the NHWC input is read as pixel PAIRS [B][H][W/2][2*in_c], which turns the layer into a 3(h) x 2(w) window with
 * stride 2 x 1 over 128-byte rows -- 6 im2col boxes per tile instead of 9 half-width ones.  w_packed is
 * [out_c][3][2][2*in_c]: (r, 0, in_c + c) = W[r][0][c], (r, 1, c) = W[r][1][c], (r, 1, in_c + c) = W[r][2][c], rest 0. */
#define B2Y_WLAYOUT_DENSE 0
#define B2Y_WLAYOUT_S2_PAIRS 1

/* y = act(conv(x, w) + bias) [+ residual]
 *   x        fp16 NHWC
 *   w_packed fp16 [out_c][k][k][in_c]  (see b2y_pack_conv_weights)
 *   bias     fp32 [out_c] or NULL
 *   residual fp16 NHWC [.., out_c] or NULL (added after the activation = the following Shortcut layer)
 *   y        fp16 / fp32 NHWC
 * in_c must be a multiple of 16 (the Cin=3 stem uses b2y_stem_conv_fwd). */
int b2y_conv2d_fwd(const b2y_conv_desc* d, const void* x, const void* w_packed, const float* bias,
                   const void* residual, void* y, void* stream);

/* Same GEMM, but also accumulates per-channel sum / sum-of-squares of the *raw* conv output into
 * stat_sum / stat_sqsum (fp32 [out_c], caller zeroes them): the batch statistics of training-mode
 * BatchNorm2d (models.py:100) come out of the conv epilogue instead of two extra passes. */
int b2y_conv2d_fwd_stats(const b2y_conv_desc* d, const void* x, const void* w_packed, const float* bias,
                         void* y, float* stat_sum, float* stat_sqsum, void* stream);

/* First layer (in_c = 1..4, NCHW fp32 image straight from the data loader, models.py:20,92):
 * direct convolution on CUDA cores, fused folded-BN bias + activation, writes NHWC fp16.
 *   x      fp32 NCHW [batch][in_c][in_h][in_w]
 *   w      fp32 [out_c][in_c][k][k]  (BN already folded), bias fp32 [out_c] */
int b2y_stem_conv_fwd(const b2y_conv_desc* d, const float* x_nchw, const float* w, const float* bias, void* y,
                      void* stream);

/* The first layer's tensor-core paths take the (in_c, ksize) pairs with odd ksize and in_c*ksize*ksize <= 32, so
 * that one output pixel's receptive field is one 32-column fp16 GEMM row (B2Y_STEM_IM2COL_SHAPES in csrc/common.cuh;
 * other pairs return B2Y_ERR_UNSUPPORTED and run on b2y_stem_conv_fwd).  The plans choose (b200yolo/layout.py,
 * stem_path): inference takes b2y_stem_conv_fwd_fused when out_c <= 64, else b2y_stem_conv_fwd_tc; training takes
 * b2y_stem_conv_fwd_tc for a stem with BatchNorm, whose weight gradient then runs as a GEMM over the same workspace.
 *
 * im2col stem: the image is written as the im2col matrix [batch*out_h*out_w][32] fp16 (workspace,
 * b2y_stem_workspace_bytes, 0 for a pair off the list), then the conv runs as one k-step GEMM on the wgmma kernel.
 *   w_stem fp16 [out_c][32] from b2y_pack_stem_weights (w already BN-folded, OIHW fp32), column (kh*k + kw)*in_c + c
 *   stat_sum/stat_sqsum optional (training BN statistics, see b2y_conv2d_fwd_stats) */
size_t b2y_stem_workspace_bytes(const b2y_conv_desc* d);
int b2y_pack_stem_weights(const float* w_oihw_folded, int out_c, int in_c, int ksize, void* w_stem, void* stream);
int b2y_stem_conv_fwd_tc(const b2y_conv_desc* d, const float* x_nchw, const void* w_stem, const float* bias,
                         void* workspace, void* y, float* stat_sum, float* stat_sqsum, void* stream);

/* Fused tensor-core stem (the pairs above, out_c <= 64): the CTA builds the im2col tile in shared memory
 * straight from the image and feeds wgmma, so only the image is read and only y is written (no workspace).
 *   x_nchw   NCHW image, x_dtype = B2Y_STEM_X_F32 / _F16 / _U8; value = raw / x_div
 *            (x_div = 256 for uint8 images: reference test.py:95, train.py:348, detect.py:101 "/ 256.0")
 *   w_stem   fp16 [out_c][32] from b2y_pack_stem_weights
 *   y        NHWC fp16 */
#define B2Y_STEM_X_F32 0
#define B2Y_STEM_X_F16 1
#define B2Y_STEM_X_U8 2
int b2y_stem_conv_fwd_fused(const b2y_conv_desc* d, const void* x_nchw, int x_dtype, float x_div, const void* w_stem,
                            const float* bias, void* y, void* stream);
/* Same kernel as the first layer of the INT8 graph (ptq_cos.py:288-296: fp32 conv of the float image with the
 * fake-quantised weights, output requantised): w_stem = b2y_pack_stem_weights of the fake-quantised fp32 weights (exact
 * in fp16), y_i8 = clamp(round_half_away(act(conv + bias_q) / out_scale)) int8 NHWC. */
int b2y_stem_conv_fwd_fused_q(const b2y_conv_desc* d, const void* x_nchw, int x_dtype, float x_div, const void* w_stem,
                              const float* bias_q, void* y_i8, float out_scale, float lo, float hi, void* stream);

/* Fold BatchNorm (running stats) into conv weights and repack OIHW fp32 -> [O][kh][kw][I] fp16.
 *   w_f = w * gamma/sqrt(var+eps);  b_f = beta - gamma*mean/sqrt(var+eps) (+ conv_bias*scale)
 * (utils/torch_utils.py:65-89, utils/quantized/quantized_ptq_cos.py:193-206).
 * gamma==NULL: no BN, bias_out = conv_bias (or 0).  w_fp32_out (optional, OIHW) receives the folded
 * fp32 weights (used by the stem). */
int b2y_pack_conv_weights(const float* w_oihw, const float* conv_bias, const float* gamma, const float* beta,
                          const float* mean, const float* var, float eps, int out_c, int in_c, int ksize,
                          void* w_packed_f16, float* bias_out, float* w_fp32_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Pointwise / data-movement layers (NHWC fp16)
 * ------------------------------------------------------------------------------------------------ */
/* nn.Upsample(scale_factor=s) nearest, models.py:224-225 */
int b2y_upsample_nearest(const void* x, long long x_pitch, void* y, long long y_pitch, int batch, int in_h, int in_w,
                         int c, int scale, void* stream);
/* nn.MaxPool2d(k, stride, (k-1)//2) and the yolov3-tiny ZeroPad2d((0,1,0,1))+MaxPool2d(2,1), models.py:207-215.
 * pad_mode 0: symmetric (k-1)//2 with -inf padding; pad_mode 1: pad right/bottom by one with zeros. */
int b2y_maxpool(const void* x, long long x_pitch, void* y, long long y_pitch, int batch, int in_h, int in_w, int c,
                int ksize, int stride, int pad_mode, void* stream);
/* channel-slice copy (FeatureConcat fallback when a producer cannot write in place), utils/layers.py:26-40 */
int b2y_copy_channels(const void* x, long long x_pitch, void* y, long long y_pitch, long long pixels, int c,
                      void* stream);
/* y = a + b (Shortcut fallback when the add is not fused in the conv epilogue), utils/layers.py:43-72 */
int b2y_add(const void* a, long long a_pitch, const void* b, long long b_pitch, void* y, long long y_pitch,
            long long pixels, int c, int dtype /* B2Y_DT_* */, void* stream);
/* standalone activation fwd/bwd on fp32 (Mish: utils/layers.py:117-128,146-148) */
int b2y_act_fwd_f32(const float* x, float* y, long long n, int act, float slope, void* stream);
int b2y_act_bwd_f32(const float* x, const float* dy, float* dx, long long n, int act, float slope, void* stream);
/* layout converters */
int b2y_nchw_f32_to_nhwc_f16(const float* x, void* y, long long y_pitch, int batch, int c, int h, int w,
                             void* stream);
int b2y_nhwc_f16_to_nchw_f32(const void* x, long long x_pitch, float* y, int batch, int c, int h, int w,
                             void* stream);

/* ------------------------------------------------------------------------------------------------
 * YOLO head: models.py:350-437 (YOLOLayer.forward)
 *   raw : fp32 [batch][ny][nx][raw_pitch] head-conv output, channel = a*no + o
 *   p   : fp32 [batch][na][ny][nx][no]  (the "training output", models.py:406)      (may be NULL)
 *   io  : fp32 rows of a [batch][total_rows][no] tensor; this layer fills rows
 *         [row_offset, row_offset + na*ny*nx) with row = a*ny*nx + y*nx + x             (may be NULL)
 *         xy=(sigmoid+grid)*stride, wh=exp*anchor_px, obj/cls=sigmoid  (models.py:415-418)
 * ------------------------------------------------------------------------------------------------ */
int b2y_yolo_decode(const float* raw, long long raw_pitch, float* p, float* io, long long total_rows,
                    long long row_offset, int batch, int na, int no, int ny, int nx, const float* anchors_px,
                    float stride, void* stream);

/* ------------------------------------------------------------------------------------------------
 * YOLO loss: utils/utils.py:368-432 (compute_loss), 725-779 (build_targets), 254-297 (bbox_iou)
 * Single yolo layer; the host sums the three layers and applies the hyp gains.
 *   p        fp32 [batch][na][ny][nx][no]
 *   targets  fp32 [nt][6] (image, class, x, y, w, h) normalised
 *   anchors  fp32 [na][2] = anchors_px / stride  (YOLOLayer.anchor_vec)
 *   out[0]=sum(1-giou) out[1]=matches out[2]=sum BCE(cls) out[3]=sum BCE(obj) (fp32[4], overwritten)
 *   dp       fp32 same shape as p: d(lbox*w_box + lobj*w_obj + lcls*w_cls)/dp with the reference's
 *            'mean' reductions (NULL = forward only)
 *   fl_gamma hyp['fl_gamma']: > 0 wraps the class and objectness BCE in the focal loss (utils/utils.py:333-360,
 *            alpha 0.25); 0 = plain BCE.  Negative or NaN: B2Y_ERR_INVALID
 *   workspace: b2y_yolo_loss_workspace_bytes(...) bytes
 * ------------------------------------------------------------------------------------------------ */
size_t b2y_yolo_loss_workspace_bytes(int batch, int na, int ny, int nx, int nt);
int b2y_yolo_loss(const float* p, const float* targets, int nt, const float* anchors, int batch, int na, int no,
                  int ny, int nx, float iou_t, float gr, float cls_pw, float obj_pw, float w_box, float w_obj,
                  float w_cls, float fl_gamma, float* out4, float* dp, void* workspace, void* stream);
/* build_targets only: writes up to na*nt matches in reference order (anchor-major, target-minor);
 *   idx int64 [4][na*nt] rows (b, a, gj, gi), tbox fp32 [na*nt][4], tcls int64 [na*nt], count int32[1].
 *   Candidates with b outside [0, batch) or a cell off the ny x nx grid are dropped, as b2y_yolo_loss drops them. */
int b2y_build_targets(const float* targets, int nt, const float* anchors, int batch, int na, int ny, int nx,
                      float iou_t, long long* idx, float* tbox, long long* tcls, int* count, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Quantisation (power-of-two scale fake-quant, BN fold, INT8 conv):
 * utils/quantized/quantized_ptq_cos.py:14-113,131-738; utils/quantized/quantized_google.py:81-219
 * ------------------------------------------------------------------------------------------------ */
/* y = clamp(round_half_away(x/scale), lo, hi) * scale   (ptq_cos.py:89-92) */
int b2y_fakequant_f32(const float* x, float* y, long long n, float scale, float lo, float hi, void* stream);
/* q = int8(clamp(round_half_away(x/scale), lo, hi)) from fp16 NHWC -> int8 NHWC */
int b2y_quantize_f16_to_i8(const void* x, long long x_pitch, void* q, long long q_pitch, long long pixels, int c,
                           float scale, float lo, float hi, void* stream);
/* COSPTQ scale search (ptq_cos.py:71-87): for each candidate step i-5, i in [0,n_cand): cosine similarity
 * between x and fakequant(x; 2^step/2^(bits-1)); out_cos fp32 [n_cand]. One pass over x. */
int b2y_cos_scale_search(const float* x, long long n, int bits, int n_cand, float* out_cos, void* workspace,
                         size_t workspace_bytes, void* stream);
/* same with the first candidate's exponent given: candidate k quantises with float_range = 2^(k + step0) */
int b2y_cos_scale_search_ex(const float* x, long long n, int bits, int n_cand, int step0, float* out_cos,
                            void* workspace, size_t workspace_bytes, void* stream);
/* per-tensor or per-channel min/max (google.py:16-77); x fp32 [rows][cols], per_row!=0 -> out [rows][2] */
int b2y_minmax_f32(const float* x, long long rows, long long cols, int per_row, float* out_minmax, void* stream);

typedef struct b2y_qconv_desc {
    b2y_conv_desc conv;   /* shapes as for the dense conv; x/w are int8, in_c multiple of 32 */
    float acc_scale;      /* s_act * s_weight (both powers of two) */
    float out_scale;      /* activation quantiser scale of this layer's output */
    float q_lo, q_hi;     /* clamp range, -2^(b-1) .. 2^(b-1)-1 */
    int out_kind;         /* B2Y_OUT_I8: requantised int8; B2Y_OUT_F32/F16: fake-quant value (heads: linear) */
    int requant;          /* 0: write act(acc*acc_scale+bias) without requantisation (linear head, ptq_cos.py:718) */
    int clamp_addends;    /* b2y_qconv2d_shortcut_fwd only.  0: the addends are rounded onto scale_x / scale_a but not
                             clamped (COSPTQuantizedShortcut, google QuantizedShortcut_min); 1: their codes are also clamped
                             to [sum_lo, sum_hi] before the add (google QuantizedShortcut_max, quantized_google.py:294) */
} b2y_qconv_desc;
/* INT8 conv on int8 wgmma with int32 accumulation (exact whenever the fp32 reference is). */
int b2y_qconv2d_fwd(const b2y_qconv_desc* d, const void* x_i8, const void* w_i8, const float* bias, void* y,
                    void* stream);
/* The same conv with the FOLLOWING quantised shortcut layer (ptq_cos.py:876-884 _min / 931-933 _max, eval) folded into its
 * epilogue: y = clamp(round((round(q*out_scale/scale_x)*scale_x + round(a*sa_in/scale_a)*scale_a) / scale_sum)), q being
 * this conv's int8 code and a the other addend's codes (NHWC int8, pitch a_pitch).  Bit-identical to b2y_qconv2d_fwd
 * followed by b2y_qshortcut_i8.  Returns B2Y_ERR_UNSUPPORTED (nothing launched) unless every scale is a power of two and
 * the layer qualifies for the short epilogue (whole channel tiles, 16-byte aligned tensors): run the two calls then. */
int b2y_qconv2d_shortcut_fwd(const b2y_qconv_desc* d, const void* x_i8, const void* w_i8, const float* bias,
                             const void* a_i8, long long a_pitch, float sa_in, float scale_x, float scale_a,
                             float scale_sum, float sum_lo, float sum_hi, void* y, void* stream);
/* BN-fold + weight quantisation + pack: OIHW fp32 -> int8 [O][kh][kw][I] with scale w_scale (ptq_cos.py:193-212) */
int b2y_pack_qconv_weights(const float* w_oihw_folded, int out_c, int in_c, int ksize, float w_scale, float lo,
                           float hi, void* w_i8, void* stream);

/* int8 graph glue (eval): quantised shortcut (ptq_cos.py:876-884, 931-933), concat requantisation (ptq_cos.py:1540-1546),
 * nearest upsample of codes, and the fp32 first layer with int8 output (the image is not on an int8 grid) */
int b2y_qshortcut_i8(const void* x, long long x_pitch, const void* a, long long a_pitch, void* out, long long out_pitch,
                     long long pixels, int c, float sx_in, float scale_x, float sa_in, float scale_a, float scale_sum,
                     float lo, float hi, void* stream);
int b2y_requant_i8(const void* x, long long x_pitch, void* out, long long out_pitch, long long pixels, int c,
                   float s_in, float s_out, float lo, float hi, void* stream);
int b2y_upsample_nearest_i8(const void* x, long long x_pitch, void* y, long long y_pitch, int batch, int in_h,
                            int in_w, int c, int scale, void* stream);
/* Max-pool of int8 NHWC codes: the plain nn.MaxPool2d (and ZeroPad2d((0,1,0,1)) + MaxPool2d(2, 1)) that the google-QAT
 * graph keeps over fake-quantised values (models.py:207-214).  Same shapes and pad_mode as b2y_maxpool: 0 = symmetric
 * (k-1)//2 padding with -inf, 1 = one zero row / column on the right and bottom (a zero value is code 0 on any grid).
 * c a multiple of 16, pitches multiples of 16 and >= c, x and y 16-byte aligned; y_pitch may exceed c (a concat slot). */
int b2y_maxpool_i8(const void* x, long long x_pitch, void* y, long long y_pitch, int batch, int in_h, int in_w, int c,
                   int ksize, int stride, int pad_mode, void* stream);
int b2y_stem_conv_fwd_q(const b2y_conv_desc* d, const float* x_nchw, const float* w_q, const float* bias_q, void* y_i8,
                        float out_scale, float lo, float hi, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Training: BatchNorm (batch statistics), backward convolutions, optimiser
 * models.py:92-113 under autograd; train.py:135-151,437-459
 * ------------------------------------------------------------------------------------------------ */
/* per-channel gradient reduce of y = act(x*scale[c] + shift[c]):  given dy (grad wrt y) and x, recompute
 * z = x*scale+shift, du = dy*act'(z); dbeta = sum(du), dgamma = sum(du*xhat) with xhat = (x-mean)*invstd
 * (mean / invstd optional: 0 / 1).  The BatchNorm layers of the conv stack use b2y_bn_train_bwd_reduce instead. */
int b2y_bn_act_bwd_reduce(const void* x, long long x_pitch, const void* dy, long long dy_pitch, const float* scale,
                          const float* shift, const float* save_mean, const float* save_invstd, float* dgamma,
                          float* dbeta, float* du_absmax /* optional: atomicMax of |du|, caller zeroes */,
                          long long pixels, int c, int act, float slope, int grad_dtype, void* stream);
/* dX = conv_transpose(dY, W)   (data gradient; implicit GEMM on wgmma) */
int b2y_conv2d_bwd_data(const b2y_conv_desc* d, const void* dy, const void* w_packed_t, void* dx, int accumulate,
                        int operand_dtype /* dY and weights */, int out_dtype /* dX */,
                        const float* inv_scale_ptr /* optional device scalar multiplied into dX */, void* stream);
/* weights for b2y_conv2d_bwd_data: OIHW fp32 -> per output-phase slabs [phase][in_c][tap][out_c] fp16
 * (stride-s data gradients are decomposed into s*s stride-1 implicit GEMMs over dY; out_c*ksize^2*in_c elements) */
int b2y_pack_dgrad_weights(const b2y_conv_desc* d, const float* w_oihw, void* w_packed_t, int grad_dtype,
                           void* stream);
/* dW[o][kh][kw][i] += scale * sum_pixels dY[p][o] * X[p@(kh,kw)][i]  (weight gradient, wgmma GEMM over the pixel
 * dimension with MN-major operands; dw fp32 [O][kh][kw][I], caller zeroes it).  The split-K partial sums are added in
 * double into an accumulator that belongs to the calling (device, stream) and then rounded into dw, so the result does
 * not depend on the order of the atomics; calls on different streams may run concurrently (the same holds for the
 * batch statistics of b2y_conv2d_fwd_stats / b2y_stem_conv_fwd_tc, b2y_bn_train_bwd_reduce, b2y_bn_act_bwd_reduce and
 * b2y_stem_conv_bwd_weight).  The first call on a stream allocates its accumulator. */
int b2y_conv2d_bwd_weight(const b2y_conv_desc* d, const void* x, const void* dy, float* dw, float scale,
                          int operand_dtype /* X and dY */, const float* inv_scale_ptr, void* stream);
/* [O][kh][kw][I] fp32 -> OIHW fp32 parameter-gradient layout: dst = alpha*src (+ dst if accumulate) */
int b2y_unpack_wgrad(const float* dw_packed, float* dw_oihw, int out_c, int in_c, int ksize, float alpha,
                     int accumulate, void* stream);
/* dst = alpha*src + beta*dst (fp32) */
int b2y_axpby_f32(const float* src, float* dst, long long n, float alpha, float beta, void* stream);
/* backward of the YOLO permute: dp fp32 [B][na][ny][nx][no] -> d(raw) fp16 [B][ny][nx][raw_pitch] * scale (models.py:406) */
int b2y_yolo_grad_to_raw(const float* dp, void* draw, long long raw_pitch, int batch, int na, int no, int ny, int nx,
                         float scale, const float* scale_ptr /* optional device scalar */, int grad_dtype,
                         void* stream);
/* backward of nn.Upsample (nearest): dx += window sums of dy (in place accumulate) */
int b2y_upsample_nearest_bwd(const void* dy, long long dy_pitch, void* dx, long long dx_pitch, int batch, int in_h,
                             int in_w, int c, int scale, int grad_dtype, void* stream);
/* backward of nn.MaxPool2d: dx[argmax] += dy (arg-max recomputed from x; first maximum wins like torch) */
int b2y_maxpool_bwd(const void* x, long long x_pitch, const void* dy, long long dy_pitch, void* dx,
                    long long dx_pitch, int batch, int in_h, int in_w, int c, int ksize, int stride, int pad_mode,
                    int grad_dtype, void* stream);
/* weight gradient of the stem (in_c <= 4, in_c*ksize*ksize <= 40): x fp32 NCHW, dz fp16 NHWC -> dw OIHW fp32 (+= scale * ...) */
int b2y_stem_conv_bwd_weight(const b2y_conv_desc* d, const float* x_nchw, const void* dz, float* dw_oihw,
                             float scale, int grad_dtype, void* stream);

/* ---- grouped optimiser steps over the flat buffers (train.py:120-150 parameter groups, :356-365 burn-in) ----
 * One CTA per tile of a device-resident tile table.  A tile is a run of elements of ONE parameter tensor, so its group
 * (and whether the BatchNorm-L1 term applies, prune_utils.py:133-138) is uniform over the CTA.  flags: bits 0-1 the
 * group index into B2YOptStep.group, bit 2 the L1 term.  At most B2Y_OPT_TILE elements per tile.  Every buffer is a
 * flat fp32 buffer with the same element layout and a 16-byte-aligned base. */
#define B2Y_OPT_MAX_GROUPS 4
#define B2Y_OPT_TILE 4096
#define B2Y_OPT_TILE_L1 4
typedef struct {
    long long start;
    int len;
    int flags;
} B2YOptTile;
typedef struct {
    float lr, momentum, weight_decay;        /* SGD; Adam uses weight_decay (L2, added to the gradient) */
    float one_minus_beta1, beta2, one_minus_beta2, eps; /* Adam; the complements are rounded from double on the host */
    float step_size, bc2_sqrt; /* Adam: lr / (1 - beta1^t) and sqrt(1 - beta2^t), computed in double on the host */
} B2YOptGroup;
typedef struct {
    B2YOptGroup group[B2Y_OPT_MAX_GROUPS];
    float grad_scale; /* 1/world after the NCCL sum */
    float l1_coeff;   /* s / grad_scale for tiles with B2Y_OPT_TILE_L1 (updateBN runs on the averaged gradient) */
    float ema_decay;  /* ModelEMA d of this update, used when `ema` is not NULL */
    int first_step;   /* SGD: the momentum buffer does not exist yet (torch: buf = grad) */
} B2YOptStep;
/* Nesterov SGD per group (torch.optim.SGD, nesterov=True, dampening=0, train.py:135-144), gradients scaled by
 * grad_scale:  g = grad*grad_scale + wd*p ; buf = first_step ? g : mu*buf + g ; p -= lr * (g + mu*buf).
 * `ema` (optional): ema = d*ema + (1-d)*p_new (utils/torch_utils.py:171-183).  `hp` is read on the host and passed to
 * the kernel by value. */
int b2y_sgd_grouped(float* param, const float* grad, float* momentum_buf, float* ema, const B2YOptTile* tiles_dev,
                    int n_tiles, const B2YOptStep* hp, void* stream);
/* Adam per group (torch.optim.Adam, amsgrad=False, maximize=False, L2 weight decay); same tiles, EMA and L1 terms */
int b2y_adam_grouped(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, float* ema,
                     const B2YOptTile* tiles_dev, int n_tiles, const B2YOptStep* hp, void* stream);

/* ---- bandwidth-oriented BatchNorm passes of the training step (csrc/bn_train.cu; models.py:100-113 under autograd) ----
 * save = fp32 [4][c]: batch mean, invstd, scale = gamma*invstd, shift = beta - mean*scale.
 * forward: derives them from the conv epilogue's channel sums (biased variance), updates the running statistics
 * (unbiased variance, `momentum`), writes `save` and y = act(z*scale+shift) [+ residual] in the same launch. */
int b2y_bn_train_fwd(const void* z, long long z_pitch, const float* stat_sum, const float* stat_sqsum, long long count,
                     const float* gamma, const float* beta, float eps, float momentum, float* running_mean,
                     float* running_var, float* save, const void* residual, long long res_pitch, void* y,
                     long long y_pitch, long long pixels, int c, int act, float slope, void* stream);
/* The same at a channel-pruned width: z, y, the residual, the statistics and `save` are c wide (c % 8 == 0), the
 * BatchNorm has c_logical channels (c - 8 < c_logical <= c).  Channels c_logical .. c-1 get y = 0 (scale and shift 0,
 * the residual's pad is zero); gamma, beta and the running statistics are read and written at [0, c_logical) only, and
 * `save` entries of the pad channels are not written.  b2y_bn_train_fwd is this with c_logical = c. */
int b2y_bn_train_fwd_lw(const void* z, long long z_pitch, const float* stat_sum, const float* stat_sqsum,
                        long long count, const float* gamma, const float* beta, float eps, float momentum,
                        float* running_mean, float* running_var, float* save, const void* residual, long long res_pitch,
                        void* y, long long y_pitch, long long pixels, int c, int c_logical, int act, float slope,
                        void* stream);
/* sums = fp32 [2][c] (caller zeroes): S1 = sum du, S2 = sum du*xhat with du = dy*act'(z*scale+shift).
 * du_absmax (optional) = fp32 [4], caller zeroes: [0] = max|du| and [3] = max|xhat| over the layer (atomicMax);
 * [1] and [2] are left to b2y_bn_train_bwd_apply's scale_out. */
int b2y_bn_train_bwd_reduce(const void* z, long long z_pitch, const void* dy, long long dy_pitch, const float* save,
                            float* sums, float* du_absmax /* optional fp32 [4], see above */,
                            long long pixels, int c, int act, float slope, int grad_dtype, void* stream);
/* dz = s * gamma*invstd*(du - S1/N - xhat*S2/N) as fp16 (s = power of two chosen on the device -> scale_out[0..1] =
 * [s, 1/s]); also emits the parameter gradients dgamma_out = S2*grad_out_scale, dbeta_out = S1*grad_out_scale.
 * s maps the bound max_c |gamma*invstd| * (max|du| + |S1|/N + max|xhat|*|S2|/N) >= max|dz| to at most 2^12, with
 * max|du| and max|xhat| read from the reduce's du_absmax[0] and [3]; without du_absmax they are taken as 1 and
 * sqrt(pixels). */
int b2y_bn_train_bwd_apply(const void* z, long long z_pitch, const void* dy, long long dy_pitch, const float* gamma,
                           const float* save, const float* sums, void* dz, long long dz_pitch, long long pixels, int c,
                           int act, float slope, int grad_dtype, const float* du_absmax, float* scale_out,
                           float* dgamma_out, float* dbeta_out, float grad_out_scale, void* stream);
/* fp32 NHWC BatchNorm + activation of the float depthwise blocks of a google-QAT graph (models.py:183-197 under
 * quantized=1): z, y dense [pixels][c], any c.  training = 1: batch statistics (biased variance) normalise, the running
 * statistics are updated with the unbiased variance and `momentum`; training = 0: the running statistics normalise.
 * save = fp32 [4][c] as above.  Sums over pixels are taken in a fixed order in double: two runs give the same bits. */
int b2y_bn_f32_fwd(const float* z, long long pixels, int c, const float* gamma, const float* beta, float eps,
                   float momentum, float* running_mean, float* running_var, int training, float* save, float* y, int act,
                   float slope, void* stream);
/* dz = gamma*invstd*(du - S1/N - xhat*S2/N) (training) or gamma*invstd*du (eval), du = dy*act'(z*scale+shift);
 * dbeta = S1 = sum du, dgamma = S2 = sum du*xhat (overwritten).  coef = fp32 [3][c] scratch. */
int b2y_bn_f32_bwd(const float* z, const float* dy, long long pixels, int c, const float* gamma, const float* save,
                   int training, float* coef, float* dz, float* dgamma, float* dbeta, int act, float slope, void* stream);

/* ---- table-driven layout kernels (csrc/multi.cu): one launch for ALL convolutions of a model ----
 * Tiles: 32 output channels x b2y_layout_tile_i(k) input channels x k*k taps; tile_begin = running sum of
 * ceil(rows/32) * ceil(in_c / tile_i) over the items (rows = out_c_pad for packing, out_c for unpacking). */
typedef struct b2y_pack_item {
    const float* w;     /* master weights, OIHW fp32 [out_c][in_c][k][k] */
    void* w_fwd;        /* fp16 [out_c_pad][k][k][in_c_pad] (rows >= out_c zero; columns >= in_c untouched) or NULL */
    void* w_dgrad;      /* fp16 [phase][in_c][tap][out_c_pad] (see b2y_pack_dgrad_weights) or NULL */
    int O, Opad, I, k, stride, pad;
    int tile_begin, Ipad; /* Ipad = row length of w_fwd (in_c rounded up to the MMA K granule of 16) */
    const int* col_map; /* device int [in_c]: the w_fwd column of each input channel, or NULL for the identity.  With a
                         * map, the columns no input channel maps to are left untouched (zero in a zero-filled buffer):
                         * the pad channels of a channel-pruned source and the gaps between the sources of a concat */
} b2y_pack_item;
typedef struct b2y_unpack_item {
    const float* src;   /* packed weight gradient fp32 [out_c_pad][k][k][in_c_pad] */
    float* dst;         /* OIHW fp32 [out_c][in_c][k][k] */
    int O, I, k, accumulate;
    int tile_begin, Ipad;
} b2y_unpack_item;
int b2y_layout_tile_i(int ksize);
int b2y_pack_conv_weights_multi(const b2y_pack_item* items_dev, int n_items, int total_tiles, void* stream);
int b2y_unpack_wgrad_multi(const b2y_unpack_item* items_dev, int n_items, int total_tiles, void* stream);

/* ---- depthwise convolution + squeeze-excite (csrc/depthwise.cu): the `depthwise` / `se` cfg blocks of the MobileNet
 * backbones, models.py:115-197, utils/layers.py:176-192.  NHWC fp16, channels % 8 == 0, weights are the fp32 module
 * parameters themselves (Conv2d(groups=C).weight [C][1][k][k]; Linear weights [C/4][C], [C][C/4]). ---- */
/* y = act(dwconv(x, w) * scale[c] + bias[c])  (scale / bias optional: folded BatchNorm for inference); training passes
 * act = linear, scale = bias = NULL and the channel sums (sum z, sum z^2; caller zeroes) of the raw output */
int b2y_dwconv_fwd(const b2y_conv_desc* d, const void* x, const float* w, const float* scale, const float* bias, void* y,
                   float* stat_sum, float* stat_sqsum, void* stream);
/* dx (+)= inv_scale * dwconv^T(dz, w)   dz fp16 NHWC [B][out_h][out_w][c], dx fp16 / bf16 [B][in_h][in_w][c] */
int b2y_dwconv_bwd_data(const b2y_conv_desc* d, const void* dz, const float* w, void* dx, int accumulate,
                        int out_dtype, const float* inv_scale_ptr, void* stream);
/* dw[c][k][k] += alpha * inv_scale * sum_pixels dz * x   (fp32, caller zeroes) */
int b2y_dwconv_bwd_weight(const b2y_conv_desc* d, const void* x, const void* dz, float* dw, float alpha,
                          const float* inv_scale_ptr, void* stream);
/* SE forward: y = x * hsigmoid(W2 relu(W1 mean_hw(x))).  ws = fp32 [batch][3c + cr] scratch that the backward reads
 * (mean [batch][c] | pre-activation v [batch][c] | gate s [batch][c] | h [batch][cr]: s, read with 16-byte loads, stays
 * aligned for every batch) */
int b2y_se_fwd(const void* x, long long x_pitch, const float* w1, const float* w2, void* y, long long y_pitch, int batch,
               int hw, int c, int cr, float* ws, void* stream);
/* SE backward: dx (+)= dy*s + dmean/hw;  dw1 [cr][c], dw2 [c][cr] = grad_scale * gradients (overwritten) */
int b2y_se_bwd(const void* x, long long x_pitch, const void* dy, long long dy_pitch, const float* w1, const float* w2,
               const float* ws, float* ws_bwd /* fp32 [batch][3c + cr] */, void* dx, long long dx_pitch, int accumulate,
               float* dw1, float* dw2, float grad_scale, int batch, int hw, int c, int cr, int grad_dtype, void* stream);
/* fp32 versions for the float depthwise / SE layers of a google-QAT graph: dense NHWC fp32 (pitch = c), any c, sums over
 * pixels in a fixed order (two runs give the same bits).
 * z = dwconv(x, w) + bias[c] (bias optional) */
int b2y_dwconv_fwd_f32(const b2y_conv_desc* d, const float* x, const float* w, const float* bias, float* z, void* stream);
/* dx = dwconv^T(dz, w) and dw[c][k][k] = sum_pixels dz * x, both overwritten; either may be NULL */
int b2y_dwconv_bwd_f32(const b2y_conv_desc* d, const float* x, const float* dz, const float* w, float* dx, float* dw,
                       void* stream);
/* per-channel batch mean and unbiased variance (torch.var) of z = dwconv(x, w) + bias[c] (bias optional), z recomputed,
 * not stored; sums in double (the statistics conv of a TPSQ depthwise layer, quantized_TPSQ.py:416-420) */
int b2y_dwconv_stats_f32(const b2y_conv_desc* d, const float* x, const float* w, const float* bias, float* mean,
                         float* var, void* stream);
/* backward of those statistics: gs = g_mean[c] / n + 2 g_var[c] (z - mean[c]) / (n - 1) (z recomputed; g_mean / g_var
 * optional, n = batch * out_h * out_w) into the workspace gs [batch][out_h][out_w][c]; then
 * dx = dwconv^T(gs, w) + dwconv^T(dz2, w2) in one gather (dz2 / w2 optional: the layer's quantised conv on the same input)
 * and dw[c][k][k] = sum_pixels gs * x.  dx and dw are overwritten; either may be NULL */
int b2y_dwconv_stats_bwd_f32(const b2y_conv_desc* d, const float* x, const float* w, const float* bias, const float* mean,
                             const float* g_mean, const float* g_var, const float* dz2, const float* w2, float* gs,
                             float* dx, float* dw, void* stream);
/* ws layout as b2y_se_fwd */
int b2y_se_fwd_f32(const float* x, const float* w1, const float* w2, float* y, int batch, int hw, int c, int cr, float* ws,
                   void* stream);
/* dx = dy*s + dmean/hw, dw1 [cr][c], dw2 [c][cr] (all overwritten) */
int b2y_se_bwd_f32(const float* x, const float* dy, const float* w1, const float* w2, const float* ws, float* ws_bwd,
                   float* dx, float* dw1, float* dw2, int batch, int hw, int c, int cr, void* stream);

/* ---- quantisation-aware training pieces (csrc/quant.cu) ----
 * straight-through backward of b2y_fakequant_f32 (google.py:81-92, 124-143): dx = g * [lo <= round(x/s) <= hi] * gain */
int b2y_fakequant_bwd_f32(const float* x, const float* g, float* dx, long long n, float scale, float lo, float hi,
                          float gain, void* stream);
/* TPSQ quantiser (quantized_TPSQ.py:66-130) with the power-of-two range P = Search_Pow2(scale):
 * y = round(softclamp(x, P) * (2^(b-1) - 1) / P) * P / 2^(b-1); backward gives dx and sum(g * dy/dP) (double) */
int b2y_tpsq_fwd_f32(const float* x, float* y, long long n, float range_pow2, int bits, void* stream);
int b2y_tpsq_bwd_f32(const float* x, const float* g, float* dx /* may be NULL */, double* dp_sum, long long n,
                     float range_pow2, int bits, void* stream);

/* ---- detection post-processing (csrc/nms.cu): replaces utils.utils.non_max_suppression (utils/utils.py:782-860) and the
 * true-positive matching loop of test.py:137, 150-170.  Two calls because the number of candidates is data dependent:
 *   1. b2y_nms_count: per-row candidate counts -> exclusive scan row_off [batch*rows + 1] and img_off [batch + 1]
 *      (device; the caller reads img_off[batch] = total to size the buffers of step 2)
 *   2. b2y_nms_run: candidates in nonzero() order, stable descending score sort per image, greedy suppression with
 *      torchvision's arithmetic (fp32 IoU, threshold compared in double), merge-NMS for 1 < n < 3000.
 * pred fp32 [batch][rows][5 + nc] (xywh px, obj, class probabilities).  det fp32 [total][6]: image b owns rows
 * img_off[b] .. img_off[b] + det_count[b] (x1, y1, x2, y2, conf, cls), in descending score order.
 * class_allow: NULL or uint8 [nc] (the `classes=` filter).  multi_label is forced off for nc == 1 like the reference. */
size_t b2y_nms_count_workspace_bytes(int batch, int rows);
int b2y_nms_count(const float* pred, int batch, int rows, int nc, float conf_thres, int multi_label,
                  const unsigned char* class_allow, int* row_off, int* img_off, void* workspace, size_t workspace_bytes,
                  void* stream);
size_t b2y_nms_run_workspace_bytes(long long total);
int b2y_nms_run(const float* pred, int batch, int rows, int nc, float conf_thres, double iou_thres, int multi_label,
                int agnostic, const unsigned char* class_allow, const int* row_off, const int* img_off, long long total,
                void* workspace, size_t workspace_bytes, float* det, int* det_count, void* stream);
/* test.py:137 + 150-170 for a whole batch: boxes clipped in place to [0, clip_w] x [0, clip_h] (skipped if clip_w <= 0),
 * then per image and class the predictions (in their given = score order) claim their best-IoU target once;
 * correct uint8 [n_det][niou] = (best IoU > iouv[q]) for the winners, 0 elsewhere.  det_off / det_count int32 [batch],
 * lab_off int32 [batch + 1] into tcls fp32 [n_lab] / tbox fp32 [n_lab][4] (xyxy px, 16-byte aligned). */
size_t b2y_tp_match_workspace_bytes(long long n_det, long long n_lab);
int b2y_tp_match(float* det, const int* det_off, const int* det_count, long long n_det, const float* tcls,
                 const float* tbox, const int* lab_off, long long n_lab, const float* iouv, int niou, int batch,
                 float clip_w, float clip_h, void* workspace, size_t workspace_bytes, unsigned char* correct,
                 void* stream);

/* ---- knowledge-distillation losses of the YOLO head (csrc/kd.cu; utils/utils.py:435-520 compute_lost_KD / KD2 / KD3) ----
 * soft targets: loss_acc[0] += sum over rows of KL(softmax(teacher / T) || softmax(student / T)) over `width` columns
 * starting at col0 of rows of row_len floats; dstudent (NULL or same shape as student) receives
 * (softmax(student / T) - softmax(teacher / T)) * grad_scale / T in those columns (other columns untouched). */
int b2y_kd_soft_rows(const float* student, const float* teacher, long long rows, int row_len, int col0, int width,
                     float temperature, float grad_scale, double* loss_acc, float* dstudent, void* stream);
/* box term on the n matched cells of b2y_build_targets (idx int64 [4][n] = image, anchor, gy, gx; tbox fp32 [n][4];
 * anchor_vec fp32 [na][2]; student / teacher fp32 [batch][na][ny][nx][no]).  mode 2 (KD2): squared distance to the
 * target box where it exceeds the teacher's (+ reg_m), reg_num counts those cells; mode 3 (KD3..5): squared distance to
 * the teacher's box.  loss_acc[0] += the sum; dstudent[cell][0..3] += gradient * grad_scale (atomic: duplicate cells add). */
int b2y_kd_box(const float* student, const float* teacher, const long long* idx, const float* tbox,
               const float* anchor_vec, int n, int na, int ny, int nx, int no, int mode, float reg_m, float grad_scale,
               double* loss_acc, int* reg_num, float* dstudent, void* stream);

/* ---- input pipeline, inference slice (csrc/preprocess.cu): datasets.letterbox (utils/datasets.py:611-646: cv2.resize
 * INTER_LINEAR to resized_w x resized_h, cv2.copyMakeBorder with `color`) fused with the loaders' BGR -> RGB / HWC -> CHW
 * shuffle (datasets.py:113).  src uint8 HWC [src_h][src_w][channels] (row pitch in bytes), dst uint8 planar
 * [channels][dst_h][dst_w] with the resized image at (top, left); swap_rb reverses the channel order.  Bit-identical to
 * OpenCV's fixed-point 8-bit INTER_LINEAR (resized == source size: plain copy). */
int b2y_letterbox_u8(const unsigned char* src, int src_h, int src_w, int channels, long long src_pitch, int resized_h,
                     int resized_w, int top, int left, unsigned char* dst, int dst_h, int dst_w, int swap_rb, int color,
                     void* stream);
/* One evaluation batch of LoadImagesAndLabels(rect=True) (utils/datasets.py:419-475, 511-531) in ONE launch: per item,
 * load_image's cv2.resize INTER_AREA of the source to rs_w x rs_h (rs == source size: plain copy), placed at (top, left)
 * of a dst_h x dst_w plane of `color` (letterbox with auto=False, scaleup=False only pads on this path), channel order
 * reversed when swap_rb, into slot `slot` of dst uint8 planar [batch][channels][dst_h][dst_w].  Bit-identical to OpenCV's
 * 8-bit INTER_AREA: integer factors (area_kx, area_ky > 0, used by cv::resize when both scales are integers within
 * DBL_EPSILON) average the block, other sizes take the fractional path (area_kx = area_ky = 0).
 * items: host table, checked (B2Y_ERR_INVALID, nothing launched, for a bad item: a size that does not fit, a scale that
 * is not 1. / ((double)rs / src), integer factors where cv::resize would not use them or vice versa, a slot out of
 * range); items_dev: the same n_items items in device memory, which the kernel reads. */
typedef struct b2y_load_item {
    const unsigned char* src;   /* device, HWC uint8 [src_h][src_w][channels] */
    long long src_pitch;        /* bytes per source row */
    int src_h, src_w;
    int rs_h, rs_w;             /* size after INTER_AREA */
    int area_kx, area_ky;       /* integer factors of the block-mean path, or 0 */
    double scale_x, scale_y;    /* src_w / rs_w, src_h / rs_h as cv::resize computes them */
    int top, left;              /* border */
    int slot;                   /* batch index written */
    int reserved;
} b2y_load_item;
int b2y_load_batch_u8(const b2y_load_item* items, const b2y_load_item* items_dev, int n_items, unsigned char* dst,
                      int batch, int channels, int dst_h, int dst_w, int swap_rb, int color, void* stream);

/* ---- input pipeline, training slice (csrc/preprocess.cu): LoadImagesAndLabels(augment=True).__getitem__
 * (utils/datasets.py:419-501) as two table-driven launches per batch.  b2y_mosaic_u8 builds load_mosaic's canvases
 * (:553-608): canvas slot `slot` of canvas uint8 HWC [batch][2s][2s][channels] is 114 outside the four tiles' rectangles
 * [x1a, x2a) x [y1a, y2a), and inside tile k the pixel (x + dx, y + dy) of load_image's tile: the source itself when
 * rs == source size, else cv2.resize(INTER_LINEAR) of the source to rs_w x rs_h (bit-identical to OpenCV's 8-bit fixed
 * point; an exact 2x downscale, which cv::resize computes as INTER_AREA, gives the same bytes).  Later tiles win where
 * rectangles overlap, as numpy's assignments in tile order do.
 * b2y_affine_hsv_u8 builds the batch from the canvases: per item, cv2.warpAffine(canvas, M, (s, s), INTER_LINEAR,
 * borderValue=114) (random_affine, :649-715) with im = invertAffineTransform(M); when hsv (colour only), augment_hsv's
 * BGR2HSV -> lut[0..255] (hue), lut[256..511] (saturation), lut[512..767] (value) -> HSV2BGR (:534-545, OpenCV's
 * default 8-bit dispatch); the left-right flip when flip; channels reversed (BGR -> RGB) into slot `slot` of dst uint8
 * planar [batch][channels][s][s].
 * items: host tables, checked (B2Y_ERR_INVALID, nothing launched, for a bad item: a null source, a pitch or a tile size
 * that does not fit, a scale that is not 1. / ((double)rs / src), a rectangle outside the canvas or reading outside its
 * tile, a map whose coordinates overflow OpenCV's fixed point, hsv on a gray-scale batch, a slot out of range);
 * items_dev: the same n_items items in device memory, which the kernels read. */
typedef struct b2y_mosaic_tile {
    const unsigned char* src;   /* device, HWC uint8 [src_h][src_w][channels] */
    long long src_pitch;        /* bytes per source row */
    int src_h, src_w;
    int rs_h, rs_w;             /* load_image's tile size */
    double scale_x, scale_y;    /* src_w / rs_w, src_h / rs_h as cv::resize computes them */
    int x1a, y1a, x2a, y2a;     /* rectangle on the canvas */
    int dx, dy;                 /* tile pixel = canvas pixel + (dx, dy) */
} b2y_mosaic_tile;
typedef struct b2y_mosaic_item {
    b2y_mosaic_tile tiles[4];
    int slot;
    int reserved;
} b2y_mosaic_item;
int b2y_mosaic_u8(const b2y_mosaic_item* items, const b2y_mosaic_item* items_dev, int n_items, unsigned char* canvas,
                  int batch, int channels, int s, void* stream);
typedef struct b2y_affine_item {
    double im[6];               /* output pixel -> canvas: invertAffineTransform(M[:2]), row-major 2 x 3 */
    unsigned char lut[768];     /* hue, saturation, value LUTs */
    int hsv;                    /* 1: the HSV stage */
    int flip;                   /* 1: left-right flip */
    int slot;                   /* canvas slot read, batch slot written */
    int reserved;
} b2y_affine_item;
int b2y_affine_hsv_u8(const b2y_affine_item* items, const b2y_affine_item* items_dev, int n_items,
                      const unsigned char* canvas, unsigned char* dst, int batch, int channels, int s, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200YOLO_H_ */
