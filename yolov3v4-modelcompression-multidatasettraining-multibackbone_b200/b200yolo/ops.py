"""Tensor-level wrappers over the C ABI: torch tensors in, torch tensors out, all math in libb200yolo.so.

Activations are NHWC fp16 tensors of shape [B, H, W, C]; a tensor may be a channel-slice *view* of a wider
buffer (stride(2) = pitch >= C), which is how route/concat layers are made zero-copy.
"""
import ctypes as C

import torch

from . import lib
from .lib import ACT, ConvDesc, QConvDesc, OUT_F16, OUT_F32, OUT_I8, DT_F16, DT_BF16, call, ptr, stream_ptr


def _gdt(t):
    """16-bit dtype code of a tensor (gradients may be bf16)."""
    return DT_BF16 if t.dtype == torch.bfloat16 else DT_F16


def _pitch(t):
    """Pixel pitch (elements) of an NHWC view; checks that only the channel dim is sliced."""
    assert t.dim() == 4 and (t.shape[3] == 1 or t.stride(3) == 1), "expected NHWC with unit channel stride"
    B, H, W, _ = t.shape
    p = t.stride(2) if W > 1 else (t.stride(1) if H > 1 else (t.stride(0) if B > 1 else t.shape[3]))
    if W == 1 and H > 1:
        p = t.stride(1)
    assert W == 1 or H == 1 or t.stride(1) == W * p, "not a pixel-contiguous NHWC view"
    assert B == 1 or t.stride(0) == H * W * p, "not a pixel-contiguous NHWC view"
    return p


def _require_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise lib.B2YError("b200yolo ops need CUDA tensors; there is no CPU fallback")


def conv_out_hw(h, w, k, stride, pad):
    return (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1


def make_conv_desc(x_shape, in_pitch, out_c, k, stride, pad, out_pitch, act="linear", slope=0.1,
                   out_dtype=OUT_F16, res_pitch=0, w_layout=0):
    B, H, W, Cin = x_shape
    Ho, Wo = conv_out_hw(H, W, k, stride, pad)
    return ConvDesc(B, H, W, Cin, in_pitch, out_c, k, stride, pad, Ho, Wo, out_pitch, ACT[act] if isinstance(act, str)
                    else int(act), float(slope), out_dtype, res_pitch, int(w_layout))


def pack_conv_weights(w, conv_bias=None, bn=None, eps=1e-5, want_fp32=False):
    """OIHW fp32 (+BN running stats) -> ([O][kh][kw][I] fp16, bias fp32[O], optional folded OIHW fp32)."""
    _require_cuda(w)
    O, I, k, _ = w.shape
    w = w.contiguous().float()
    wp = torch.empty((O, k, k, I), dtype=torch.float16, device=w.device)
    bias = torch.empty((O,), dtype=torch.float32, device=w.device)
    w32 = torch.empty_like(w) if want_fp32 else None
    g = b = m = v = None
    if bn is not None:
        g, b, m, v = [t.contiguous().float() for t in bn]
    cb = conv_bias.contiguous().float() if conv_bias is not None else None
    call("b2y_pack_conv_weights", ptr(w), ptr(cb), ptr(g), ptr(b), ptr(m), ptr(v), float(eps), O, I, k, ptr(wp),
         ptr(bias), ptr(w32), stream_ptr())
    return wp, bias, w32


def s2_pair_weights(w_oihw):
    """[O][I][3][3] -> [O][3][2][2I]: the B2Y_WLAYOUT_S2_PAIRS form of a 3x3 / stride-2 / pad-1 filter
    (include/b200yolo.h): window column 0 = the pixel pair left of the output, whose second pixel meets tap kw = 0;
    column 1 = the output's own pair = taps kw = 1, 2."""
    O, I = w_oihw.shape[:2]
    w = w_oihw.permute(0, 2, 3, 1)                       # [O][kh][kw][I]
    out = torch.zeros((O, 3, 2, 2 * I), dtype=w_oihw.dtype, device=w_oihw.device)
    out[:, :, 0, I:] = w[:, :, 0]
    out[:, :, 1, :I] = w[:, :, 1]
    out[:, :, 1, I:] = w[:, :, 2]
    return out.contiguous()


def s1_pair_weights(w_oihw):
    """[O][I][3][3] -> [2O][2I][3][3]: the 3x3 / stride-1 / pad-1 filter over tensors viewed as pixel pairs
    [B,H,W/2,2C].  Output sub-pixel o_sub and input sub-pixel i_sub of pair column kwp meet the original tap
    s = 2(kwp-1) + i_sub - o_sub + 1; the other entries are zero."""
    O, I = w_oihw.shape[:2]
    out = torch.zeros((2 * O, 2 * I, 3, 3), dtype=torch.float32, device=w_oihw.device)
    for o_sub in range(2):
        for i_sub in range(2):
            for kwp in range(3):
                s = 2 * (kwp - 1) + i_sub - o_sub + 1
                if 0 <= s <= 2:
                    out[o_sub * O:(o_sub + 1) * O, i_sub * I:(i_sub + 1) * I, :, kwp] = w_oihw[:, :, :, s]
    return out


def conv2d(x, w_packed, bias, k, stride, pad, act="linear", slope=0.1, residual=None, out=None,
           out_dtype=torch.float16, stats=None, w_layout=0):
    """y = act(conv(x, w) + bias) [+ residual]; x NHWC fp16 view, w_packed [O][k][k][I] fp16."""
    _require_cuda(x, w_packed)
    B, H, W, Cin = x.shape
    O = w_packed.shape[0]
    Ho, Wo = conv_out_hw(H, W, k, stride, pad)
    if out is None:
        out = torch.empty((B, Ho, Wo, O), dtype=out_dtype, device=x.device)
    assert out.shape == (B, Ho, Wo, O)
    od = OUT_F32 if out.dtype == torch.float32 else OUT_F16
    d = make_conv_desc(x.shape, _pitch(x), O, k, stride, pad, _pitch(out), act, slope, od,
                       _pitch(residual) if residual is not None else 0, w_layout)
    if stats is not None:
        assert residual is None
        call("b2y_conv2d_fwd_stats", C.byref(d), ptr(x), ptr(w_packed), ptr(bias), ptr(out), ptr(stats[0]),
             ptr(stats[1]), stream_ptr())
    else:
        call("b2y_conv2d_fwd", C.byref(d), ptr(x), ptr(w_packed), ptr(bias), ptr(residual), ptr(out), stream_ptr())
    return out


def stem_conv(x_nchw, w_oihw, bias, k, stride, pad, act="linear", slope=0.1, out=None):
    _require_cuda(x_nchw, w_oihw)
    B, Cin, H, W = x_nchw.shape
    O = w_oihw.shape[0]
    Ho, Wo = conv_out_hw(H, W, k, stride, pad)
    if out is None:
        out = torch.empty((B, Ho, Wo, O), dtype=torch.float16, device=x_nchw.device)
    d = make_conv_desc((B, H, W, Cin), Cin, O, k, stride, pad, _pitch(out), act, slope, OUT_F16)
    call("b2y_stem_conv_fwd", C.byref(d), ptr(x_nchw.contiguous()), ptr(w_oihw.contiguous()), ptr(bias), ptr(out),
         stream_ptr())
    return out


def pack_stem_weights(w_oihw_folded, out=None):
    """OIHW fp32 -> the [O][32] fp16 im2col rows of both tensor-core stems (layout.stem_path)."""
    O, I, k, _ = w_oihw_folded.shape
    if out is None:
        out = torch.empty((O, 32), dtype=torch.float16, device=w_oihw_folded.device)
    assert out.shape == (O, 32) and out.dtype == torch.float16 and out.is_contiguous()
    call("b2y_pack_stem_weights", ptr(w_oihw_folded.contiguous().float()), O, I, k, ptr(out), stream_ptr())
    return out


def stem_workspace_bytes(desc):
    from .lib import raw
    return int(raw().b2y_stem_workspace_bytes(C.byref(desc)))


def stem_workspace(desc, device):
    return torch.empty((stem_workspace_bytes(desc) // 2,), dtype=torch.float16, device=device)


def stem_conv_tc(x_nchw, w_stem, bias, in_c, k, stride, pad, act="linear", slope=0.1, out=None, workspace=None,
                 stats=None):
    """im2col workspace + GEMM stem: NCHW fp32 image -> NHWC fp16 (layout.stem_path). Returns (out, workspace)."""
    B, Cin, H, W = x_nchw.shape
    O = w_stem.shape[0]
    Ho, Wo = conv_out_hw(H, W, k, stride, pad)
    if out is None:
        out = torch.empty((B, Ho, Wo, O), dtype=torch.float16, device=x_nchw.device)
    d = make_conv_desc((B, H, W, Cin), Cin, O, k, stride, pad, _pitch(out), act, slope, OUT_F16)
    if workspace is None:
        workspace = stem_workspace(d, x_nchw.device)
    call("b2y_stem_conv_fwd_tc", C.byref(d), ptr(x_nchw), ptr(w_stem), ptr(bias), ptr(workspace), ptr(out),
         ptr(stats[0]) if stats is not None else None, ptr(stats[1]) if stats is not None else None, stream_ptr())
    return out, workspace


STEM_X = {torch.float32: 0, torch.float16: 1, torch.uint8: 2}


def stem_conv_fused(x_nchw, w_stem, bias, k, stride, pad, act="linear", slope=0.1, out=None, x_div=1.0):
    """Fused tensor-core stem (layout.stem_path): NCHW fp32/fp16/uint8 image -> NHWC fp16, no workspace."""
    _require_cuda(x_nchw)
    B, Cin, H, W = x_nchw.shape
    O = w_stem.shape[0]
    Ho, Wo = conv_out_hw(H, W, k, stride, pad)
    if out is None:
        out = torch.empty((B, Ho, Wo, O), dtype=torch.float16, device=x_nchw.device)
    x_nchw = x_nchw.contiguous()
    d = make_conv_desc((B, H, W, Cin), Cin, O, k, stride, pad, _pitch(out), act, slope, OUT_F16)
    call("b2y_stem_conv_fwd_fused", C.byref(d), ptr(x_nchw), STEM_X[x_nchw.dtype], float(x_div), ptr(w_stem), ptr(bias),
         ptr(out), stream_ptr())
    return out


def upsample(x, scale, out=None):
    B, H, W, Cc = x.shape
    if out is None:
        out = torch.empty((B, H * scale, W * scale, Cc), dtype=x.dtype, device=x.device)
    call("b2y_upsample_nearest", ptr(x), _pitch(x), ptr(out), _pitch(out), B, H, W, Cc, int(scale), stream_ptr())
    return out


def maxpool(x, k, stride, tiny_pad=False, out=None):
    B, H, W, Cc = x.shape
    if tiny_pad:
        Ho, Wo = (H + 1 - k) // stride + 1, (W + 1 - k) // stride + 1
    else:
        p = (k - 1) // 2
        Ho, Wo = (H + 2 * p - k) // stride + 1, (W + 2 * p - k) // stride + 1
    if out is None:
        out = torch.empty((B, Ho, Wo, Cc), dtype=x.dtype, device=x.device)
    call("b2y_maxpool", ptr(x), _pitch(x), ptr(out), _pitch(out), B, H, W, Cc, int(k), int(stride),
         1 if tiny_pad else 0, stream_ptr())
    return out


def copy_channels(x, out):
    B, H, W, Cc = x.shape
    call("b2y_copy_channels", ptr(x), _pitch(x), ptr(out), _pitch(out), B * H * W, Cc, stream_ptr())
    return out


def add(a, b, out=None):
    B, H, W, Cc = a.shape
    if out is None:
        out = torch.empty((B, H, W, Cc), dtype=a.dtype, device=a.device)
    assert a.dtype == b.dtype == out.dtype
    call("b2y_add", ptr(a), _pitch(a), ptr(b), _pitch(b), ptr(out), _pitch(out), B * H * W, Cc, _gdt(a), stream_ptr())
    return out


def act_fwd(x, act, slope=0.1):
    x = x.contiguous().float()
    y = torch.empty_like(x)
    call("b2y_act_fwd_f32", ptr(x), ptr(y), x.numel(), ACT[act], float(slope), stream_ptr())
    return y


def act_bwd(x, dy, act, slope=0.1):
    x = x.contiguous().float()
    dy = dy.contiguous().float()
    dx = torch.empty_like(x)
    call("b2y_act_bwd_f32", ptr(x), ptr(dy), ptr(dx), x.numel(), ACT[act], float(slope), stream_ptr())
    return dx


def nchw_to_nhwc(x, out=None):
    B, Cc, H, W = x.shape
    x = x.contiguous().float()
    if out is None:
        out = torch.empty((B, H, W, Cc), dtype=torch.float16, device=x.device)
    call("b2y_nchw_f32_to_nhwc_f16", ptr(x), ptr(out), _pitch(out), B, Cc, H, W, stream_ptr())
    return out


def nhwc_to_nchw(x):
    B, H, W, Cc = x.shape
    out = torch.empty((B, Cc, H, W), dtype=torch.float32, device=x.device)
    call("b2y_nhwc_f16_to_nchw_f32", ptr(x), _pitch(x), ptr(out), B, Cc, H, W, stream_ptr())
    return out


def yolo_decode(raw, na, no, anchors_px, stride, io=None, row_offset=0, want_p=True):
    """raw: fp32 [B, ny, nx, pitch>=na*no] head output. Returns (io_rows_view_or_None, p)."""
    B, ny, nx, _ = raw.shape
    p = torch.empty((B, na, ny, nx, no), dtype=torch.float32, device=raw.device) if want_p else None
    total_rows = io.shape[1] if io is not None else 0
    call("b2y_yolo_decode", ptr(raw), raw.stride(2), ptr(p), ptr(io), total_rows, row_offset, B, na, no, ny, nx,
         ptr(anchors_px), float(stride), stream_ptr())
    return io, p


def yolo_loss_layer(p, targets, anchor_vec, iou_t, gr, cls_pw, obj_pw, w_box, w_obj, w_cls, want_grad=True,
                    fl_gamma=0.0):
    """One yolo layer of compute_loss. Returns (out4 fp32[4] = [sum(1-giou), nb, sum bce cls, sum bce obj], dp).
    fl_gamma > 0: the class and objectness terms are focal-modulated BCE (alpha 0.25)."""
    B, na, ny, nx, no = p.shape
    p = p.contiguous()
    nt = int(targets.shape[0])
    out4 = torch.empty(4, dtype=torch.float32, device=p.device)
    dp = torch.empty_like(p) if want_grad else None
    ws_bytes = lib.raw().b2y_yolo_loss_workspace_bytes(B, na, ny, nx, nt)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=p.device)
    t = targets.contiguous().float() if nt else None
    call("b2y_yolo_loss", ptr(p), ptr(t), nt, ptr(anchor_vec), B, na, no, ny, nx, float(iou_t), float(gr),
         float(cls_pw), float(obj_pw), float(w_box), float(w_obj), float(w_cls), float(fl_gamma), ptr(out4), ptr(dp),
         ptr(ws),
         stream_ptr())
    return out4, dp


def build_targets_layer(targets, anchor_vec, batch, ny, nx, iou_t):
    """One yolo layer of build_targets -> (idx int64 [4, n] = (b, a, gj, gi), tbox fp32 [n, 4], tcls int64 [n]), in the
    reference's order (anchor-major, target-minor).  Candidates outside the batch or the ny x nx grid are dropped."""
    nt = int(targets.shape[0])
    na = int(anchor_vec.shape[0])
    cap = max(1, na * nt)
    dev = anchor_vec.device
    idx = torch.zeros((4, cap), dtype=torch.int64, device=dev)
    tbox = torch.zeros((cap, 4), dtype=torch.float32, device=dev)
    tcls = torch.zeros((cap,), dtype=torch.int64, device=dev)
    count = torch.zeros((1,), dtype=torch.int32, device=dev)
    t = targets.contiguous().float() if nt else None
    call("b2y_build_targets", ptr(t), nt, ptr(anchor_vec), int(batch), na, ny, nx, float(iou_t), ptr(idx), ptr(tbox),
         ptr(tcls), ptr(count), stream_ptr())
    n = int(count.item())
    return idx[:, :n], tbox[:n], tcls[:n]


# ---------------------------------------------------------------------------------------------------------------
# training kernels
# ---------------------------------------------------------------------------------------------------------------
def dgrad_weight_numel(out_c, in_c, k):
    return out_c * in_c * k * k


def pack_dgrad_weights(w_oihw, stride, pad, in_hw, dtype=torch.float16):
    """OIHW fp32 -> phase-decomposed dgrad weights (fp16) for b2y_conv2d_bwd_data."""
    O, I, k, _ = w_oihw.shape
    H, W = in_hw
    Ho, Wo = conv_out_hw(H, W, k, stride, pad)
    out = torch.empty(O * I * k * k, dtype=dtype, device=w_oihw.device)
    d = ConvDesc(1, H, W, I, I, O, k, stride, pad, Ho, Wo, O, 0, 0.0, OUT_F16, 0)
    call("b2y_pack_dgrad_weights", C.byref(d), ptr(w_oihw.contiguous().float()), ptr(out), _gdt(out), stream_ptr())
    return out


def conv2d_bwd_data(dy, w_packed_t, in_shape, k, stride, pad, out=None, accumulate=False, inv_scale=None):
    """dx (+)= conv^T(dy, W) [* inv_scale]: dy NHWC 16-bit [B,Ho,Wo,O] (same format as the packed weights) -> dx NHWC
    fp16 or bf16 [B,H,W,I]; inv_scale: optional device scalar multiplied into the result."""
    B, H, W, I = in_shape
    _, Ho, Wo, O = dy.shape
    if out is None:
        out = torch.empty((B, H, W, I), dtype=dy.dtype, device=dy.device)
        assert not accumulate
    assert dy.dtype == w_packed_t.dtype, "dY and the packed weights must share one 16-bit format"
    d = ConvDesc(B, H, W, I, _pitch(out), O, k, stride, pad, Ho, Wo, _pitch(dy), 0, 0.0, OUT_F16, 0)
    call("b2y_conv2d_bwd_data", C.byref(d), ptr(dy), ptr(w_packed_t), ptr(out), 1 if accumulate else 0, _gdt(dy),
         _gdt(out), ptr(inv_scale), stream_ptr())
    return out


def conv2d_bwd_weight(x, dy, k, stride, pad, scale=1.0, dw=None, inv_scale=None):
    """dW [O][k][k][I] fp32 (+)= scale [* inv_scale] * sum_pixels dy (x) x   (x and dy share one 16-bit format)."""
    B, H, W, I = x.shape
    _, Ho, Wo, O = dy.shape
    if dw is None:
        dw = torch.zeros((O, k, k, I), dtype=torch.float32, device=x.device)
    d = ConvDesc(B, H, W, I, _pitch(x), O, k, stride, pad, Ho, Wo, _pitch(dy), 0, 0.0, OUT_F16, 0)
    assert x.dtype == dy.dtype, "wgmma needs both operands in the same 16-bit format"
    call("b2y_conv2d_bwd_weight", C.byref(d), ptr(x), ptr(dy), ptr(dw), float(scale), _gdt(dy), ptr(inv_scale),
         stream_ptr())
    return dw


def unpack_wgrad(dw_packed, out_oihw, alpha=1.0, accumulate=False):
    O, k, _, I = dw_packed.shape
    call("b2y_unpack_wgrad", ptr(dw_packed), ptr(out_oihw), O, I, k, float(alpha), 1 if accumulate else 0,
         stream_ptr())
    return out_oihw


def axpby(src, dst, alpha=1.0, beta=0.0):
    call("b2y_axpby_f32", ptr(src), ptr(dst), src.numel(), float(alpha), float(beta), stream_ptr())
    return dst


def bn_train_fwd(z, s1, s2, gamma, beta, eps, momentum, running_mean, running_var, act, slope=0.1, residual=None,
                 out=None, save=None):
    """Fused finalize + apply of training-mode BatchNorm (csrc/bn_train.cu). Returns (y, save[4][C])."""
    B, H, W, Cc = z.shape
    if out is None:
        out = torch.empty((B, H, W, Cc), dtype=torch.float16, device=z.device)
    if save is None:
        save = torch.empty((4, Cc), dtype=torch.float32, device=z.device)
    n = B * H * W
    call("b2y_bn_train_fwd", ptr(z), _pitch(z), ptr(s1), ptr(s2), n, ptr(gamma), ptr(beta), float(eps),
         float(momentum), ptr(running_mean), ptr(running_var), ptr(save), ptr(residual),
         _pitch(residual) if residual is not None else 0, ptr(out), _pitch(out), n, Cc,
         ACT[act] if isinstance(act, str) else int(act), float(slope), stream_ptr())
    return out, save


def bn_train_bwd(z, dy, gamma, save, act, slope=0.1, grad_out_scale=1.0):
    """Backward of bn_train_fwd. Returns (dz fp16 = s * gradient, dgamma, dbeta, aux=[max|du|, s, 1/s, max|xhat|]).

    aux is the 4-float row the reduce and apply kernels share: the reduce writes max|du| and max|xhat| with atomicMax
    into the zeroed row, and the apply derives the power of two s from them so that max|dz * s| <= 2^12."""
    B, H, W, Cc = z.shape
    dev = z.device
    n = B * H * W
    a = ACT[act] if isinstance(act, str) else int(act)
    sums = torch.zeros((2, Cc), dtype=torch.float32, device=dev)
    aux = torch.zeros(4, dtype=torch.float32, device=dev)
    dz = torch.empty((B, H, W, Cc), dtype=torch.float16, device=dev)
    dgamma = torch.empty(Cc, dtype=torch.float32, device=dev)
    dbeta = torch.empty(Cc, dtype=torch.float32, device=dev)
    call("b2y_bn_train_bwd_reduce", ptr(z), _pitch(z), ptr(dy), _pitch(dy), ptr(save), ptr(sums), ptr(aux), n, Cc, a,
         float(slope), _gdt(dy), stream_ptr())
    call("b2y_bn_train_bwd_apply", ptr(z), _pitch(z), ptr(dy), _pitch(dy), ptr(gamma), ptr(save), ptr(sums), ptr(dz),
         _pitch(dz), n, Cc, a, float(slope), _gdt(dy), ptr(aux), C.c_void_p(aux.data_ptr() + 4), ptr(dgamma),
         ptr(dbeta), float(grad_out_scale), stream_ptr())
    return dz, dgamma, dbeta, aux


def bias_act_bwd_reduce(x, dy, scale, shift, act, slope=0.1, dbeta=None):
    """dbias = sum dy*act'(x*scale+shift) for a conv without BN (dgamma not needed)."""
    B, H, W, Cc = x.shape
    if dbeta is None:
        dbeta = torch.zeros(Cc, dtype=torch.float32, device=x.device)
    call("b2y_bn_act_bwd_reduce", ptr(x), _pitch(x), ptr(dy), _pitch(dy), ptr(scale), ptr(shift), None, None, None,
         ptr(dbeta), None, B * H * W, Cc, ACT[act] if isinstance(act, str) else int(act), float(slope), _gdt(dy),
         stream_ptr())
    return dbeta


# ---------------------------------------------------------------------------------------------------------------
# depthwise convolution + squeeze-excite (MobileNet backbones)
# ---------------------------------------------------------------------------------------------------------------
def dwconv2d(x, w, k, stride, pad, scale=None, bias=None, act="linear", slope=0.1, out=None, stats=None):
    """Depthwise conv: x NHWC fp16 [B,H,W,C], w fp32 [C,1,k,k] (the module parameter).  y = act(conv*scale + bias)."""
    _require_cuda(x, w)
    B, H, W, Cc = x.shape
    Ho, Wo = conv_out_hw(H, W, k, stride, pad)
    if out is None:
        out = torch.empty((B, Ho, Wo, Cc), dtype=torch.float16, device=x.device)
    d = make_conv_desc(x.shape, _pitch(x), Cc, k, stride, pad, _pitch(out), act, slope, OUT_F16)
    assert w.is_contiguous() and w.dtype == torch.float32 and w.numel() == Cc * k * k
    call("b2y_dwconv_fwd", C.byref(d), ptr(x), ptr(w), ptr(scale), ptr(bias), ptr(out),
         ptr(stats[0]) if stats is not None else None, ptr(stats[1]) if stats is not None else None, stream_ptr())
    return out


def dwconv2d_bwd_data(dz, w, in_shape, k, stride, pad, out=None, accumulate=False, inv_scale=None):
    B, H, W, Cc = in_shape
    _, Ho, Wo, _ = dz.shape
    if out is None:
        out = torch.zeros((B, H, W, Cc), dtype=torch.float16, device=dz.device)
    d = ConvDesc(B, H, W, Cc, _pitch(out), Cc, k, stride, pad, Ho, Wo, _pitch(dz), 0, 0.0, OUT_F16, 0)
    call("b2y_dwconv_bwd_data", C.byref(d), ptr(dz), ptr(w), ptr(out), 1 if accumulate else 0, _gdt(out),
         ptr(inv_scale), stream_ptr())
    return out


def dwconv2d_bwd_weight(x, dz, k, stride, pad, alpha=1.0, dw=None, inv_scale=None):
    B, H, W, Cc = x.shape
    _, Ho, Wo, _ = dz.shape
    if dw is None:
        dw = torch.zeros((Cc, 1, k, k), dtype=torch.float32, device=x.device)
    d = ConvDesc(B, H, W, Cc, _pitch(x), Cc, k, stride, pad, Ho, Wo, _pitch(dz), 0, 0.0, OUT_F16, 0)
    call("b2y_dwconv_bwd_weight", C.byref(d), ptr(x), ptr(dz), ptr(dw), float(alpha), ptr(inv_scale), stream_ptr())
    return dw


def se_workspace(batch, c, cr, device):
    return torch.empty((batch, 3 * c + cr), dtype=torch.float32, device=device)


def se_fwd(x, w1, w2, out=None, ws=None):
    """Squeeze-excite: x NHWC fp16, w1 [C/r, C], w2 [C, C/r] fp32 (nn.Linear weights). Returns (y, ws)."""
    B, H, W, Cc = x.shape
    cr = w1.shape[0]
    if out is None:
        out = torch.empty((B, H, W, Cc), dtype=torch.float16, device=x.device)
    if ws is None:
        ws = se_workspace(B, Cc, cr, x.device)
    assert w1.is_contiguous() and w2.is_contiguous() and w1.dtype == torch.float32
    call("b2y_se_fwd", ptr(x), _pitch(x), ptr(w1), ptr(w2), ptr(out), _pitch(out), B, H * W, Cc, cr, ptr(ws),
         stream_ptr())
    return out, ws


def se_bwd(x, dy, w1, w2, ws, dx, accumulate=False, dw1=None, dw2=None, grad_scale=1.0, ws_bwd=None):
    B, H, W, Cc = x.shape
    cr = w1.shape[0]
    if ws_bwd is None:
        ws_bwd = se_workspace(B, Cc, cr, x.device)
    if dw1 is None:
        dw1 = torch.empty_like(w1)
        dw2 = torch.empty_like(w2)
    call("b2y_se_bwd", ptr(x), _pitch(x), ptr(dy), _pitch(dy), ptr(w1), ptr(w2), ptr(ws), ptr(ws_bwd), ptr(dx),
         _pitch(dx), 1 if accumulate else 0, ptr(dw1), ptr(dw2), float(grad_scale), B, H * W, Cc, cr, _gdt(dy),
         stream_ptr())
    return dx, dw1, dw2


def _opt_check(tiles, *flat):
    _require_cuda(tiles, *flat)
    assert tiles.dtype == torch.int64 and tiles.dim() == 2 and tiles.shape[1] == 2 and tiles.is_contiguous()
    n = flat[0].numel()
    for t in flat:
        if t is not None:
            assert t.dtype == torch.float32 and t.is_contiguous() and t.numel() == n


def sgd_grouped(param, grad, buf, tiles, hp, ema=None):
    """Nesterov SGD per parameter group over flat buffers in one launch (csrc/train.cu opt_grouped_kernel).  `tiles` is
    the int64 [n][2] device table of B2YOptTile rows, `hp` a lib.OptStep passed by value."""
    _opt_check(tiles, param, grad, buf, ema)
    call("b2y_sgd_grouped", ptr(param), ptr(grad), ptr(buf), ptr(ema), ptr(tiles), int(tiles.shape[0]), C.byref(hp),
         stream_ptr())


def adam_grouped(param, grad, exp_avg, exp_avg_sq, tiles, hp, ema=None):
    """Adam per parameter group over flat buffers in one launch (torch.optim.Adam semantics, amsgrad=False)."""
    _opt_check(tiles, param, grad, exp_avg, exp_avg_sq, ema)
    call("b2y_adam_grouped", ptr(param), ptr(grad), ptr(exp_avg), ptr(exp_avg_sq), ptr(ema), ptr(tiles),
         int(tiles.shape[0]), C.byref(hp), stream_ptr())


# ---------------------------------------------------------------------------------------------------------------
# quantisation kernels
# ---------------------------------------------------------------------------------------------------------------
def fakequant(x, scale, bits=8):
    x = x.contiguous().float()
    y = torch.empty_like(x)
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    call("b2y_fakequant_f32", ptr(x), ptr(y), x.numel(), float(scale), float(lo), float(hi), stream_ptr())
    return y


def fakequant_range(x, scale, lo, hi):
    """clamp(round_half_away(x / scale), lo, hi) * scale with an explicit code range (+-3e38 = "round, do not clamp":
    the quantised shortcuts round their addends without clamping, ptq_cos.py:876-884)."""
    x = x.contiguous().float()
    y = torch.empty_like(x)
    call("b2y_fakequant_f32", ptr(x), ptr(y), x.numel(), float(scale), float(lo), float(hi), stream_ptr())
    return y


def quantize_to_i8(x, scale, bits=8, out=None):
    B, H, W, Cc = x.shape
    if out is None:
        out = torch.empty((B, H, W, Cc), dtype=torch.int8, device=x.device)
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    call("b2y_quantize_f16_to_i8", ptr(x), _pitch(x), ptr(out), _pitch(out), B * H * W, Cc, float(scale), float(lo),
         float(hi), stream_ptr())
    return out


def cos_scale_search(x, bits=8, n_cand=None, step0=-5):
    """Cosine similarities of x vs fakequant(x; 2^(i+step0)/2^(bits-1)), i in range(n_cand) -> fp32 [n_cand] (device).
    Defaults = the conv quantisers' search (bits+7 candidates from 2^-5)."""
    x = x.contiguous().float()
    if n_cand is None:
        n_cand = bits + 7
    out = torch.empty(n_cand, dtype=torch.float32, device=x.device)
    ws = torch.empty(8 * (1 + 2 * n_cand), dtype=torch.uint8, device=x.device)
    call("b2y_cos_scale_search_ex", ptr(x), x.numel(), bits, n_cand, int(step0), ptr(out), ptr(ws), ws.numel(),
         stream_ptr())
    return out


def minmax(x2d, per_row=False):
    x2d = x2d.contiguous().float()
    rows, cols = x2d.shape
    out = torch.empty((rows if per_row else 1, 2), dtype=torch.float32, device=x2d.device)
    call("b2y_minmax_f32", ptr(x2d), rows, cols, 1 if per_row else 0, ptr(out), stream_ptr())
    return out


def pack_qconv_weights(w_folded_oihw, w_scale, bits=8):
    O, I, k, _ = w_folded_oihw.shape
    out = torch.empty((O, k, k, I), dtype=torch.int8, device=w_folded_oihw.device)
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    call("b2y_pack_qconv_weights", ptr(w_folded_oihw.contiguous().float()), O, I, k, float(w_scale), float(lo),
         float(hi), ptr(out), stream_ptr())
    return out


def qconv2d(x_i8, w_i8, bias, k, stride, pad, acc_scale, out_scale, act="linear", slope=0.1, bits=8, out=None,
            out_kind=OUT_I8, requant=True, w_layout=0):
    """INT8 conv: y = requant(act(acc*acc_scale + bias)); x int8 NHWC, w int8 [O][k][k][I]."""
    B, H, W, Cin = x_i8.shape
    O = w_i8.shape[0]
    Ho, Wo = conv_out_hw(H, W, k, stride, pad)
    if out is None:
        dt = {OUT_I8: torch.int8, OUT_F16: torch.float16, OUT_F32: torch.float32}[out_kind]
        out = torch.empty((B, Ho, Wo, O), dtype=dt, device=x_i8.device)
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    cd = make_conv_desc(x_i8.shape, _pitch(x_i8), O, k, stride, pad, _pitch(out), act, slope, out_kind, 0, w_layout)
    qd = QConvDesc(cd, float(acc_scale), float(out_scale), float(lo), float(hi), out_kind, 1 if requant else 0)
    call("b2y_qconv2d_fwd", C.byref(qd), ptr(x_i8), ptr(w_i8), ptr(bias), ptr(out), stream_ptr())
    return out
