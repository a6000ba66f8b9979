"""Quantisation-aware-training execution (quantized=1 google, quantized=2 TPSQ) on sm_90a.

Reference: utils/quantized/quantized_google.py:235-836 / quantized_TPSQ.py:349-589.  A QAT layer is two convolutions per
training step (a plain one for the BatchNorm batch statistics, one on the fake-quantised folded weights), fake-quant with
straight-through gradients on weights / bias / activations, and a BN fold whose gradient flows through the batch
statistics.  That chain is data dependent per step (range trackers, freeze steps), so it is not captured in a static plan:
the module forwards of utils/quantized/*.py are executed one by one over NHWC fp32 tensors, composed from the autograd
Functions below -- each of which runs the hand-written kernels (wgmma forward / data-gradient / weight-gradient convs,
fake-quant forward / STE backward, activation forward / backward) -- while torch.autograd only chains them and handles the
per-channel [C]-sized fold arithmetic.

Exactness: fake-quantised activations and weights are int8 codes times a power of two, exact in fp16, and their products
/ fp32 partial sums are exact, so the quantised conv equals the reference's fp32 F.conv2d on the same values.
"""
import ctypes

import torch

from . import ops
from .lib import ConvDesc, call, ptr, stream_ptr


def _pow2_scale(g):
    """device-side power-of-two factor that brings max|g| to ~2^12 (fp16 operand of the gradient GEMMs)"""
    amax = g.abs().max().clamp(min=1e-30)
    s = ((4096.0 / amax).float().view(torch.int32) & 0x7F800000).view(torch.float32).clamp(1e-30, 1e30)
    return torch.stack([s, 1.0 / s]).contiguous()


class ConvFn(torch.autograd.Function):
    """y[, sum_c y, sum_c y^2] = conv2d(x NHWC fp32, w OIHW fp32) on the wgmma fp16 kernel with fp32 accumulation / output.
    backward: weight gradient + data gradient on the wgmma backward kernels (dz as fp16 x 2^k, k chosen on the device).
    The optional channel sums come out of the conv epilogue and are differentiable (their gradients are folded into dz)."""

    @staticmethod
    def forward(ctx, x, w, k, s, p, want_stats):
        ctx.set_materialize_grads(False)
        B, H, W, C = x.shape
        O, I = w.shape[0], w.shape[1]
        x16 = x.half()
        Ik = (I + 15) // 16 * 16
        if C != Ik:                                  # first layer: image channels padded to the MMA K granule
            xp = torch.zeros((B, H, W, Ik), dtype=torch.float16, device=x.device)
            xp[..., :C] = x16
            x16 = xp
        wk = w.detach().float()
        if Ik != I:
            wk = torch.nn.functional.pad(wk, (0, 0, 0, 0, 0, Ik - I))
        stats = None
        if want_stats:
            # The statistics pass multiplies the (exactly fp16-representable) activations with the FLOAT weights
            # (google.py:326-338).  fp16-rounded weights would move the batch statistics by ~1e-3, enough to flip
            # quantised weight codes after the fold, so the weights go in as a two-term split in ONE tensor-core conv
            # over a doubled K:  [x | x * 2^-12] * [hi | lo * 2^12]  =  x * (hi + lo), every product exact, fp32 sums.
            hi = wk.half().float()
            lo = ((wk - hi) * 4096.0).half().float()
            xa = torch.cat([x16, (x16.float() * (1.0 / 4096.0)).half()], 3).contiguous()
            wp, _, _ = ops.pack_conv_weights(torch.cat([hi, lo], 1).contiguous())
            stats = torch.zeros((2, O), dtype=torch.float32, device=x.device)
            y = ops.conv2d(xa, wp, None, k, s, p, out_dtype=torch.float32, stats=(stats[0], stats[1]))
        else:
            wp, _, _ = ops.pack_conv_weights(wk.contiguous())
            y = ops.conv2d(x16, wp, None, k, s, p, out_dtype=torch.float32)
        ctx.geom = (k, s, p, C, I, Ik, O, (B, H, W))
        ctx.want_stats = want_stats
        ctx.save_for_backward(x16, wk, y if want_stats else None)
        ctx.x_needs = x.requires_grad
        if want_stats:
            return y, stats[0], stats[1]
        return y, None, None

    @staticmethod
    def backward(ctx, gy, gs1, gs2):
        k, s, p, C, I, Ik, O, (B, H, W) = ctx.geom
        x16, wk, y = ctx.saved_tensors
        g = gy
        if ctx.want_stats and (gs1 is not None or gs2 is not None):
            extra = 0
            if gs1 is not None:
                extra = gs1.view(1, 1, 1, -1)
            if gs2 is not None:
                extra = extra + 2.0 * gs2.view(1, 1, 1, -1) * y
            g = extra.expand_as(y) if g is None else g + extra
        if g is None:
            return None, None, None, None, None, None
        g = g.contiguous().float()
        sc = _pow2_scale(g)
        dz = (g * sc[0]).half()
        Ok = (O + 15) // 16 * 16
        if Ok != O:
            dzp = torch.zeros(dz.shape[:3] + (Ok,), dtype=torch.float16, device=dz.device)
            dzp[..., :O] = dz
            dz = dzp
        # weight gradient: packed fp32 [Ok][k][k][Ik] -> OIHW
        dwp = torch.zeros((Ok, k, k, Ik), dtype=torch.float32, device=dz.device)
        ops.conv2d_bwd_weight(x16, dz, k, s, p, scale=1.0, dw=dwp, inv_scale=sc[1:2])
        dw = dwp[:O, :, :, :I].permute(0, 3, 1, 2).contiguous()
        dx = None
        if ctx.x_needs:
            wpad = wk[:, :I]
            if Ok != O:
                wpad = torch.nn.functional.pad(wpad, (0, 0, 0, 0, 0, 0, 0, Ok - O))
            wT = ops.pack_dgrad_weights(wpad.contiguous(), s, p, (H, W), dtype=torch.float16)
            out = torch.zeros((B, H, W, I), dtype=torch.bfloat16, device=dz.device)
            ops.conv2d_bwd_data(dz, wT, (B, H, W, I), k, s, p, out=out, accumulate=False, inv_scale=sc[1:2])
            dx = out.float()
        return dx, dw, None, None, None, None


def conv2d(x, w, k, s, p, want_stats=False):
    y, s1, s2 = ConvFn.apply(x, w, k, s, p, want_stats)
    return (y, s1, s2) if want_stats else y


class FakeQuantFn(torch.autograd.Function):
    """y = clamp(round_half_away(x / s), lo, hi) * s ; dx = g * [lo <= round(x/s) <= hi]   (google.py:81-143)"""

    @staticmethod
    def forward(ctx, x, scale, lo, hi):
        ctx.save_for_backward(x)
        ctx.q = (float(scale), float(lo), float(hi))
        return ops.fakequant_range(x, scale, lo, hi).view_as(x)

    @staticmethod
    def backward(ctx, g):
        x, = ctx.saved_tensors
        scale, lo, hi = ctx.q
        xc, gc = x.contiguous().float(), g.contiguous().float()
        dx = torch.empty_like(xc)
        call("b2y_fakequant_bwd_f32", ptr(xc), ptr(gc), ptr(dx), xc.numel(), scale, lo, hi, 1.0, stream_ptr())
        return dx.view_as(x), None, None, None


def fake_quant(x, scale, bits, sign=True, clamp=True):
    if sign:
        lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    else:
        lo, hi = 0, (1 << bits) - 1
    if not clamp:
        lo, hi = -3.0e38, 3.0e38
    return FakeQuantFn.apply(x, float(scale), float(lo), float(hi))


class ActFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, act, slope):
        ctx.save_for_backward(x)
        ctx.a = (act, slope)
        return ops.act_fwd(x, act, slope).view_as(x)

    @staticmethod
    def backward(ctx, g):
        x, = ctx.saved_tensors
        act, slope = ctx.a
        return ops.act_bwd(x, g, act, slope).view_as(x), None, None


def activation(x, name, maxabsscaler=False):
    # 'none' (GhostNet's cfg): the reference layers print a warning and leave the output unchanged
    if name in ('linear', 'none'):
        return x
    return ActFn.apply(x, name, 0.25 if maxabsscaler else 0.1)


class TpsqFn(torch.autograd.Function):
    """TPSQ quantiser with the power-of-two range P = Search_Pow2(scale parameter) (quantized_TPSQ.py:29-130).
    Returns y; gradients: dx (soft-clamp mask x (2^(b-1)-1)/2^(b-1)) and d/dscale = (P / scale) * sum(g * dy/dP)
    (Search_Pow2.backward multiplies by output / input)."""

    @staticmethod
    def forward(ctx, x, scale_param, P, bits):
        xc = x.contiguous().float()
        y = torch.empty_like(xc)
        call("b2y_tpsq_fwd_f32", ptr(xc), ptr(y), xc.numel(), float(P), int(bits), stream_ptr())
        ctx.save_for_backward(xc)
        # the parameter value BEFORE Search_Pow2 snaps it in place (quantized_TPSQ.py:33, 41-45)
        ctx.q = (float(P), int(bits), x.requires_grad, float(scale_param.reshape(-1)[0]), tuple(scale_param.shape))
        return y.view_as(x)

    @staticmethod
    def backward(ctx, g):
        xc, = ctx.saved_tensors
        P, bits, need_x, scale_before, sshape = ctx.q
        gc = g.contiguous().float()
        dx = torch.empty_like(xc) if need_x else None
        acc = torch.zeros(1, dtype=torch.float64, device=xc.device)
        call("b2y_tpsq_bwd_f32", ptr(xc), ptr(gc), ptr(dx), ptr(acc), xc.numel(), P, bits, stream_ptr())
        dscale = (acc.float() * (P / scale_before)).reshape(sshape)
        return (dx.view_as(g) if need_x else None), dscale, None, None


def search_pow2(scale_value):
    """Search_Pow2.forward (quantized_TPSQ.py:31-46): clip to [2^-5 (if negative), 2^13], nearest power of two."""
    import math
    v = float(scale_value)
    if v < 0:
        v = 2.0 ** -5
    if v > 2.0 ** 13:
        v = 2.0 ** 13
    ce, fl = 2.0 ** math.ceil(math.log2(v)), 2.0 ** math.floor(math.log2(v))
    return ce if abs(ce - v) < abs(fl - v) else fl


def _dw_desc(x, C, k, s, p):
    B, H, W, _ = x.shape
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    return ConvDesc(B, H, W, C, C, C, k, s, p, Ho, Wo, C, 0, 0.0, 0, 0, 0), (B, Ho, Wo, C)


class DepthwiseBlockFn(torch.autograd.Function):
    """The float [depthwise] block of a google-QAT graph (reference models.py:175-197 under quantized=1): z =
    Conv2d(groups=C)(x), y = act(BatchNorm2d(z)), batch statistics in training (running statistics updated in place),
    running statistics in eval.  fp32 NHWC in both directions on the kernels of depthwise.cu / bn_train.cu."""

    @staticmethod
    def forward(ctx, x, w, gamma, beta, rmean, rvar, k, s, p, act, slope, training, momentum, eps):
        C = x.shape[3]
        x = x.contiguous()
        wk = w.detach().contiguous()
        d, shape = _dw_desc(x, C, k, s, p)
        z = torch.empty(shape, dtype=torch.float32, device=x.device)
        call("b2y_dwconv_fwd_f32", ctypes.byref(d), ptr(x), ptr(wk), None, ptr(z), stream_ptr())
        y = torch.empty_like(z)
        save = torch.empty((4, C), dtype=torch.float32, device=x.device)
        call("b2y_bn_f32_fwd", ptr(z), z.numel() // C, C, ptr(gamma.detach()), ptr(beta.detach()), float(eps),
             float(momentum), ptr(rmean), ptr(rvar), int(training), ptr(save), ptr(y), ops.ACT[act], float(slope),
             stream_ptr())
        ctx.save_for_backward(x, wk, gamma.detach(), z, save)
        ctx.geom = (d, int(training), ops.ACT[act], float(slope))
        return y

    @staticmethod
    def backward(ctx, gy):
        x, wk, gamma, z, save = ctx.saved_tensors
        d, training, act, slope = ctx.geom
        C = z.shape[3]
        gy = gy.contiguous().float()
        dz = torch.empty_like(z)
        coef = torch.empty((3, C), dtype=torch.float32, device=z.device)
        dgamma = torch.empty(C, dtype=torch.float32, device=z.device)
        dbeta = torch.empty_like(dgamma)
        call("b2y_bn_f32_bwd", ptr(z), ptr(gy), z.numel() // C, C, ptr(gamma), ptr(save), training, ptr(coef), ptr(dz),
             ptr(dgamma), ptr(dbeta), act, slope, stream_ptr())
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dw = torch.empty_like(wk)
        call("b2y_dwconv_bwd_f32", ctypes.byref(d), ptr(x), ptr(dz), ptr(wk), ptr(dx), ptr(dw), stream_ptr())
        return dx, dw, dgamma, dbeta, None, None, None, None, None, None, None, None, None, None


class DwGradLink:
    """Couples the two depthwise convolutions of a TPSQ layer on one input (quantized_TPSQ.py:404-420, 530-538): the
    statistics conv with the float weights and the quantised conv with W_q, whose weights are folded from those
    statistics.  W_q's gradient feeds the variance's gradient through the fold, so the quantised conv's backward runs
    first and must return dW_q; it leaves its output gradient here instead of computing its data gradient, and the
    statistics conv's backward adds both data gradients in one gather."""

    def __init__(self):
        self.gy, self.w = None, None


class DwConvFn(torch.autograd.Function):
    """y = dwconv(x, w) over NHWC fp32 (groups = C).  backward: dw, and dx unless a DwGradLink hands gy to the statistics
    conv on the same input (DwConvStatsFn)."""

    @staticmethod
    def forward(ctx, x, w, k, s, p, link):
        C = x.shape[3]
        x = x.contiguous()
        wk = w.detach().contiguous()
        d, shape = _dw_desc(x, C, k, s, p)
        y = torch.empty(shape, dtype=torch.float32, device=x.device)
        call("b2y_dwconv_fwd_f32", ctypes.byref(d), ptr(x), ptr(wk), None, ptr(y), stream_ptr())
        ctx.save_for_backward(x, wk)
        ctx.geom = (d, link)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, wk = ctx.saved_tensors
        d, link = ctx.geom
        gy = gy.contiguous().float()
        # the statistics conv's backward only runs if W_q's gradient can reach the statistics through the fold
        deferred = link is not None and ctx.needs_input_grad[1]
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] and not deferred else None
        dw = torch.empty_like(wk) if ctx.needs_input_grad[1] else None
        if dx is not None or dw is not None:
            call("b2y_dwconv_bwd_f32", ctypes.byref(d), ptr(x), ptr(gy), ptr(wk), ptr(dx), ptr(dw), stream_ptr())
        if deferred:
            link.gy, link.w = gy, wk
        return dx, dw, None, None, None, None


class DwConvStatsFn(torch.autograd.Function):
    """Per-channel batch mean and unbiased variance (torch.var) of z = dwconv(x, w) + b, the statistics conv of a TPSQ
    depthwise layer; z is recomputed in the forward and the backward, never stored.  Both outputs are differentiable:
    gz = g_mean / n + 2 g_var (z - mean) / (n - 1), and dx adds the linked quantised conv's data gradient."""

    @staticmethod
    def forward(ctx, x, w, b, k, s, p, link):
        C = x.shape[3]
        x = x.contiguous()
        wk = w.detach().contiguous()
        bk = b.detach().contiguous() if b is not None else None
        d, shape = _dw_desc(x, C, k, s, p)
        mean = torch.empty(C, dtype=torch.float32, device=x.device)
        var = torch.empty_like(mean)
        call("b2y_dwconv_stats_f32", ctypes.byref(d), ptr(x), ptr(wk), ptr(bk), ptr(mean), ptr(var), stream_ptr())
        ctx.save_for_backward(x, wk, bk, mean)
        ctx.geom = (d, shape, link)
        return mean, var

    @staticmethod
    def backward(ctx, g_mean, g_var):
        x, wk, bk, mean = ctx.saved_tensors
        d, shape, link = ctx.geom
        gy, wq = (link.gy, link.w) if link is not None else (None, None)
        if link is not None:
            link.gy = link.w = None
        gm = g_mean.contiguous().float() if g_mean is not None else None
        gv = g_var.contiguous().float() if g_var is not None else None
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dw = torch.empty_like(wk) if ctx.needs_input_grad[1] else None
        if dx is not None or dw is not None:
            gs = torch.empty(shape, dtype=torch.float32, device=x.device)
            call("b2y_dwconv_stats_bwd_f32", ctypes.byref(d), ptr(x), ptr(wk), ptr(bk), ptr(mean), ptr(gm), ptr(gv),
                 ptr(gy), ptr(wq), ptr(gs), ptr(dx), ptr(dw), stream_ptr())
        # sum_pixels gz = g_mean: the bias moves the mean and leaves the variance
        db = (gm if gm is not None else torch.zeros_like(mean)) if ctx.needs_input_grad[2] else None
        return dx, dw, db, None, None, None, None


def dwconv2d(x, w, k, s, p, link=None):
    """y = Conv2d(groups=C)(x, w) over NHWC fp32 on the kernels of depthwise.cu"""
    return DwConvFn.apply(x, w, k, s, p, link)


def dwconv_stats(x, w, b, k, s, p, link=None):
    """(mean, var) of dwconv(x, w) + b over batch and pixels, differentiable; `link` couples the backward with the
    quantised conv dwconv2d(x, W_q, ..., link) on the same input"""
    return DwConvStatsFn.apply(x, w, b, k, s, p, link)


def check_groups(layer):
    """dense (groups = 1) and depthwise (groups = in = out channels) QAT layers run; other groupings are refused"""
    if layer.groups != 1 and not layer.groups == layer.in_channels == layer.out_channels:
        raise NotImplementedError("grouped convolution (1 < groups < channels) in a %s layer"
                                  % layer.__class__.__name__)
    return layer.groups != 1


def fold_batch_norm(layer, x, k, s, p, freeze_step):
    """Training-mode BatchNorm fold of a google / TPSQ QAT conv layer with bn=1 (quantized_google.py:320-374,
    quantized_TPSQ.py:404-440): the batch statistics of the float-weight conv (the mean shifted by the conv bias, the
    unbiased variance), the running-statistics update seeded on the first call, and before `freeze_step` the fold on the
    batch statistics, with their gradient, after it the fold on the running statistics.  Returns the folded weight and
    bias and the DwGradLink the quantised depthwise conv on `x` must take (None for dense layers)."""
    cb = layer.bias if layer.bias is not None else 0
    link = None
    if layer.groups == 1:
        y1, s1, s2 = conv2d(x, layer.weight, k, s, p, want_stats=True)   # channel sums from the conv epilogue
        n = float(y1.shape[0] * y1.shape[1] * y1.shape[2])
        mean = s1 / n + cb
        var = (s2 - s1 * (s1 / n)) / (n - 1.0)                           # torch.var: unbiased
    elif float(layer.step) < freeze_step:
        # the fold takes the batch statistics: both convolutions of the layer share one backward
        link = DwGradLink()
        mean, var = dwconv_stats(x, layer.weight, layer.bias, k, s, p, link)
    else:
        with torch.no_grad():                                            # only the running statistics read them
            mean, var = dwconv_stats(x, layer.weight, layer.bias, k, s, p)
    layer.batch_mean, layer.batch_var = mean, var
    with torch.no_grad():
        if float(layer.first_bn) == 0 and not bool(layer.running_mean.any()) and not bool(layer.running_var.any()):
            layer.first_bn.add_(1)
            layer.running_mean.add_(mean)
            layer.running_var.add_(var)
        else:
            layer.running_mean.mul_(1 - layer.momentum).add_(mean * layer.momentum)
            layer.running_var.mul_(1 - layer.momentum).add_(var * layer.momentum)
    if float(layer.step) < freeze_step:
        sc = layer.gamma / torch.sqrt(var + layer.eps)
        bias = layer.beta + (cb - mean) * sc
    else:
        sc = layer.gamma / torch.sqrt(layer.running_var + layer.eps)
        bias = layer.beta + (cb - layer.running_mean) * sc
    return layer.weight * sc.reshape(-1, 1, 1, 1), bias.reshape(-1), link


def qconv(layer, x, w, k, s, p, link=None):
    """the layer's convolution on its quantised weights: the wgmma conv, or for groups = C the fp32 depthwise conv"""
    if layer.groups == 1:
        return conv2d(x, w, k, s, p)
    return dwconv2d(x, w, k, s, p, link)


def depthwise_block(block, d, x, training):
    """module tree Sequential(DepthWise2d, BatchNorm2d[, activation]) of models._conv_block -> NHWC fp32 output"""
    conv = block[0]
    if len(block) < 2 or block[1].__class__.__name__ != 'BatchNorm2d':
        raise NotImplementedError("depthwise block without BatchNorm in the QAT graph")
    bn = block[1]
    k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
    if training and bn.momentum is None:
        raise NotImplementedError("cumulative-average BatchNorm in the QAT graph")
    slope = block[2].negative_slope if d['activation'] == 'leaky' else 0.1
    y = DepthwiseBlockFn.apply(x, conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, k, s, p,
                               d['activation'] if len(block) > 2 else 'linear', slope, training, bn.momentum, bn.eps)
    if training:
        bn.num_batches_tracked.add_(1)
    return y


class SEFn(torch.autograd.Function):
    """SE (utils/layers.py:154-166) over NHWC fp32: y = x * hsigmoid(W2 relu(W1 mean_hw(x)))"""

    @staticmethod
    def forward(ctx, x, w1, w2):
        B, H, W, C = x.shape
        Cr = w1.shape[0]
        x = x.contiguous()
        w1d, w2d = w1.detach().contiguous(), w2.detach().contiguous()
        y = torch.empty_like(x)
        ws = torch.empty(B * (3 * C + Cr), dtype=torch.float32, device=x.device)
        call("b2y_se_fwd_f32", ptr(x), ptr(w1d), ptr(w2d), ptr(y), B, H * W, C, Cr, ptr(ws), stream_ptr())
        ctx.save_for_backward(x, w1d, w2d, ws)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, w1, w2, ws = ctx.saved_tensors
        B, H, W, C = x.shape
        Cr = w1.shape[0]
        gy = gy.contiguous().float()
        dx = torch.empty_like(x)
        dw1, dw2 = torch.empty_like(w1), torch.empty_like(w2)
        wsb = torch.empty(B * (3 * C + Cr), dtype=torch.float32, device=x.device)
        call("b2y_se_bwd_f32", ptr(x), ptr(gy), ptr(w1), ptr(w2), ptr(ws), ptr(wsb), ptr(dx), ptr(dw1), ptr(dw2), B,
             H * W, C, Cr, stream_ptr())
        return dx, dw1, dw2


def se_layer(se, x):
    return SEFn.apply(x, se.fc[0].weight, se.fc[2].weight)


# ----------------------------------------------------------------------------------------------------------------------
class QatRunner:
    """Executes the module list of a quantized=1 / 2 Darknet (training or eval) over NHWC fp32 tensors."""

    def __init__(self, model):
        self.model = model

    def forward(self, x):
        from .engine import LazyFeatures
        from .layout import feature_slots
        model = self.model
        defs, mods = model.module_defs, model.module_list
        dev = x.device
        h = x.float().permute(0, 2, 3, 1).contiguous()      # NCHW image -> NHWC fp32 (layout plumbing)
        outs = []
        yolo_out, io_list = [], []
        for i, (d, m) in enumerate(zip(defs, mods)):
            t = d['type']
            if t == 'convolutional':
                h = m[0](h)
            elif t == 'depthwise':
                if hasattr(m[0], 'weight_quantizer'):     # TPSQ: one quantised BN-folded layer (models.py:140-155)
                    h = m[0](h)
                else:                                     # google QAT: the float block
                    h = depthwise_block(m, d, h, model.training)
            elif t == 'se':
                h = se_layer(m.se, h)
            elif t == 'shortcut':
                name = m.__class__.__name__
                if name == 'Shortcut':           # TPSQ graphs keep the plain layers (models.py:275-305)
                    if getattr(m, 'weight', False):
                        raise NotImplementedError("weighted shortcut in the QAT graph")
                    for l in m.layers:
                        a = outs[l]
                        na, nx = a.shape[3], h.shape[3]
                        h = h + a if na == nx else (h + a[..., :nx] if na > nx else
                                                    torch.cat([h[..., :na] + a, h[..., na:]], 3))
                elif not hasattr(m, 'layers'):
                    pass        # shortcut_way not in {1, 2}: the reference leaves an empty Sequential (adds are skipped)
                else:
                    h = m(h, outs)
            elif t == 'route':
                if m.__class__.__name__ == 'FeatureConcat':
                    if m.multiple:
                        h = torch.cat([outs[l] for l in m.layers], 3)
                    else:
                        h = outs[m.layers[0]]
                        if getattr(m, 'groups', False):
                            h = h[..., h.shape[3] // 2:]
                else:
                    h = m(h, outs)
            elif t == 'upsample':
                s = int(d['stride'])
                h = h.repeat_interleave(s, dim=1).repeat_interleave(s, dim=2)
            elif t == 'maxpool':
                # plain nn.MaxPool2d (+ ZeroPad2d for the tiny k=2 s=1 variant) in the reference's QAT graphs as well
                # (models.py:207-215): values already sit on the producer's grid and pass through unchanged
                h = m(h.permute(0, 3, 1, 2)).permute(0, 2, 3, 1).contiguous()
            elif t == 'yolo':
                B, ny, nx, _ = h.shape
                m.nx, m.ny = nx, ny
                p = h[..., :m.na * m.no].reshape(B, ny, nx, m.na, m.no).permute(0, 3, 1, 2, 4).contiguous()
                if model.training:
                    yolo_out.append(p)
                else:
                    raw = h.contiguous()
                    io, pp = ops.yolo_decode(raw, m.na, m.no, m.anchors.to(dev).float().contiguous(), m.stride,
                                             io=torch.empty((B, m.na * ny * nx, m.no), dtype=torch.float32, device=dev))
                    io_list.append(io)
                    yolo_out.append(pp)
            else:
                raise NotImplementedError("layer type '%s' in the QAT graph" % t)
            outs.append(h if model.routs[i] else None)
        feats = LazyFeatures([None] * len(feature_slots(model)))
        if model.training:
            return yolo_out, feats
        return torch.cat(io_list, 1), tuple(yolo_out), feats
