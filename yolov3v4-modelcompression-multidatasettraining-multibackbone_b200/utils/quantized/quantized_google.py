"""QAT layer zoo (quantized=1) under the reference's class names (reference utils/quantized/quantized_google.py):
RangeTracker family :16-77, Round (STE) :81, Quantizer family :95-219, BNFold_QuantizedConv2d_For_FPGA :235-836,
QuantizedShortcut_max/min :839/1066, QuantizedFeatureConcat :1305.

The module forwards run on NHWC fp32 tensors (b200yolo/qat.py QatRunner drives them from Darknet.forward) and are
composed of the sm_90a kernels: wgmma convolutions (forward / data gradient / weight gradient, fp32 accumulation,
BatchNorm channel sums from the conv epilogue), b2y_minmax_f32 (range trackers), b2y_fakequant_f32 with its
straight-through backward, activation forward / backward.  torch.autograd chains them and differentiates the [C]-sized
fold arithmetic (batch-statistics fold -> frozen running-statistics fold at 0.9 * steps, google.py:349-370).
Depthwise layers (groups = channels: GhostNet's cheap operations, [convolutional] groups=C) run both convolutions on the
fp32 depthwise kernels (qat.dwconv_stats / qat.dwconv2d) with the same fold, as the TPSQ layer does; other grouped
convolutions are refused.
"""
import math
import torch
import torch.nn as nn
from torch.autograd import Function
from torch.nn import Parameter


class RangeTracker(nn.Module):
    def __init__(self, q_level):
        super().__init__()
        self.q_level = q_level

    def update_range(self, min_val, max_val):
        raise NotImplementedError

    @torch.no_grad()
    def forward(self, input):
        from b200yolo import ops
        if self.q_level == 'L':
            mm = ops.minmax(input.reshape(1, -1), per_row=False)
            min_val, max_val = mm[0, 0].reshape(1), mm[0, 1].reshape(1)
        else:  # 'C': per output channel (dim 0)
            mm = ops.minmax(input.reshape(input.shape[0], -1), per_row=True)
            min_val, max_val = mm[:, 0].reshape(-1, 1, 1, 1), mm[:, 1].reshape(-1, 1, 1, 1)
        self.update_range(min_val, max_val)


class GlobalRangeTracker(RangeTracker):
    def __init__(self, q_level, out_channels):
        super().__init__(q_level)
        shape = (1,) if q_level == 'L' else (out_channels, 1, 1, 1)
        self.register_buffer('min_val', torch.zeros(shape))
        self.register_buffer('max_val', torch.zeros(shape))
        self.register_buffer('first_w', torch.zeros(1))

    def update_range(self, min_val, max_val):
        if self.first_w == 0:
            self.first_w.add_(1)
            self.min_val.add_(min_val)
            self.max_val.add_(max_val)
        else:
            self.min_val.copy_(torch.min(min_val, self.min_val))
            self.max_val.copy_(torch.max(max_val, self.max_val))


class AveragedRangeTracker(RangeTracker):
    def __init__(self, q_level, out_channels, momentum=0.1):
        super().__init__(q_level)
        self.momentum = momentum
        shape = (1,) if q_level == 'L' else (out_channels, 1, 1, 1)
        self.register_buffer('min_val', torch.zeros(shape))
        self.register_buffer('max_val', torch.zeros(shape))
        self.register_buffer('first_a', torch.zeros(1))

    def update_range(self, min_val, max_val):
        if self.first_a == 0:
            self.first_a.add_(1)
            self.min_val.add_(min_val)
            self.max_val.add_(max_val)
        else:
            self.min_val.mul_(1 - self.momentum).add_(min_val * self.momentum)
            self.max_val.mul_(1 - self.momentum).add_(max_val * self.momentum)


class Round(Function):
    @staticmethod
    def forward(ctx, input):
        return torch.sign(input) * torch.floor(torch.abs(input) + 0.5)

    @staticmethod
    def backward(ctx, grad_output):
        return grad_output.clone()


class Quantizer(nn.Module):
    """reference :95-168.  NB the reference signature is (bits, range_tracker, out_channels, Scale_freeze_step, sign)."""

    def __init__(self, bits, range_tracker, out_channels, Scale_freeze_step, sign=True):
        super().__init__()
        self.bits, self.range_tracker, self.Scale_freeze_step, self.sign = bits, range_tracker, Scale_freeze_step, sign
        shape = (1,) if out_channels == -1 else (out_channels, 1, 1, 1)
        self.register_buffer('step', torch.zeros(1))
        self.register_buffer('scale', torch.zeros(shape))
        self.register_buffer('zero_point', torch.zeros(shape))

    def update_params(self):
        raise NotImplementedError

    def forward(self, input):
        from b200yolo import qat
        if self.bits == 32:
            return input
        assert self.bits != 1, 'Binary quantization is not supported'
        if not input.is_cuda:
            raise RuntimeError("QAT quantisers run on the CUDA device only (no CPU fallback)")
        if self.training and float(self.step) < self.Scale_freeze_step:
            self.range_tracker(input.detach())
            self.update_params()
        if self.scale.numel() != 1 or float(self.zero_point.reshape(-1)[0]) != 0.0:
            raise NotImplementedError("per-channel / asymmetric fake-quant (the FPGA layers use layer-level symmetric)")
        out = qat.fake_quant(input, float(self.scale.reshape(-1)[0]), self.bits, sign=self.sign)
        self.step += 1
        return out

    def get_quantize_value(self, input):
        if self.bits == 32:
            return input
        q = Round.apply(input / self.scale + self.zero_point)
        lo, hi = (-(1 << (self.bits - 1)), (1 << (self.bits - 1)) - 1) if self.sign else (0, (1 << self.bits) - 1)
        return torch.clamp(q, lo, hi)

    def get_scale(self):
        import numpy as np
        return np.array(math.log2(self.scale)).reshape(1, -1)


def _nearest_pow2(v):
    """2^floor(log2 v) or 2^ceil(log2 v), whichever is closer; ties go to the floor (reference :186-196)"""
    fl, ce = 2.0 ** math.floor(math.log2(v)), 2.0 ** math.ceil(math.log2(v))
    return ce if abs(ce - v) < abs(fl - v) else fl


class SymmetricQuantizer(Quantizer):
    def update_params(self):
        qr = float(1 << (self.bits - 1)) if self.sign else float((1 << self.bits) - 1)
        fmax = float(torch.max(self.range_tracker.min_val.abs(), self.range_tracker.max_val.abs()).reshape(-1)[0])
        self.scale = torch.full_like(self.scale, _nearest_pow2(fmax) / qr)
        self.zero_point = torch.zeros_like(self.scale)


class AsymmetricQuantizer(Quantizer):
    def update_params(self):
        lo, hi = (-(1 << (self.bits - 1)), (1 << (self.bits - 1)) - 1) if self.sign else (0, (1 << self.bits) - 1)
        fr = float((self.range_tracker.max_val - self.range_tracker.min_val).reshape(-1)[0])
        self.scale = torch.full_like(self.scale, _nearest_pow2(fr) / float(hi - lo))
        self.zero_point = torch.round(hi - self.range_tracker.max_val / self.scale)


def reshape_to_activation(x):
    return x.reshape(1, -1, 1, 1)


def reshape_to_weight(x):
    return x.reshape(-1, 1, 1, 1)


def reshape_to_bias(x):
    return x.reshape(-1)


class BNFold_QuantizedConv2d_For_FPGA(nn.Conv2d):
    """reference :235-836.  forward(input): NHWC fp32 -> NHWC fp32 (values on the activation quantiser's grid)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=False,
                 eps=1e-5, momentum=0.01, a_bits=8, w_bits=8, q_type=0, bn=0, activate='leaky', steps=0,
                 quantizer_output=False, reorder=False, TM=32, TN=32, name='', layer_idx=-1, maxabsscaler=False):
        super().__init__(in_channels=in_channels, out_channels=out_channels, kernel_size=kernel_size, stride=stride,
                         padding=padding, dilation=dilation, groups=groups, bias=bias)
        self.bn, self.activate, self.eps, self.momentum = bn, activate, eps, momentum
        self.BN_freeze_step = int(steps * 0.9)
        self.Scale_freeze_step = int(steps * 0.1)
        self.gamma = Parameter(torch.Tensor(out_channels))
        self.beta = Parameter(torch.Tensor(out_channels))
        self.register_buffer('running_mean', torch.zeros(out_channels))
        self.register_buffer('running_var', torch.zeros(out_channels))
        self.register_buffer('batch_mean', torch.zeros(out_channels))
        self.register_buffer('batch_var', torch.zeros(out_channels))
        self.register_buffer('first_bn', torch.zeros(1))
        self.register_buffer('step', torch.zeros(1))
        self.quantizer_output, self.reorder, self.TM, self.TN = quantizer_output, reorder, TM, TN
        self.name, self.layer_idx, self.w_bits, self.a_bits, self.maxabsscaler = name, layer_idx, w_bits, a_bits, maxabsscaler
        nn.init.normal_(self.gamma, 1, 0.5)
        nn.init.zeros_(self.beta)
        Q = SymmetricQuantizer if q_type == 0 else AsymmetricQuantizer
        sign = q_type == 0
        self.activation_quantizer = Q(bits=a_bits, range_tracker=AveragedRangeTracker(q_level='L', out_channels=-1),
                                      out_channels=-1, Scale_freeze_step=self.Scale_freeze_step, sign=sign)
        self.weight_quantizer = Q(bits=w_bits, range_tracker=GlobalRangeTracker(q_level='L', out_channels=-1),
                                  out_channels=-1, Scale_freeze_step=self.Scale_freeze_step, sign=sign)
        self.bias_quantizer = Q(bits=w_bits, range_tracker=GlobalRangeTracker(q_level='L', out_channels=-1),
                                out_channels=-1, Scale_freeze_step=self.Scale_freeze_step, sign=sign)

    def BN_fuse(self):
        if self.bn:
            s = self.gamma / torch.sqrt(self.running_var + self.eps)
            bias = reshape_to_bias(self.beta + ((self.bias if self.bias is not None else 0) - self.running_mean) * s)
            return self.weight * reshape_to_weight(s), bias
        return self.weight, self.bias

    def forward(self, input):
        from b200yolo import qat
        qat.check_groups(self)
        if not input.is_cuda:
            raise RuntimeError("QAT layers run on the CUDA device only (no CPU fallback)")
        k, st, pd = self.kernel_size[0], self.stride[0], self.padding[0]
        link = None
        if self.training:
            self.step += 1
            if self.bn:
                # plain conv for the batch statistics (:326-338), then the fold (:349-370)
                weight, bias, link = qat.fold_batch_norm(self, input, k, st, pd, self.BN_freeze_step)
            else:
                bias, weight = self.bias, self.weight
        else:
            weight, bias = self.BN_fuse()
        q_weight = self.weight_quantizer(weight)
        q_bias = self.bias_quantizer(bias)
        out = qat.qconv(self, input, q_weight, k, st, pd, link) + q_bias
        out = qat.activation(out, self.activate, self.maxabsscaler)
        return self.activation_quantizer(out)


class _QShortcut(nn.Module):
    def __init__(self, layers, weight=False, bits=8, quantizer_output=False, reorder=False, TM=32, TN=32, name='',
                 layer_idx=-1):
        super().__init__()
        self.layers, self.weight, self.n, self.bits = layers, weight, len(layers) + 1, bits
        self.range_tracker_x = AveragedRangeTracker(q_level='L', out_channels=-1)
        self.range_tracker_a = AveragedRangeTracker(q_level='L', out_channels=-1)
        self.quantizer_output, self.reorder, self.TM, self.TN, self.name, self.layer_idx = \
            quantizer_output, reorder, TM, TN, name, layer_idx
        if weight:
            self.w = nn.Parameter(torch.zeros(self.n), requires_grad=True)

    def _pow2_scale(self, fmin, fmax):
        v = max(abs(float(fmin)), abs(float(fmax)))
        return _nearest_pow2(v) / float(1 << (self.bits - 1))

    @staticmethod
    def _add(x, a):
        nx, na = x.shape[3], a.shape[3]
        if nx == na:
            return x + a
        if nx > na:
            return torch.cat([x[..., :na] + a, x[..., na:]], 3)
        return x + a[..., :nx]


class QuantizedShortcut_max(_QShortcut):
    """reference :839-1063: one scale from the joint range of x, a and x + a; addends and sum are clamped."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.range_tracker_sum = AveragedRangeTracker(q_level='L', out_channels=-1)
        self.register_buffer('scale', torch.zeros(1))

    def forward(self, x, outputs):
        from b200yolo import qat
        if self.weight:
            w = torch.sigmoid(self.w) * (2 / self.n)
            x = x * w[0]
        for i in range(self.n - 1):
            a = outputs[self.layers[i]] * w[i + 1] if self.weight else outputs[self.layers[i]]
            if self.training:
                self.range_tracker_a(x.detach())          # (sic: the reference feeds x to tracker_a and a to tracker_x)
                self.range_tracker_x(a.detach())
                self.range_tracker_sum(self._add(x, a).detach())
                fmax = max(float(self.range_tracker_sum.max_val), float(self.range_tracker_x.max_val),
                           float(self.range_tracker_a.max_val))
                fmin = min(float(self.range_tracker_sum.min_val), float(self.range_tracker_x.min_val),
                           float(self.range_tracker_a.min_val))
                self.scale = torch.full_like(self.scale, self._pow2_scale(fmin, fmax))
            s = float(self.scale)
            x = self._add(qat.fake_quant(x, s, self.bits), qat.fake_quant(a, s, self.bits))
            x = qat.fake_quant(x, s, self.bits)
        return x


class QuantizedShortcut_min(_QShortcut):
    """reference :1066-1302: addends rounded (not clamped) onto the smaller of the two ranges, the sum is quantised with
    the sum tracker's own scale."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.range_tracker_sum = AveragedRangeTracker(q_level='L', out_channels=-1)
        self.register_buffer('scale', torch.zeros(1))
        self.register_buffer('input_scale', torch.zeros(1))

    def forward(self, x, outputs):
        from b200yolo import qat
        if self.weight:
            w = torch.sigmoid(self.w) * (2 / self.n)
            x = x * w[0]
        for i in range(self.n - 1):
            a = outputs[self.layers[i]] * w[i + 1] if self.weight else outputs[self.layers[i]]
            if self.training:
                self.range_tracker_a(a.detach())
                self.range_tracker_x(x.detach())
                fmax = min(float(self.range_tracker_x.max_val), float(self.range_tracker_a.max_val))
                fmin = max(float(self.range_tracker_x.min_val), float(self.range_tracker_a.min_val))
                self.input_scale = torch.full_like(self.input_scale, self._pow2_scale(fmin, fmax))
            si = float(self.input_scale)
            x = self._add(qat.fake_quant(x, si, self.bits, clamp=False), qat.fake_quant(a, si, self.bits, clamp=False))
            if self.training:
                self.range_tracker_sum(x.detach())
                self.scale = torch.full_like(self.scale, self._pow2_scale(float(self.range_tracker_sum.min_val),
                                                                          float(self.range_tracker_sum.max_val)))
            x = qat.fake_quant(x, float(self.scale), self.bits)
        return x


class QuantizedFeatureConcat(nn.Module):
    """reference :1305-1500: EMA of the per-input |max| -> nearest power of two -> every input requantised onto it."""

    def __init__(self, layers, groups, bits=8, quantizer_output=False, reorder=False, TM=32, TN=32, name='',
                 layer_idx=-1):
        super().__init__()
        self.layers, self.groups, self.multiple, self.bits, self.momentum = layers, groups, len(layers) > 1, bits, 0.1
        self.register_buffer('scale', torch.zeros(1))
        self.register_buffer('float_max_list', torch.zeros(len(layers)))
        self.quantizer_output, self.reorder, self.TM, self.TN, self.name, self.layer_idx = \
            quantizer_output, reorder, TM, TN, name, layer_idx

    def forward(self, x, outputs):
        from b200yolo import ops, qat
        if self.multiple:
            if self.training:
                with torch.no_grad():
                    for j, i in enumerate(self.layers):
                        mm = ops.minmax(outputs[i].detach().reshape(1, -1))[0]
                        amax = torch.max(mm[1], mm[0].abs())
                        if float(self.float_max_list[j]) == 0:
                            self.float_max_list[j].add_(amax)
                        else:
                            self.float_max_list[j].mul_(1 - self.momentum).add_(amax * self.momentum)
                    fmax = float(self.float_max_list.max())
                    self.scale = torch.full_like(self.scale, _nearest_pow2(fmax) / float(1 << (self.bits - 1)))
            s = float(self.scale)
            for i in self.layers:        # (the reference overwrites the stored outputs with their requantised version)
                outputs[i] = qat.fake_quant(outputs[i], s, self.bits)
            return torch.cat([outputs[i] for i in self.layers], 3)
        if self.groups:
            return x[..., x.shape[3] // 2:]
        return outputs[self.layers[0]]
