"""TPSQ layer zoo (quantized=2) under the reference's class names (reference utils/quantized/quantized_TPSQ.py):
Round :15, Search_Pow2 :29-63, Quantizer :66-130, range trackers :133-163, Bias_Quantizer :166-243, Weight_Quantizer
:245-287, Activattion_Quantizer :290-333, TPSQ_BNFold_QuantizedConv2d_For_FPGA :349-589.

The quantisation range is a LEARNED parameter `scale`, snapped to the nearest power of two P in every forward
(Search_Pow2, which also overwrites the parameter's data with P), with a soft clamp 0.5 (|x + P| - |x - P|), codes
round(c (2^(b-1) - 1) / P) and values code * P / 2^(b-1).  Forward and backward of that quantiser are device kernels
(b2y_tpsq_fwd_f32 / b2y_tpsq_bwd_f32: dx and the reduction sum(g * dy/dP) in one pass); the convolutions and the BN-fold
chain are the same as in the google QAT layer (b200yolo/qat.py).  Depthwise layers (groups = channels, MobileNet's
[depthwise] blocks) run both convolutions on the fp32 depthwise kernels (qat.dwconv_stats / qat.dwconv2d) with the same
fold; other grouped convolutions are not supported.  Module forwards take / return NHWC fp32 tensors.

Reference quirks kept: Weight_Quantizer passes `warmup` in the out_channels slot of its base class, so weights are never
warmed up (their scale parameter starts at 1.0); activations warm up on their first forward (99 candidates
max(x) / 100 * i, cosine similarity, first maximum wins).
"""
import math

import numpy as np
import torch
import torch.nn as nn
from torch.autograd import Function
from torch.nn import Parameter


class Round(Function):
    @staticmethod
    def forward(ctx, input):
        return torch.sign(input) * torch.floor(torch.abs(input) + 0.5)

    @staticmethod
    def backward(ctx, grad_output):
        return grad_output.clone()


class Quantizer(nn.Module):
    def __init__(self, bits, out_channels, warmup=False):
        super().__init__()
        self.first = True
        self.momentum = 0.1
        self.bits = bits
        self.register_buffer('warmup', torch.ones(1) if warmup else torch.zeros(1))

    def _pow2(self):
        from b200yolo import qat
        return qat.search_pow2(float(self.scale.detach().reshape(-1)[0]))

    def quantise_with(self, input, P):
        from b200yolo import qat
        out = qat.TpsqFn.apply(input, self.scale, P, self.bits)
        with torch.no_grad():
            self.scale.data.fill_(P)     # Search_Pow2.forward writes the snapped value into the parameter
        return out

    def warm_up(self, input):
        """99 candidate ranges step * i, step = max(x) / 100; keep the first one with the best cosine similarity."""
        from b200yolo import qat
        with torch.no_grad():
            x = input.detach().contiguous().float()
            step = float(x.max()) / 100.0
            cache, best, best_i = {}, -1.0, -5
            xn = x.reshape(-1)
            for i in range(1, 100):
                P = qat.search_pow2(step * i)
                if P not in cache:
                    y = qat.TpsqFn.apply(x, self.scale.detach(), P, self.bits).reshape(-1)
                    cache[P] = float(torch.nn.functional.cosine_similarity(xn, y, dim=0))
                if cache[P] > best:
                    best, best_i = cache[P], i
            self.scale.data.fill_(step * best_i)
            self.warmup.add_(-1)

    def forward(self, input):
        if self.bits == 32:
            return input
        assert self.bits != 1, 'Binary quantization is not supported'
        if not input.is_cuda:
            raise RuntimeError("TPSQ quantisers run on the CUDA device only (no CPU fallback)")
        if bool(self.warmup):
            self.warm_up(input)
        return self.quantise_with(input, self._pow2())

    def get_scale(self):
        return np.array(math.log2(self._pow2())).reshape(1, -1)


class Weight_Quantizer(Quantizer):
    def __init__(self, bits, out_channels, warmup):
        super().__init__(bits, warmup)           # (sic) reference :247: warmup lands in the out_channels slot -> no warm-up
        self.out_channels = out_channels
        self.scale = Parameter(torch.ones(1) if out_channels == -1 else torch.ones(out_channels, 1, 1, 1))


class Activattion_Quantizer(Quantizer):
    def __init__(self, bits, out_channels, warmup):
        super().__init__(bits, out_channels, warmup)
        self.out_channels = out_channels
        self.scale = Parameter(torch.ones(1) if out_channels == -1 else torch.ones(1, out_channels, 1, 1))


class RangeTracker(nn.Module):
    def update_range(self, min_val, max_val):
        raise NotImplementedError

    @torch.no_grad()
    def forward(self, input):
        from b200yolo import ops
        mm = ops.minmax(input.detach().reshape(1, -1), per_row=False)
        self.update_range(mm[0, 0].reshape(1), mm[0, 1].reshape(1))


class GlobalRangeTracker(RangeTracker):
    def __init__(self):
        super().__init__()
        self.register_buffer('min_val', torch.zeros(1))
        self.register_buffer('max_val', torch.zeros(1))
        self.register_buffer('first_w', torch.zeros(1))

    def update_range(self, min_val, max_val):
        if self.first_w == 0:
            self.first_w.add_(1)
            self.min_val.add_(min_val)
            self.max_val.add_(max_val)
        else:
            self.min_val.copy_(torch.min(min_val, self.min_val))
            self.max_val.copy_(torch.max(max_val, self.max_val))


class Bias_Quantizer(nn.Module):
    """symmetric power-of-two fake-quant on the running global |max| of the folded bias (reference :166-243)"""

    def __init__(self, bits, range_tracker):
        super().__init__()
        self.bits, self.range_tracker = bits, range_tracker
        self.register_buffer('scale', torch.zeros(1))

    def update_params(self):
        fmax = float(torch.max(self.range_tracker.min_val.abs(), self.range_tracker.max_val.abs()))
        fl, ce = 2.0 ** math.floor(math.log2(fmax)), 2.0 ** math.ceil(math.log2(fmax))
        self.scale = torch.full_like(self.scale, (ce if abs(ce - fmax) < abs(fl - fmax) else fl) / float(1 << (self.bits - 1)))

    def forward(self, input):
        from b200yolo import qat
        if self.bits == 32:
            return input
        if self.training:
            self.range_tracker(input)
            self.update_params()
        return qat.fake_quant(input, float(self.scale), self.bits)

    def get_scale(self):
        return np.array(math.log2(self.scale)).reshape(1, -1)


def reshape_to_activation(x):
    return x.reshape(1, -1, 1, 1)


def reshape_to_weight(x):
    return x.reshape(-1, 1, 1, 1)


def reshape_to_bias(x):
    return x.reshape(-1)


class TPSQ_BNFold_QuantizedConv2d_For_FPGA(nn.Conv2d):
    """reference :349-589.  forward(input): NHWC fp32 -> NHWC fp32."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=False,
                 eps=1e-5, momentum=0.01, a_bits=8, w_bits=8, bn=0, activate='leaky', steps=0, quantizer_output=False,
                 maxabsscaler=False, warmup=True):
        super().__init__(in_channels=in_channels, out_channels=out_channels, kernel_size=kernel_size, stride=stride,
                         padding=padding, dilation=dilation, groups=groups, bias=bias)
        self.bn, self.activate, self.eps, self.momentum = bn, activate, eps, momentum
        self.freeze_step = int(steps * 0.9)
        self.gamma = Parameter(torch.Tensor(out_channels))
        self.beta = Parameter(torch.Tensor(out_channels))
        self.register_buffer('running_mean', torch.zeros(out_channels))
        self.register_buffer('running_var', torch.zeros(out_channels))
        self.register_buffer('batch_mean', torch.zeros(out_channels))
        self.register_buffer('batch_var', torch.zeros(out_channels))
        self.register_buffer('first_bn', torch.zeros(1))
        self.register_buffer('step', torch.zeros(1))
        self.quantizer_output, self.maxabsscaler = quantizer_output, maxabsscaler
        nn.init.normal_(self.gamma, 1, 0.5)
        nn.init.zeros_(self.beta)
        self.activation_quantizer = Activattion_Quantizer(bits=a_bits, out_channels=-1, warmup=warmup)
        self.weight_quantizer = Weight_Quantizer(bits=w_bits, out_channels=-1, warmup=warmup)
        self.bias_quantizer = Bias_Quantizer(bits=w_bits, range_tracker=GlobalRangeTracker())

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
            raise RuntimeError("TPSQ layers run on the CUDA device only (no CPU fallback)")
        k, st, pd = self.kernel_size[0], self.stride[0], self.padding[0]
        link = None
        if self.training:
            self.step += 1
            if self.bn:
                weight, bias, link = qat.fold_batch_norm(self, input, k, st, pd, self.freeze_step)
            else:
                bias, weight = self.bias, self.weight
        else:
            weight, bias = self.BN_fuse()
        q_weight = self.weight_quantizer(weight)
        q_bias = self.bias_quantizer(bias)
        out = qat.qconv(self, input, q_weight, k, st, pd, link) + q_bias
        out = qat.activation(out, self.activate, self.maxabsscaler)
        return self.activation_quantizer(out)
