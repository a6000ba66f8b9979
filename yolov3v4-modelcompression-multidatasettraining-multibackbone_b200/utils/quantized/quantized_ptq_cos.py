"""Post-training quantisation layer zoo (quantized=3) under the reference's class names
(reference utils/quantized/quantized_ptq_cos.py): Round :14, Quantizer :23-113, BNFold_COSPTQuantizedConv2d_For_FPGA
:131-738, COSPTQuantizedShortcut_min :741 / _max :1058, COSPTQuantizedFeatureConcat :1364.

The modules carry the same parameters / buffers (state_dict keys of a reference-calibrated PTQ.pt load unchanged);
the calibrated eval forward of the whole graph is executed in true INT8 by b200yolo/qengine.py
(int8 wgmma convs, int32 accumulation, power-of-two rescale in the epilogue).
"""
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F  # noqa: F401
from torch.autograd import Function
from torch.nn import Parameter


def reshape_to_activation(x):
    return x.reshape(1, -1, 1, 1)


def reshape_to_weight(x):
    return x.reshape(-1, 1, 1, 1)


def reshape_to_bias(x):
    return x.reshape(-1)


class Round(Function):
    """round half away from zero: sign(x) * floor(|x| + 0.5)   (b2y_fakequant_f32 uses the same rule)"""

    @staticmethod
    def forward(ctx, input):
        return torch.sign(input) * torch.floor(torch.abs(input) + 0.5)

    @staticmethod
    def backward(ctx, grad_output):
        return grad_output.clone()


class Quantizer(nn.Module):
    """layer-level power-of-two quantiser: scale = 2^step / 2^(bits-1); calibration picks `step` by cosine similarity
    over the bits+7 candidates step = i-5 and a running vote (scale_list), one fused pass on the device."""

    def __init__(self, bits, out_channels):
        super().__init__()
        self.bits = bits
        shape = (1,) if out_channels == -1 else (out_channels, 1, 1, 1)
        self.register_buffer('scale', torch.zeros(shape))
        self.register_buffer('float_range', torch.zeros(shape))
        self.scale_list = [0 for _ in range(bits + 7)]

    def update_params(self, step):
        quantized_range = float(1 << (self.bits - 1))
        self.float_range.fill_(2.0 ** step)
        self.scale = self.float_range / quantized_range

    def quantize(self, input):
        return input / self.scale

    def round(self, input):
        return Round.apply(input)

    def clamp(self, input):
        return torch.clamp(input, -(1 << (self.bits - 1)), (1 << (self.bits - 1)) - 1)

    def dequantize(self, input):
        return input * self.scale

    def calibrate(self, input):
        """one calibration vote (reference :71-87): argmax of the cosine similarities with the first-wins '>' rule."""
        from b200yolo import ops
        cos = ops.cos_scale_search(input, self.bits).cpu().numpy()
        best, best_i = -1.0, 0
        for i, c in enumerate(cos):
            if c > best:
                best, best_i = c, i
        self.scale_list[best_i] += 1
        self.update_params(self.scale_list.index(max(self.scale_list)) - 5)

    def forward(self, input):
        if self.bits == 32:
            return input
        assert self.bits != 1, 'Binary quantization is not supported'
        if not input.is_cuda:
            raise RuntimeError("Quantizer runs on the CUDA device only (no CPU fallback)")
        from b200yolo import ops
        if self.training:
            self.calibrate(input)
        return ops.fakequant(input, float(self.scale.reshape(-1)[0]), self.bits).view_as(input)

    def get_quantize_value(self, input):
        if self.bits == 32:
            return input
        return self.clamp(self.round(self.quantize(input)))

    def get_scale(self):
        return np.array(math.log2(self.scale)).reshape(1, -1)


class BNFold_COSPTQuantizedConv2d_For_FPGA(nn.Conv2d):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=False,
                 eps=1e-5, momentum=0.1, a_bits=8, w_bits=8, bn=0, activate='leaky', quantizer_output=False,
                 reorder=False, TM=32, TN=32, name='', layer_idx=-1, maxabsscaler=False):
        super().__init__(in_channels=in_channels, out_channels=out_channels, kernel_size=kernel_size, stride=stride,
                         padding=padding, dilation=dilation, groups=groups, bias=bias)
        self.bn = bn
        if bias is False:
            self.bias = Parameter(torch.zeros(out_channels))
        self.activate = activate
        self.eps = eps
        self.momentum = momentum
        self.gamma = Parameter(torch.ones(out_channels))
        self.beta = Parameter(torch.zeros(out_channels))
        self.register_buffer('running_mean', torch.zeros(out_channels))
        self.register_buffer('running_var', torch.zeros(out_channels))
        self.register_buffer('q_bias', torch.zeros(out_channels))
        self.register_buffer('q_weight', torch.zeros(self.weight.shape))
        self.efficency = 0
        self.deviation = 0
        self.stop = False
        self.quantized = False
        self.quantizer_output = quantizer_output
        self.reorder, self.TM, self.TN = reorder, TM, TN
        self.name, self.layer_idx, self.maxabsscaler = name, layer_idx, maxabsscaler
        self.a_bits, self.w_bits = a_bits, w_bits
        self.activation_quantizer = Quantizer(bits=a_bits, out_channels=-1)
        self.weight_quantizer = Quantizer(bits=w_bits, out_channels=-1)
        self.bias_quantizer = Quantizer(bits=w_bits, out_channels=-1)

    def BN_fuse(self):
        """(folded weight, folded bias) without touching the module (reference :723-738)."""
        if self.bn:
            s = self.gamma / torch.sqrt(self.running_var + self.eps)
            bias = reshape_to_bias(self.beta + (self.bias - self.running_mean) * s)
            return self.weight * reshape_to_weight(s), bias
        return self.weight, self.bias

    def fold_and_quantize(self):
        """First-call behaviour of the reference forward (:193-212): destructive BN fold into weight.data / bias.data,
        then quantise W and b once with their layer-level quantisers (whose scales must be calibrated or loaded)."""
        if self.quantized:
            return
        from b200yolo import ops
        with torch.no_grad():
            if self.bn:
                s = self.gamma / torch.sqrt(self.running_var + self.eps)
                self.bias.data = reshape_to_bias(self.beta + (self.bias - self.running_mean) * s)
                self.weight.data = self.weight * reshape_to_weight(s)
            for q, src, dst in ((self.weight_quantizer, self.weight, 'q_weight'),
                                (self.bias_quantizer, self.bias, 'q_bias')):
                if float(q.scale.reshape(-1)[0]) == 0.0:
                    q.calibrate(src.detach())
                setattr(self, dst, ops.fakequant(src.detach(), float(q.scale.reshape(-1)[0]), q.bits).view_as(src))
        self.quantized = True

    def forward(self, input):
        raise RuntimeError("BNFold_COSPTQuantizedConv2d_For_FPGA is executed by the INT8 graph engine "
                           "(Darknet.forward on a CUDA device); module-level forward is not part of the hot path")


class _QuantShortcutBase(nn.Module):
    def __init__(self, layers, weight=False, bits=8, quantizer_output=False, reorder=False, TM=32, TN=32, name='',
                 layer_idx=-1):
        super().__init__()
        self.layers = layers
        self.weight = weight
        self.n = len(layers) + 1
        self.bits = bits
        for tag in ('x', 'a', 'sum'):
            self.register_buffer('scale_' + tag, torch.zeros(1))
            self.register_buffer('float_range_' + tag, torch.zeros(1))
            setattr(self, 'scale_list_' + tag, [0 for _ in range(bits)])
        self.quantizer_output = quantizer_output
        self.reorder, self.TM, self.TN, self.name, self.layer_idx = reorder, TM, TN, name, layer_idx
        if weight:
            self.w = nn.Parameter(torch.zeros(self.n), requires_grad=True)

    def forward(self, x, outputs):
        raise RuntimeError("quantised shortcut layers are executed by the INT8 graph engine (b2y_qshortcut_i8)")


class COSPTQuantizedShortcut_min(_QuantShortcutBase):
    """addends rounded (not clamped) onto the smaller of their two power-of-two ranges, sum requantised + clamped."""
    clamp_addends = False


class COSPTQuantizedShortcut_max(_QuantShortcutBase):
    """as _min, but the common addend scale comes from a joint search (reference :1158-1197)."""
    clamp_addends = False


class COSPTQuantizedFeatureConcat(nn.Module):
    def __init__(self, layers, groups, bits=8, quantizer_output=False, reorder=False, TM=32, TN=32, name='',
                 layer_idx=-1):
        super().__init__()
        self.layers = layers
        self.groups = groups
        self.multiple = len(layers) > 1
        self.register_buffer('scale', torch.zeros(1))
        self.register_buffer('float_max_list', torch.zeros(len(layers)))
        self.bits = bits
        self.momentum = 0.1
        self.quantizer_output = quantizer_output
        self.reorder, self.TM, self.TN, self.name, self.layer_idx = reorder, TM, TN, name, layer_idx

    def forward(self, x, outputs):
        raise RuntimeError("quantised concat layers are executed by the INT8 graph engine (b2y_requant_i8)")
