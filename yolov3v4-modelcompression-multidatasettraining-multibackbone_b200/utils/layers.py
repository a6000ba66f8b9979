"""Layer library under the reference's class names (reference utils/layers.py): FeatureConcat :26, Shortcut :43,
Mish :146 (analytic backward :117-128), Swish :141, ReLU6 :151, HardSwish :159, HardSigmoid :167, SE :176.

These nn.Modules define the *graph* (class names are what Darknet.forward_once dispatches on, models.py:525-543)
and hold parameters; on a CUDA device the whole graph is executed by the fused sm_90a engine
(b200yolo/engine.py), and the standalone activation modules call the CUDA kernels directly."""
from utils.utils import *  # noqa: F401,F403  (the reference's star-import chain: torch, nn, F, np, math ...)


def make_divisible(v, divisor):
    return math.ceil(v / divisor) * divisor


class Flatten(nn.Module):
    def forward(self, x):
        return x.view(x.size(0), -1)


class Concat(nn.Module):
    def __init__(self, dimension=1):
        super().__init__()
        self.d = dimension

    def forward(self, x):
        return torch.cat(x, self.d)


class FeatureConcat(nn.Module):
    """route layer: concat of earlier outputs along C, alias of one output, or its upper channel half (groups)."""

    def __init__(self, layers, groups):
        super().__init__()
        self.layers = layers
        self.groups = groups
        self.multiple = len(layers) > 1

    def forward(self, x, outputs):
        if self.multiple:
            return torch.cat([outputs[i] for i in self.layers], 1)
        if self.groups:
            return x[:, (x.shape[1] // 2):]
        return outputs[self.layers[0]]


class Shortcut(nn.Module):
    """residual add of earlier outputs (optionally sigmoid-weighted, channel-sliced when widths differ)."""

    def __init__(self, layers, weight=False):
        super().__init__()
        self.layers = layers
        self.weight = weight
        self.n = len(layers) + 1
        if weight:
            self.w = nn.Parameter(torch.zeros(self.n), requires_grad=True)

    def forward(self, x, outputs):
        if self.weight:
            w = torch.sigmoid(self.w) * (2 / self.n)
            x = x * w[0]
        nx = x.shape[1]
        for i in range(self.n - 1):
            a = outputs[self.layers[i]] * w[i + 1] if self.weight else outputs[self.layers[i]]
            na = a.shape[1]
            if nx == na:
                x = x + a
            elif nx > na:
                x[:, :na] = x[:, :na] + a
            else:
                x = x + a[:, :nx]
        return x


class _B2YActivation(torch.autograd.Function):
    """Elementwise activation forward/backward through the CUDA kernels (b2y_act_fwd_f32 / b2y_act_bwd_f32)."""

    @staticmethod
    def forward(ctx, x, act, slope):
        from b200yolo import ops
        ctx.save_for_backward(x)
        ctx.act, ctx.slope = act, slope
        return ops.act_fwd(x, act, slope).view_as(x).to(x.dtype)

    @staticmethod
    def backward(ctx, grad_output):
        from b200yolo import ops
        (x,) = ctx.saved_tensors
        return ops.act_bwd(x, grad_output, ctx.act, ctx.slope).view_as(x).to(x.dtype), None, None


def _device_act(x, act, slope=0.1):
    if not x.is_cuda:
        raise RuntimeError("b200yolo activations run on a CUDA device only (no CPU fallback); got a %s tensor"
                           % x.device.type)
    return _B2YActivation.apply(x, act, slope)


class SwishImplementation(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return _B2YActivation.forward(ctx, x, 'swish', 0.0)

    @staticmethod
    def backward(ctx, grad_output):
        return _B2YActivation.backward(ctx, grad_output)[0]


class MishImplementation(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return _B2YActivation.forward(ctx, x, 'mish', 0.0)

    @staticmethod
    def backward(ctx, grad_output):
        return _B2YActivation.backward(ctx, grad_output)[0]


class MemoryEfficientSwish(nn.Module):
    def forward(self, x):
        return SwishImplementation.apply(x)


class MemoryEfficientMish(nn.Module):
    def forward(self, x):
        return MishImplementation.apply(x)


class Swish(nn.Module):
    def forward(self, x):
        return _device_act(x, 'swish')


class Mish(nn.Module):
    """x * tanh(softplus(x)), softplus threshold 20 (csrc/common.cuh mish_f)."""

    def forward(self, x):
        return _device_act(x, 'mish')


class ReLU6(nn.Module):
    def forward(self, x):
        return _device_act(x, 'relu6')


class HardSwish(nn.Module):
    def forward(self, x):
        return _device_act(x, 'h_swish')


class HardSigmoid(nn.Module):
    def forward(self, x):
        return F.relu6(x + 3.0) / 6.0


class SE(nn.Module):
    """squeeze-excite: avgpool -> Linear(C, C/r) -> ReLU -> Linear(C/r, C) -> HardSigmoid -> channel scale."""

    def __init__(self, channel, reduction=4):
        super().__init__()
        self.avg_pool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Sequential(nn.Linear(channel, channel // reduction, bias=False), nn.ReLU(inplace=True),
                                nn.Linear(channel // reduction, channel, bias=False), HardSigmoid())

    def forward(self, x):
        b, c = x.shape[:2]
        gate = self.fc(self.avg_pool(x).view(b, c)).view(b, c, 1, 1)
        return x * gate.expand_as(x)
