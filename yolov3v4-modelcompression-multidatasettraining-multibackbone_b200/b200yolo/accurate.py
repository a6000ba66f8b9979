"""fp32-accurate inference mode (`model.accurate = True`, eval only).

The production path keeps activations and weights in fp16 (BASELINE configs[1]); every stored activation carries a
2^-11 relative rounding, which is what separates its detections from the fp32 reference's by ~1e-3 in probability and
keeps the held-batch mAP from matching to 1e-4 (a few candidates straddle the confidence threshold).  This mode exists
for that gate (SURVEY.md section 7 "hard parts"): the same wgmma convolution kernels, but

  * activations live in fp32 (NHWC) between layers and enter a conv as a two-term fp16 split x = x_hi + x_lo,
  * folded weights likewise w = w_hi + w_lo,
  * y = conv(x_hi, w_hi) + 2^-12 * conv([x_lo * 2^12 | x_hi], [w_hi | w_lo * 2^12])        (the x_lo * w_lo term, 2^-24, is dropped)

i.e. two launches of the fp16 implicit-GEMM kernel with fp32 accumulation and fp32 output per layer (the second over a
doubled K), every product exact, error ~2^-22 relative: fp32-class results at ~3x the tensor work.  Bias / activation /
shortcut / decode run in fp32 (activation + decode kernels; adds, nearest upsample and max-pool are torch tensor ops in
this verification mode).
"""
import torch

from . import ops
from .engine import LazyFeatures, fold_bn
from .layout import _block_parts, feature_slots


class AccurateRunner:
    def __init__(self, model):
        self.model = model
        self.cache = {}

    def _weights(self, i, conv, bn):
        key = (i, conv.weight._version, conv.weight.data_ptr())
        c = self.cache.get(i)
        if c is not None and c[0] == key:
            return c[1]
        w = conv.weight.detach().float()
        s, b = fold_bn(conv, bn)
        if s is not None:
            w = w * s.view(-1, 1, 1, 1)
        if b is None:
            b = torch.zeros(w.shape[0], device=w.device)
        I = w.shape[1]
        Ik = (I + 15) // 16 * 16
        if Ik != I:
            w = torch.nn.functional.pad(w, (0, 0, 0, 0, 0, Ik - I))
        hi = w.half().float()
        lo = ((w - hi) * 4096.0).half().float()
        w1, _, _ = ops.pack_conv_weights(hi.contiguous())
        w2, _, _ = ops.pack_conv_weights(torch.cat([hi, lo], 1).contiguous())
        out = (w1, w2, b.contiguous(), Ik)
        self.cache[i] = (key, out)
        return out

    def _conv(self, i, conv, bn, act, slope, x):
        w1, w2, b, Ik = self._weights(i, conv, bn)
        k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
        if x.shape[3] != Ik:
            x = torch.nn.functional.pad(x, (0, Ik - x.shape[3]))
        xh = x.half()
        xl = ((x - xh.float()) * 4096.0).half()
        y = ops.conv2d(xh.contiguous(), w1, None, k, s, p, out_dtype=torch.float32)
        y2 = ops.conv2d(torch.cat([xl, xh], 3).contiguous(), w2, None, k, s, p, out_dtype=torch.float32)
        y = y + y2 * (1.0 / 4096.0) + b
        if act != 'linear':
            y = ops.act_fwd(y, act, slope).view_as(y)
        return y

    @torch.no_grad()
    def forward(self, x):
        model = self.model
        if model.training:
            raise RuntimeError("model.accurate is an inference-only verification mode")
        defs, mods = model.module_defs, model.module_list
        dev = x.device
        h = x.float().permute(0, 2, 3, 1).contiguous()
        if x.dtype == torch.uint8:
            h = h / 256.0
        outs, io_list, p_list = [], [], []
        for i, (d, m) in enumerate(zip(defs, mods)):
            t = d['type']
            if t == 'convolutional':
                conv, bn, act, slope = _block_parts(m)
                if conv.groups != 1:
                    raise NotImplementedError("grouped convolution in the accurate mode")
                if conv.out_channels % 8 and not (i + 1 < len(defs) and defs[i + 1]['type'] == 'yolo'):
                    raise NotImplementedError("layer %d: %d channels; the accurate mode needs multiples of 8 outside "
                                              "the YOLO heads" % (i, conv.out_channels))
                h = self._conv(i, conv, bn, act, slope, h)
            elif t == 'shortcut':
                if getattr(m, 'weight', False):
                    raise NotImplementedError("weighted shortcut in the accurate mode")
                for l in m.layers:
                    a = outs[l]
                    n = min(a.shape[3], h.shape[3])
                    h = torch.cat([h[..., :n] + a[..., :n], h[..., n:]], 3) if h.shape[3] > n else h + a[..., :n]
            elif t == 'route':
                if m.multiple:
                    h = torch.cat([outs[l] for l in m.layers], 3)
                else:
                    h = outs[m.layers[0]]
                    if getattr(m, 'groups', False):
                        h = h[..., h.shape[3] // 2:]
            elif t == 'upsample':
                s = int(d['stride'])
                h = h.repeat_interleave(s, dim=1).repeat_interleave(s, dim=2)
            elif t == 'maxpool':
                k, s = int(d['size']), int(d['stride'])
                hc = h.permute(0, 3, 1, 2)
                if k == 2 and s == 1:
                    hc = torch.nn.functional.pad(hc, (0, 1, 0, 1))
                    hc = torch.nn.functional.max_pool2d(hc, k, s, 0)
                else:
                    hc = torch.nn.functional.max_pool2d(hc, k, s, (k - 1) // 2)
                h = hc.permute(0, 2, 3, 1).contiguous()
            elif t == 'yolo':
                B, ny, nx, _ = h.shape
                m.nx, m.ny = nx, ny
                raw = h.contiguous()
                io, pp = ops.yolo_decode(raw, m.na, m.no, m.anchors.to(dev).float().contiguous(), m.stride,
                                         io=torch.empty((B, m.na * ny * nx, m.no), dtype=torch.float32, device=dev))
                io_list.append(io)
                p_list.append(pp)
            else:
                raise NotImplementedError("layer type '%s' in the accurate mode" % t)
            outs.append(h if model.routs[i] else None)
        return torch.cat(io_list, 1), tuple(p_list), LazyFeatures([None] * len(feature_slots(model)))
