"""PTQ calibration forward (quantized=3, model.train()) on sm_90a -- what the reference's PTQ.py:76-88 calls before
the INT8 eval graph (qengine.py) can run.  Reference: utils/quantized/quantized_ptq_cos.py
  conv      :193-296 (fold, quantise W / b once, quantised conv + "correct" conv, bias correction), :543-567 activation,
            :717-721 activation quantiser vote
  shortcut  :836-884 (_min: per-addend votes, common scale = the smaller range, addends rounded NOT clamped, sum vote),
            :1158-1207 (_max: joint vote over the summed cosine similarities)
  concat    :1409-1432 (EMA of the per-input |max|, nearest power of two)

How it runs here.  In the reference every tensor of the quantised branch is an fp32 tensor whose values sit on a
power-of-two grid (int8 code x 2^e) and every conv is F.conv2d on those floats.  Such values (and the fake-quantised
weights) are exact in fp16 and their products / fp32 partial sums are exact, so the quantised conv runs on the wgmma
fp16 kernel with fp32 output and reproduces the reference's accumulators exactly (the int8 kernel cannot be used during
calibration: a concat of tensors with different scales has no single int8 scale, and the reference does not requantise
in training mode, :1533-1534).  The "correct" conv (quantised input x FLOAT folded weights, fp32 in the reference) uses a
two-term fp16 split of the weights (w = hi + lo * 2^-12), two tensor-core convs, ~2^-22 relative error.  The cosine
votes are the one-pass device kernel (b2y_cos_scale_search_ex); the few scalar statistics of the bias-correction rule are
torch reductions.  The reference's parallel FLOAT branch (float_output, second element of the [q, float] pairs) never
influences a scale, a bias or an output of the quantised branch; it is not computed.
"""
import math

import torch

from . import ops
from .engine import LazyFeatures
from .layout import feature_slots, sources


def _vote(values, scale_list, offset):
    """reference argmax rule: strict '>' from -1 keeps the FIRST maximum; then the mode of the vote histogram"""
    best, best_i = -1.0, 0
    for i, c in enumerate(values):
        if c > best:
            best, best_i = c, i
    scale_list[best_i] += 1
    return scale_list.index(max(scale_list)) + offset


class QCalibPlan:
    def __init__(self, model, x_shape, device):
        self.model, self.device = model, device
        self.B, self.Cin, self.H, self.W = x_shape

    # -- helpers ---------------------------------------------------------------------------------------------------
    @staticmethod
    def _round_noclamp(x, scale):
        return ops.fakequant_range(x, scale, -3.0e38, 3.0e38)

    def _conv(self, x16, w_oihw_f32_vals, k, s, p):
        """wgmma conv of fp16 NHWC values with weights given as fp32 OIHW whose values are exact in fp16 -> fp32"""
        wp, _, _ = ops.pack_conv_weights(w_oihw_f32_vals.contiguous())
        return ops.conv2d(x16, wp, None, k, s, p, out_dtype=torch.float32)

    def _conv_layer(self, i, conv, x16, is_first):
        k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
        if conv.groups != 1:
            raise NotImplementedError("depthwise PTQ calibration")
        conv.fold_and_quantize()            # fold BN, vote + quantise W and b once (:193-212)
        wq = conv.q_weight.detach().float()
        if float(wq.abs().max()) > 6.0e4:
            raise NotImplementedError("fake-quantised weights beyond the fp16 range")
        pad_c = x16.shape[3] - wq.shape[1]
        if pad_c:                            # layer 0: image channels padded to the MMA K granule
            wq = torch.nn.functional.pad(wq, (0, 0, 0, 0, 0, pad_c))
        acc = self._conv(x16, wq, k, s, p)                      # exact: sum of (code x 2^e) products
        if not conv.stop:
            out = acc + conv.q_bias.detach().float()
            w = conv.weight.detach().float()
            if pad_c:
                w = torch.nn.functional.pad(w, (0, 0, 0, 0, 0, pad_c))
            hi = w.half().float()
            lo = ((w - hi) * 4096.0).half().float()
            correct = self._conv(x16, hi, k, s, p) + self._conv(x16, lo, k, s, p) * (1.0 / 4096.0) \
                + conv.bias.detach().float()
            rate = 0.05
            error = out - correct
            noise = float(error.pow(2).mean())
            if noise > 0:
                eff = 1.25 * math.log10(float(correct.pow(2).mean()) / noise)
                dev = math.fabs(eff - conv.efficency)
                if dev > 0:
                    conv.efficency = (conv.efficency * 4 + eff) * 0.2
                    conv.deviation = (conv.deviation * 4 + dev) * 0.2
                    if conv.efficency > 4.0:
                        rate = rate * 0.5
                    if conv.efficency > 4.3 or (conv.deviation / conv.efficency) < 0.05 or \
                            math.fabs(dev - conv.deviation / dev) < 0.05:
                        conv.stop = True
                else:
                    conv.stop = True
            else:
                conv.stop = True
            if not conv.stop:
                with torch.no_grad():
                    conv.bias.data = conv.bias.data - rate * error.mean(dim=(0, 1, 2))
                    conv.q_bias = conv.bias_quantizer(conv.bias.detach())       # training mode: votes again
        out = acc + conv.q_bias.detach().float()
        slope = 0.25 if conv.maxabsscaler else 0.1
        if conv.activate != 'linear':
            out = ops.act_fwd(out, conv.activate, slope).view_as(out)
        return conv.activation_quantizer(out)                   # vote + fake-quantise (fp32 values on the new grid)

    def _shortcut(self, m, x, a):
        bits = m.bits
        qr = float(1 << (bits - 1))
        if getattr(m, 'weight', False):
            raise NotImplementedError("weighted quantised shortcut")
        if m.__class__.__name__ == 'COSPTQuantizedShortcut_min':
            for tag, t in (('a', a), ('x', x)):
                cos = ops.cos_scale_search(t, bits, n_cand=bits, step0=0).cpu().numpy()
                step = _vote(cos, getattr(m, 'scale_list_' + tag), 0)
                getattr(m, 'float_range_' + tag).fill_(2.0 ** step)
            fr = min(float(m.float_range_a), float(m.float_range_x))
            m.float_range_a.fill_(fr)
            m.float_range_x.fill_(fr)
            m.scale_a = m.float_range_a / qr
            m.scale_x = m.float_range_x / qr
        else:
            cos = None
            for t in (a, x, x + a):
                c = ops.cos_scale_search(t, bits, n_cand=bits, step0=0).cpu().numpy().astype('float32')
                cos = c if cos is None else cos + c
            if not hasattr(m, 'scale_list'):
                m.scale_list = [0 for _ in range(bits)]
            step = _vote(cos, m.scale_list, 0)
            for tag in ('a', 'x', 'sum'):
                getattr(m, 'float_range_' + tag).fill_(2.0 ** step)
                setattr(m, 'scale_' + tag, getattr(m, 'float_range_' + tag) / qr)
        xs = self._round_noclamp(x, float(m.scale_x)) + self._round_noclamp(a, float(m.scale_a))
        if m.__class__.__name__ == 'COSPTQuantizedShortcut_min':
            cos = ops.cos_scale_search(xs, bits, n_cand=bits, step0=0).cpu().numpy()
            step = _vote(cos, m.scale_list_sum, 0)
            m.float_range_sum.fill_(2.0 ** step)
            m.scale_sum = m.float_range_sum / qr
        return ops.fakequant(xs, float(m.scale_sum), bits).view_as(xs)

    def _concat(self, m, srcs):
        qr = float(1 << (m.bits - 1))
        with torch.no_grad():
            for j, t in enumerate(srcs):
                mx = ops.minmax(t.reshape(1, -1))[0]
                amax = torch.max(mx[1], mx[0].abs())
                if float(m.float_max_list[j]) == 0:
                    m.float_max_list[j].add_(amax)
                else:
                    m.float_max_list[j].mul_(1 - m.momentum).add_(amax * m.momentum)
            fmax = float(m.float_max_list.max())
            fl, ce = 2.0 ** math.floor(math.log2(fmax)), 2.0 ** math.ceil(math.log2(fmax))
            fr = ce if abs(ce - fmax) < abs(fl - fmax) else fl
            m.scale = torch.full_like(m.scale, fr / qr)
        return torch.cat(srcs, 3)           # training mode: no requantisation (:1533-1534)

    # -- forward ---------------------------------------------------------------------------------------------------
    def forward(self, x):
        model, dev = self.model, self.device
        defs, mods = model.module_defs, model.module_list
        B = x.shape[0]
        x = x.contiguous().float()
        img = torch.zeros((B, x.shape[2], x.shape[3], 16), dtype=torch.float16, device=dev)
        ops.nchw_to_nhwc(x, out=img[..., :x.shape[1]])
        outs = [None] * len(defs)
        cur = img            # fp16 NHWC for conv inputs; layer outputs are kept as fp32 NHWC values on their grids
        yolo_out = []
        for i, (d, m) in enumerate(zip(defs, mods)):
            t = d['type']
            if t == 'convolutional':
                src = img if i == 0 else outs[i - 1].half()
                outs[i] = self._conv_layer(i, m[0], src.contiguous(), i == 0)
            elif t == 'shortcut':
                if m.__class__.__name__ not in ('COSPTQuantizedShortcut_min', 'COSPTQuantizedShortcut_max'):
                    raise RuntimeError("quantized=3 needs shortcut_way 1 or 2 (models.py:275-305)")
                if len(d['from']) != 1:
                    raise NotImplementedError("multi-source quantised shortcut")
                outs[i] = self._shortcut(m, outs[i - 1], outs[sources(i, d['from'])[0]])
            elif t == 'route':
                srcs = sources(i, d['layers'])
                if len(srcs) == 1:
                    if 'groups' in d:
                        raise NotImplementedError("grouped route in the PTQ graph")
                    outs[i] = outs[srcs[0]]
                else:
                    outs[i] = self._concat(m, [outs[s] for s in srcs])
            elif t == 'upsample':
                outs[i] = ops.upsample(outs[i - 1].half().contiguous(), int(d['stride'])).float()
            elif t == 'yolo':
                raw = outs[i - 1].contiguous()
                _, p = ops.yolo_decode(raw, m.na, m.no, m.anchors.to(dev).float().contiguous(), m.stride, io=None)
                m.nx, m.ny = raw.shape[2], raw.shape[1]
                yolo_out.append(p)
            else:
                raise NotImplementedError("layer type '%s' in the PTQ graph" % t)
        return yolo_out, LazyFeatures([None] * len(feature_slots(model)))
