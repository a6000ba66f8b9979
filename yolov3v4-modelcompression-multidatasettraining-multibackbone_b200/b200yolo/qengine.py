"""INT8 graph executor for a PTQ-calibrated Darknet (quantized=3, reference PTQ.py:92-102 eval path).

The reference *simulates* int8 in fp32: every tensor is a float on a power-of-two grid, convs are F.conv2d on those
floats (utils/quantized/quantized_ptq_cos.py:288-296).  Because all scales are powers of two the products are exact
integers times a power of two, so the same arithmetic runs here on the real int8 codes:

   conv      int8 x int8 -> int32 on int8 wgmma, epilogue  acc*(s_in*s_w) + q_bias -> act -> requant(s_act)
   shortcut  folded into the epilogue of the conv that feeds it (b2y_qconv2d_shortcut_fwd) when nothing else reads that
             conv's output; otherwise b2y_qshortcut_i8 (both addends rounded onto scale_x / scale_a, sum requantised)
   concat    b2y_requant_i8 of every source onto the concat scale, written into its channel slot
   upsample  nearest copy of codes
   layer 0   fp32 direct conv of the float image on the fake-quantised weights (as the reference), int8 out
   heads     fp32 fake-quant values for the (fp32) YOLO decode kernel
"""
import ctypes as C
import os

import torch

from . import ops
from .layout import _Tensor, infer_shapes, sources, stem_path
from .lib import OUT_F32, OUT_I8, WLAYOUT_S2_PAIRS, B2YError, call, ptr, stream_ptr


def _pairs(t):
    """[B,H,W,C] int8 tensor seen as pixel pairs [B,H,W/2,2C] (same memory)"""
    return t.buf.view(t.buf.shape[0], t.H, t.W // 2, 2 * t.C)


def _s(t):
    return float(t.reshape(-1)[0])


class QPlan:
    def __init__(self, model, x_shape, device):
        self.model, self.device = model, device
        self.B, self.Cin, self.H, self.W = x_shape
        self.steps = []
        self.prepared = False
        self.runs = 0
        self.graph = None
        self._scal = {}
        self._fusable = {}
        self._build()

    def _build(self):
        model, B, dev = self.model, self.B, self.device
        defs, mods = model.module_defs, model.module_list
        n = len(defs)
        shapes = infer_shapes(model, (self.Cin, self.H, self.W),
                              ('convolutional', 'shortcut', 'route', 'upsample', 'yolo'),
                              "layer type '%s' in the int8 graph (the reference cannot PTQ-calibrate maxpool cfgs either, "
                              "models.py:537-539)")
        tens = [None] * n
        self.yolo = []
        row_off = 0
        # layers whose output is read by somebody other than the next layer (route sources, shortcut 'from' addends)
        readers = set()
        for j, dj in enumerate(defs):
            if dj['type'] == 'route':
                readers.update(sources(j, dj['layers']))
            elif dj['type'] == 'shortcut':
                readers.update(sources(j, dj['from']))
        for i, (d, m) in enumerate(zip(defs, mods)):
            t = d['type']
            Cc, H, W = shapes[i]
            if t == 'convolutional':
                conv = m[0]
                head = i + 1 < n and defs[i + 1]['type'] == 'yolo'
                out = _Tensor(Cc, H, W, torch.float32 if head else torch.int8)
                pitch = 256 if head else Cc
                out.buf = torch.empty((B, H, W, pitch), dtype=out.dtype, device=dev)
                if not head and Cc % 16 != 0:
                    raise NotImplementedError("layer %d: int8 graph needs channel counts that are multiples of 16 "
                                              "(got %d)" % (i, Cc))
                if i == 0:
                    self.stem_fused = stem_path(self.Cin, conv.kernel_size[0], Cc) == 'fused'
                self.steps.append(('conv', i, None if i == 0 else tens[i - 1], out, conv, head))
                tens[i] = out
            elif t == 'shortcut':
                if m.__class__.__name__ not in ('COSPTQuantizedShortcut_min', 'COSPTQuantizedShortcut_max'):
                    raise RuntimeError("quantized=3 needs shortcut_way 1 or 2 (the reference silently drops the "
                                       "residual adds otherwise, models.py:275-305)")
                if len(d['from']) != 1 or getattr(m, 'weight', False):
                    raise NotImplementedError("weighted / multi-source quantised shortcut")
                src = tens[sources(i, d['from'])[0]]
                out = _Tensor(Cc, H, W, torch.int8)
                out.buf = torch.empty((B, H, W, Cc), dtype=torch.int8, device=dev)
                prev_step = self.steps[-1] if self.steps else None
                fuse = (os.environ.get('B2Y_Q_FUSE_SHORTCUT', '1') != '0' and prev_step is not None
                        and prev_step[0] == 'conv' and prev_step[1] == i - 1 and prev_step[2] is not None
                        and not prev_step[5] and (i - 1) not in readers and src is not tens[i - 1])
                if fuse:
                    # the conv writes the shortcut's result; its own output tensor is never materialised
                    self.steps[-1] = ('conv_sc', i - 1, prev_step[2], out, prev_step[4], (i, src, m, tens[i - 1]))
                    tens[i - 1].buf = None
                else:
                    self.steps.append(('shortcut', i, tens[i - 1], src, out, m))
                tens[i] = out
            elif t == 'route':
                srcs = sources(i, d['layers'])
                if 'groups' in d:
                    raise NotImplementedError("grouped route in the int8 graph")
                if len(srcs) == 1:
                    tens[i] = tens[srcs[0]]
                else:
                    out = _Tensor(Cc, H, W, torch.int8)
                    out.buf = torch.empty((B, H, W, Cc), dtype=torch.int8, device=dev)
                    self.steps.append(('concat', i, [tens[s] for s in srcs], out, m))
                    tens[i] = out
            elif t == 'upsample':
                out = _Tensor(Cc, H, W, torch.int8)
                out.buf = torch.empty((B, H, W, Cc), dtype=torch.int8, device=dev)
                self.steps.append(('upsample', i, tens[i - 1], out, d['stride']))
                tens[i] = out
            elif t == 'yolo':
                raw = tens[i - 1]
                rows = m.na * raw.H * raw.W
                self.yolo.append((m, raw, row_off, rows))
                row_off += rows
        self.total_rows = row_off
        self.anchors_px = [m.anchors.to(dev).float().contiguous() for (m, _, _, _) in self.yolo]

    def _pack_qconv(self, src, conv, s_w):
        """int8 weight codes [O][kh][kw][I] + bias, in the pixel-pair forms for the two narrow (Cin = 32) 3x3 layers:
        's1' = ops.s1_pair_weights (the tensors viewed as [B,H,W/2,2C], doubled output channels), 's2' =
        B2Y_WLAYOUT_S2_PAIRS.  q_weight holds code * s_w exactly, so the codes are recovered without rounding."""
        k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
        bias = conv.q_bias.detach().float().contiguous()
        qw = conv.q_weight.detach().float()
        O, I = conv.out_channels, conv.in_channels
        lo, hi = -(1 << (conv.w_bits - 1)), (1 << (conv.w_bits - 1)) - 1
        pair_ok = os.environ.get('B2Y_PAIRPACK', '1') != '0' and k == 3 and p == 1 and I == 32 and src.W % 2 == 0
        if pair_ok and s == 1 and O <= 128 and O % 8 == 0:
            w2 = ops.s1_pair_weights(qw)
            return ops.pack_qconv_weights(w2, s_w, conv.w_bits), torch.cat([bias, bias]).contiguous(), 's1'
        if pair_ok and s == 2:
            codes = (ops.s2_pair_weights(qw) / s_w).round().clamp(lo, hi).to(torch.int8).contiguous()
            return codes, bias, 's2'
        return ops.pack_qconv_weights(qw, s_w, conv.w_bits), bias, None

    def prepare(self):
        """fold BN + quantise weights (reference first-call behaviour), pack int8 weights, resolve tensor scales."""
        scale_of = {}
        self.packed = {}
        for st in self.steps:
            kind = st[0]
            if kind == 'conv':
                _, i, src, out, conv, head = st
                conv.fold_and_quantize()
                s_w, s_a = _s(conv.weight_quantizer.scale), _s(conv.activation_quantizer.scale)
                if s_w <= 0 or s_a <= 0:
                    raise RuntimeError("layer %d is not calibrated (scale == 0): load a calibrated state_dict" % i)
                bits_w, bits_a = conv.w_bits, conv.a_bits
                if bits_w > 8 or bits_a > 8:
                    raise NotImplementedError("the int8 wgmma path covers <= 8 bit weights and activations")
                act = conv.activate
                slope = 0.25 if conv.maxabsscaler else 0.1
                if src is None:
                    self.packed[i] = (conv.q_weight.detach().float().contiguous(), conv.q_bias.detach().float(), s_a,
                                      act, slope, bits_a)
                else:
                    w8, bq, mode = self._pack_qconv(src, conv, s_w)
                    self.packed[i] = (w8, bq, scale_of[id(src)] * s_w, s_a, act, slope, bits_a, mode)
                scale_of[id(out)] = s_a
            elif kind == 'conv_sc':
                _, i, src, out, conv, (isc, a, m, own) = st
                conv.fold_and_quantize()
                s_w, s_a = _s(conv.weight_quantizer.scale), _s(conv.activation_quantizer.scale)
                if s_w <= 0 or s_a <= 0:
                    raise RuntimeError("layer %d is not calibrated (scale == 0): load a calibrated state_dict" % i)
                if conv.w_bits > 8 or conv.a_bits > 8:
                    raise NotImplementedError("the int8 wgmma path covers <= 8 bit weights and activations")
                w8, bq, mode = self._pack_qconv(src, conv, s_w)
                self.packed[i] = (w8, bq, scale_of[id(src)] * s_w, s_a, conv.activate,
                                  0.25 if conv.maxabsscaler else 0.1, conv.a_bits, mode)
                scale_of[id(own)] = s_a
                scale_of[id(out)] = _s(m.scale_sum)
            elif kind == 'shortcut':
                _, i, x, a, out, m = st
                scale_of[id(out)] = _s(m.scale_sum)
            elif kind == 'concat':
                scale_of[id(st[3])] = _s(st[4].scale)
            elif kind == 'upsample':
                scale_of[id(st[3])] = scale_of[id(st[2])]
        self.scale_of = scale_of
        self.stem_w = {}
        self.prepared = True

    def forward(self, x):
        """Eval forward of the INT8 graph; after one eager call the static launch sequence replays from a CUDA graph
        (the quantiser state is frozen in eval; call plan.invalidate() after re-calibrating)."""
        if not self.prepared:
            self.prepare()
        x = x.contiguous().float()
        use_graph = getattr(self.model, 'use_cuda_graph', os.environ.get('B2Y_NO_GRAPH', '0') != '1')
        if not use_graph or self.runs < 1:
            self.runs += 1
            return self._forward_eager(x)
        if self.graph is None:
            self.static_x = x.clone()
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self.static_out = self._forward_eager(self.static_x)
            self.graph = g
        self.static_x.copy_(x)
        self.graph.replay()
        io, p, feats = self.static_out
        if getattr(self.model, 'static_outputs', False):
            return io, p, feats
        return io.clone(), tuple(t.clone() for t in p), feats

    def _sv(self, t):
        """python float of a scale buffer, read once (a host sync is illegal while the forward is being captured)"""
        v = self._scal.get(id(t))
        if v is None:
            v = self._scal[id(t)] = _s(t)
        return v

    def invalidate(self):
        self.graph = None
        self._scal = {}
        self.prepared = False
        self.runs = 0

    def _forward_eager(self, x):
        B = self.B
        sc = self.scale_of
        for st in self.steps:
            kind = st[0]
            if kind == 'conv':
                _, i, src, out, conv, head = st
                k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
                if src is None:
                    wq, bq, s_a, act, slope, bits = self.packed[i]
                    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
                    d = ops.make_conv_desc((B, self.H, self.W, self.Cin), self.Cin, conv.out_channels, k, s, p,
                                           ops._pitch(out.view()), act, slope, OUT_I8)
                    ws = self.stem_w.get(i)
                    if ws is None:
                        # fused tensor-core stem when the fake-quantised weights (int8 code x 2^-n) are exact in fp16
                        fits = self.stem_fused and float(wq.abs().max()) < 6.0e4
                        ws = self.stem_w[i] = ops.pack_stem_weights(wq) if fits else False
                    if ws is not False:
                        call("b2y_stem_conv_fwd_fused_q", C.byref(d), ptr(x), 0, 1.0, ptr(ws), ptr(bq), ptr(out.buf), s_a,
                             float(lo), float(hi), stream_ptr())
                    else:
                        call("b2y_stem_conv_fwd_q", C.byref(d), ptr(x), ptr(wq), ptr(bq), ptr(out.buf), s_a, float(lo),
                             float(hi), stream_ptr())
                else:
                    w8, bq, acc_scale, s_a, act, slope, bits, mode = self.packed[i]
                    if head:
                        ops.qconv2d(src.view(), w8, bq, k, s, p, acc_scale, s_a, act=act, slope=slope, bits=bits,
                                    out=out.buf[..., :conv.out_channels], out_kind=OUT_F32, requant=True)
                    elif mode == 's1':
                        ops.qconv2d(_pairs(src), w8, bq, k, s, p, acc_scale, s_a, act=act, slope=slope, bits=bits,
                                    out=_pairs(out), out_kind=OUT_I8)
                    else:
                        ops.qconv2d(src.view(), w8, bq, k, s, p, acc_scale, s_a, act=act, slope=slope, bits=bits,
                                    out=out.view(), out_kind=OUT_I8, w_layout=WLAYOUT_S2_PAIRS if mode == 's2' else 0)
            elif kind == 'conv_sc':
                _, i, src, out, conv, (isc, at, m, own) = st
                k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
                w8, bq, acc_scale, s_a, act, slope, bits, mode = self.packed[i]
                slo, shi = -(1 << (m.bits - 1)), (1 << (m.bits - 1)) - 1
                if mode == 's1':
                    xv, av, ov = _pairs(src), _pairs(at), _pairs(out)
                else:
                    xv, av, ov = src.view(), at.view(), out.view()
                fused = self._fusable.get(i, True)
                if fused:
                    cd = ops.make_conv_desc(xv.shape, ops._pitch(xv), w8.shape[0], k, s, p, ops._pitch(ov), act,
                                            slope, OUT_I8, 0, WLAYOUT_S2_PAIRS if mode == 's2' else 0)
                    qd = ops.QConvDesc(cd, float(acc_scale), float(s_a), float(-(1 << (bits - 1))),
                                       float((1 << (bits - 1)) - 1), OUT_I8, 1)
                    try:
                        call("b2y_qconv2d_shortcut_fwd", C.byref(qd), ptr(xv), ptr(w8), ptr(bq), ptr(av), ops._pitch(av),
                             sc[id(at)], self._sv(m.scale_x), self._sv(m.scale_a), self._sv(m.scale_sum), float(slo),
                             float(shi), ptr(ov), stream_ptr())
                    except B2YError as e:
                        if 'unsupported' not in str(e).lower():
                            raise
                        fused = self._fusable[i] = False       # e.g. a scale that is not a power of two
                if not fused:
                    if own.buf is None:
                        own.buf = torch.empty((B, own.H, own.W, own.C), dtype=torch.int8, device=self.device)
                    ops.qconv2d(xv, w8, bq, k, s, p, acc_scale, s_a, act=act, slope=slope, bits=bits,
                                out=_pairs(own) if mode == 's1' else own.view(), out_kind=OUT_I8,
                                w_layout=WLAYOUT_S2_PAIRS if mode == 's2' else 0)
                    wv = _pairs(own) if mode == 's1' else own.view()
                    call("b2y_qshortcut_i8", ptr(wv), ops._pitch(wv), ptr(av), ops._pitch(av), ptr(ov), ops._pitch(ov),
                         wv.shape[0] * wv.shape[1] * wv.shape[2], wv.shape[3], s_a, self._sv(m.scale_x), sc[id(at)],
                         self._sv(m.scale_a),
                         self._sv(m.scale_sum), float(slo), float(shi), stream_ptr())
            elif kind == 'shortcut':
                _, i, xt, at, out, m = st
                lo, hi = -(1 << (m.bits - 1)), (1 << (m.bits - 1)) - 1
                xv, av, ov = xt.view(), at.view(), out.view()
                call("b2y_qshortcut_i8", ptr(xv), ops._pitch(xv), ptr(av), ops._pitch(av), ptr(ov), ops._pitch(ov),
                     B * out.H * out.W, out.C, sc[id(xt)], self._sv(m.scale_x), sc[id(at)], self._sv(m.scale_a), self._sv(m.scale_sum),
                     float(lo), float(hi), stream_ptr())
            elif kind == 'concat':
                _, i, srcs, out, m = st
                lo, hi = -(1 << (m.bits - 1)), (1 << (m.bits - 1)) - 1
                off = 0
                for t in srcs:
                    tv = t.view()
                    ov = out.buf[..., off:off + t.C]
                    call("b2y_requant_i8", ptr(tv), ops._pitch(tv), ptr(ov), ops._pitch(ov), B * t.H * t.W, t.C,
                         sc[id(t)], self._sv(m.scale), float(lo), float(hi), stream_ptr())
                    off += t.C
            elif kind == 'upsample':
                _, i, src, out, s = st
                sv, ov = src.view(), out.view()
                call("b2y_upsample_nearest_i8", ptr(sv), ops._pitch(sv), ptr(ov), ops._pitch(ov), B, src.H, src.W,
                     src.C, int(s), stream_ptr())
        no = self.yolo[0][0].no
        io = torch.empty((B, self.total_rows, no), dtype=torch.float32, device=self.device)
        p_out = []
        for (m, raw, row_off, rows), anc in zip(self.yolo, self.anchors_px):
            _, p = ops.yolo_decode(raw.buf, m.na, m.no, anc, m.stride, io=io, row_offset=row_off)
            m.nx, m.ny = raw.W, raw.H
            p_out.append(p)
        return io, tuple(p_out), []
