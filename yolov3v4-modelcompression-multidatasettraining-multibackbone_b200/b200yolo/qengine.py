"""INT8 graph executor for a PTQ-calibrated Darknet (quantized=3, reference PTQ.py:92-102 eval path) and for the eval
forward of a google-QAT Darknet (quantized=1) that int8_graph_refusal accepts.

The reference *simulates* int8 in fp32: every tensor is a float on a power-of-two grid, convs are F.conv2d on those
floats (utils/quantized/quantized_ptq_cos.py:288-296).  Because all scales are powers of two the products are exact
integers times a power of two, so the same arithmetic runs here on the real int8 codes:

   conv      int8 x int8 -> int32 on int8 wgmma, epilogue  acc*(s_in*s_w) + q_bias -> act -> requant(s_act)
   shortcut  folded into the epilogue of the conv that feeds it (b2y_qconv2d_shortcut_fwd) when nothing else reads that
             conv's output; otherwise b2y_qshortcut_i8 (both addends rounded onto scale_x / scale_a, sum requantised)
   concat    b2y_requant_i8 of every source onto the concat scale, written into its channel slot
   upsample  nearest copy of codes
   maxpool   max of codes (quantized=1 only: the QAT graph keeps a plain nn.MaxPool2d over values on one grid)
   layer 0   fp32 direct conv of the float image on the fake-quantised weights (as the reference), int8 out
   heads     fp32 fake-quant values for the (fp32) YOLO decode kernel

quantized=1 (utils/quantized/quantized_google.py) holds the same arithmetic with other names: the conv is
act(conv(x, fq(W_fold)) + fq(b_fold)) -> fq(s_act) with the running-statistics fold of BN_fuse, every quantiser symmetric
with the same round-half-away rule and signed clamp as the COSPTQ ones; QuantizedShortcut_min rounds its addends onto
input_scale unclamped (the COSPTQ shortcut with scale_x = scale_a = input_scale), QuantizedShortcut_max clamps them onto
its one scale (the clamp_addends mode of b2y_qconv2d_shortcut_fwd, or b2y_requant_i8 of both addends); concats
requantise onto QuantizedFeatureConcat.scale.
"""
import ctypes as C
import os

import torch

from . import ops
from .layout import _Tensor, infer_shapes, sources, stem_path
from .lib import OUT_F32, OUT_I8, WLAYOUT_S2_PAIRS, B2YError, call, ptr, stream_ptr

_GOOGLE_SHORTCUTS = ('QuantizedShortcut_min', 'QuantizedShortcut_max')
_Q1_LAYERS = ('convolutional', 'shortcut', 'route', 'upsample', 'maxpool', 'yolo')


def int8_graph_refusal(model):
    """The one rule that decides whether the eval forward of a google-QAT (quantized=1) model runs as the INT8 graph:
    None when it does, else why it keeps running on qat.QatRunner.  It reads only the model's structure, which its state
    never changes, so it is decided once, when the plan would be built."""
    if model.a_bit > 8 or model.w_bit > 8:
        # codes of more than 8 bits are not int8 wgmma operands
        return "a_bit %d / w_bit %d: the int8 graph holds codes of at most 8 bits" % (model.a_bit, model.w_bit)
    defs, mods = model.module_defs, model.module_list
    n = len(defs)
    if not n or defs[0]['type'] != 'convolutional':
        return "the int8 graph starts with the fp32 stem convolution of the image"
    late_readers = {}          # layer -> the layers after it that read it through a route or a shortcut
    for j, dj in enumerate(defs):
        for s in sources(j, dj.get('layers', []) if dj['type'] == 'route' else dj.get('from', [])
                         if dj['type'] == 'shortcut' else []):
            late_readers.setdefault(s, []).append(j)
    for i, (d, m) in enumerate(zip(defs, mods)):
        t = d['type']
        if t not in _Q1_LAYERS:
            # [depthwise] / [se] stay float under google QAT (models.py _conv_block), and the other types have no int8
            # kernel: there is no integer network to run
            return "layer %d: '%s' has no int8 form in the QAT graph" % (i, t)
        if t == 'convolutional':
            conv = m[0]
            head = i + 1 < n and defs[i + 1]['type'] == 'yolo'
            if conv.groups != 1:
                return "layer %d: grouped convolution (stays on the QAT module forwards)" % i
            if any(q.__class__.__name__ != 'SymmetricQuantizer' for q in
                   (conv.weight_quantizer, conv.bias_quantizer, conv.activation_quantizer)):
                # the int8 kernels hold codes without a zero point
                return "layer %d: asymmetric quantisers (q_type 1)" % i
            if i > 0 and conv.kernel_size[0] not in (1, 3):
                # the int8 implicit-GEMM conv covers the 1x1 and 3x3 taps of the Darknet cfgs
                return "layer %d: %dx%d convolution" % (i, conv.kernel_size[0], conv.kernel_size[1])
            if not head and conv.out_channels % 16:
                # int8 activations are whole 16-byte channel vectors (the same condition as for quantized=3)
                return "layer %d: %d channels, not a multiple of 16" % (i, conv.out_channels)
            if head and late_readers.get(i):
                # a head's output is fp32 fake-quant values for the decode, not int8 codes another layer could read
                return "layer %d: a YOLO head's output is read by layer %d" % (i, late_readers[i][0])
        elif t == 'shortcut':
            if m.__class__.__name__ not in _GOOGLE_SHORTCUTS:
                # shortcut_way other than 1 / 2: the reference leaves an empty Sequential and drops the add, and
                # QatRunner replays exactly that
                return "layer %d: shortcut_way not in (1, 2), the residual add is dropped" % i
            if len(d['from']) != 1 or getattr(m, 'weight', False):
                return "layer %d: weighted or multi-source shortcut" % i
            src = sources(i, d['from'])[0]
            if defs[src]['type'] == 'yolo' or defs[i - 1]['type'] == 'yolo':
                return "layer %d: shortcut next to a YOLO layer" % i
        elif t == 'route':
            srcs = sources(i, d['layers'])
            if 'groups' in d:
                # no QAT fixture covers the grouped routes of yolov4-tiny
                return "layer %d: grouped route" % i
            if len(srcs) > 1:
                for s in srcs:
                    later = [j for j in late_readers.get(s, []) if j > i]
                    if later:
                        # QuantizedFeatureConcat overwrites its sources' stored outputs with their requantised values,
                        # which a later reader of the source would see
                        return "layer %d: concat source %d is read again by layer %d" % (i, s, later[0])
    shapes = infer_shapes(model, (3, 416, 416), _Q1_LAYERS)
    for i, d in enumerate(defs):
        if d['type'] == 'shortcut' and shapes[sources(i, d['from'])[0]][0] != shapes[i - 1][0]:
            # b2y_qshortcut_i8 adds tensors of one width
            return "layer %d: shortcut over addends of different widths" % i
    return None


def _pairs(t):
    """[B,H,W,C] int8 tensor seen as pixel pairs [B,H,W/2,2C] (same memory)"""
    return t.buf.view(t.buf.shape[0], t.H, t.W // 2, 2 * t.C)


def _s(t):
    return float(t.reshape(-1)[0])


def _stem_fp16_exact(w, b):
    """True when the fused fp16 stem holds the first layer's weights and bias exactly: every weight is one fp16, the bias
    the sum of its fp16 rounding and the fp16 rounding of the rest (csrc/stem_tc.cu)"""
    hi = b.half().float()
    return torch.equal(w.half().float(), w) and torch.equal(hi + (b - hi).half().float(), b)


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
        self._scratch = {}
        # quantized=1: the QAT state the plan was packed from (see _state_fingerprint); Engine.weights_changed() clears it
        self.q1 = model.quantized == 1
        self.param_version = None
        self._build()

    def _build(self):
        model, B, dev = self.model, self.B, self.device
        defs, mods = model.module_defs, model.module_list
        n = len(defs)
        shapes = infer_shapes(model, (self.Cin, self.H, self.W),
                              _Q1_LAYERS if self.q1 else ('convolutional', 'shortcut', 'route', 'upsample', 'yolo'),
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
                src = None if i == 0 else tens[i - 1]
                if self.q1 and src is not None and src.Cp % 32:
                    # the int8 conv reads whole 32-byte K chunks: a 16-channel input (yolov3-tiny) is stored in a
                    # zero-filled buffer of 32 channels, which its producer writes through view(), and the packed
                    # weights get zero columns there (_pack_qconv)
                    src.Cp = (src.Cp + 31) // 32 * 32
                    src.buf = torch.zeros((B, src.H, src.W, src.Cp), dtype=torch.int8, device=dev)
                self.steps.append(('conv', i, None if i == 0 else tens[i - 1], out, conv, head))
                tens[i] = out
            elif t == 'shortcut':
                kinds = _GOOGLE_SHORTCUTS if self.q1 else ('COSPTQuantizedShortcut_min', 'COSPTQuantizedShortcut_max')
                if m.__class__.__name__ not in kinds:
                    raise RuntimeError("quantized=%d needs shortcut_way 1 or 2 (the reference silently drops the "
                                       "residual adds otherwise, models.py:275-305)" % model.quantized)
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
            elif t == 'maxpool':
                out = _Tensor(Cc, H, W, torch.int8)
                out.buf = torch.empty((B, H, W, Cc), dtype=torch.int8, device=dev)
                k, s = d['size'], d['stride']
                self.steps.append(('maxpool', i, tens[i - 1], out, k, s, k == 2 and s == 1))
                tens[i] = out
            elif t == 'yolo':
                raw = tens[i - 1]
                rows = m.na * raw.H * raw.W
                self.yolo.append((m, raw, row_off, rows))
                row_off += rows
        self.total_rows = row_off
        self.anchors_px = [m.anchors.to(dev).float().contiguous() for (m, _, _, _) in self.yolo]

    def _pack_qconv(self, src, conv, qw, bias, s_w):
        """int8 weight codes [O][kh][kw][I] + bias, in the pixel-pair forms for the two narrow (Cin = 32) 3x3 layers:
        's1' = ops.s1_pair_weights (the tensors viewed as [B,H,W/2,2C], doubled output channels), 's2' =
        B2Y_WLAYOUT_S2_PAIRS.  q_weight holds code * s_w exactly, so the codes are recovered without rounding."""
        k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
        O, I = conv.out_channels, conv.in_channels
        lo, hi = -(1 << (conv.w_bits - 1)), (1 << (conv.w_bits - 1)) - 1
        pair_ok = os.environ.get('B2Y_PAIRPACK', '1') != '0' and k == 3 and p == 1 and I == 32 and src.W % 2 == 0
        if pair_ok and s == 1 and O <= 128 and O % 8 == 0:
            w2 = ops.s1_pair_weights(qw)
            return ops.pack_qconv_weights(w2, s_w, conv.w_bits), torch.cat([bias, bias]).contiguous(), 's1'
        if pair_ok and s == 2:
            codes = (ops.s2_pair_weights(qw) / s_w).round().clamp(lo, hi).to(torch.int8).contiguous()
            return codes, bias, 's2'
        if src.Cp != I:
            qw = torch.nn.functional.pad(qw, (0, 0, 0, 0, 0, src.Cp - I))
        return ops.pack_qconv_weights(qw, s_w, conv.w_bits), bias, None

    def _quantised_conv(self, i, conv):
        """(fake-quantised folded weights, fake-quantised bias, s_w, s_a) of conv layer i.  quantized=3: the reference's
        first-call fold (fold_and_quantize); quantized=1: the eval branch of BNFold_QuantizedConv2d_For_FPGA.forward
        (BN_fuse with the running statistics, then the weight and bias quantisers), on the same kernels as QatRunner."""
        if self.q1:
            s_w, s_b, s_a = (_s(q.scale) for q in (conv.weight_quantizer, conv.bias_quantizer, conv.activation_quantizer))
        else:
            conv.fold_and_quantize()
            s_w, s_b, s_a = _s(conv.weight_quantizer.scale), 1.0, _s(conv.activation_quantizer.scale)
        if s_w <= 0 or s_b <= 0 or s_a <= 0:
            raise RuntimeError("layer %d is not calibrated (scale == 0): load a calibrated state_dict" % i)
        if conv.w_bits > 8 or conv.a_bits > 8:
            raise NotImplementedError("the int8 wgmma path covers <= 8 bit weights and activations")
        if self.q1:
            from .qat import fake_quant
            with torch.no_grad():
                w, b = conv.BN_fuse()
                qw, qb = fake_quant(w, s_w, conv.w_bits), fake_quant(b, s_b, conv.w_bits)
        else:
            qw, qb = conv.q_weight, conv.q_bias
        return qw.detach().float().contiguous(), qb.detach().float().contiguous(), s_w, s_a

    def _shortcut_scales(self, m):
        """(scale_x, scale_a, scale_sum, clamp_addends) of a quantised shortcut (module eval forwards)"""
        name = m.__class__.__name__
        if name == 'QuantizedShortcut_min':
            v = (_s(m.input_scale), _s(m.input_scale), _s(m.scale), 0)
        elif name == 'QuantizedShortcut_max':
            v = (_s(m.scale), _s(m.scale), _s(m.scale), 1)
        else:
            v = (_s(m.scale_x), _s(m.scale_a), _s(m.scale_sum), 0)
        if self.q1 and min(v[:3]) <= 0:
            raise RuntimeError("shortcut %s is not calibrated (scale == 0): load a calibrated state_dict" % m.name)
        return v

    def prepare(self):
        """fold BN + quantise weights (reference first-call behaviour), pack int8 weights, resolve tensor scales."""
        scale_of = {}
        self.packed = {}
        self.sc_scales = {}
        self.q_steps = []
        for st in self.steps:
            kind = st[0]
            if kind in ('conv', 'conv_sc'):
                i, src, out, conv = st[1], st[2], st[3], st[4]
                qw, qb, s_w, s_a = self._quantised_conv(i, conv)
                act, slope, bits_a = conv.activate, 0.25 if conv.maxabsscaler else 0.1, conv.a_bits
                if src is None:
                    self.packed[i] = (qw, qb, s_a, act, slope, bits_a)
                else:
                    w8, bq, mode = self._pack_qconv(src, conv, qw, qb, s_w)
                    self.packed[i] = (w8, bq, scale_of[id(src)] * s_w, s_a, act, slope, bits_a, mode)
                if self.q1:
                    # the quantisers count their forwards in eval too (quantized_google.py Quantizer.forward)
                    self.q_steps += [conv.weight_quantizer.step, conv.bias_quantizer.step,
                                     conv.activation_quantizer.step]
                if kind == 'conv':
                    scale_of[id(out)] = s_a
                else:
                    isc, m, own = st[5][0], st[5][2], st[5][3]
                    self.sc_scales[isc] = self._shortcut_scales(m)
                    scale_of[id(own)] = s_a
                    scale_of[id(out)] = self.sc_scales[isc][2]
            elif kind == 'shortcut':
                self.sc_scales[st[1]] = self._shortcut_scales(st[5])
                scale_of[id(st[4])] = self.sc_scales[st[1]][2]
            elif kind == 'concat':
                scale_of[id(st[3])] = _s(st[4].scale)
            elif kind in ('upsample', 'maxpool'):
                scale_of[id(st[3])] = scale_of[id(st[2])]
        self.scale_of = scale_of
        self.stem_w = {}
        self.prepared = True

    def _state_fingerprint(self):
        """(tensors, fingerprint) of the quantized=1 state the plan packs: every parameter and buffer of the model except
        the quantisers' forward counters, which the eval forward advances itself.  QAT training moves parameters and
        running statistics in place (a version bump) and re-assigns the quantisers' scale tensors (a new tensor): the
        plan holds the tensors it fingerprinted, so a new tensor can never reuse an id and data pointer of the old."""
        held = list(self.model.parameters()) + [b for name, b in self.model.named_buffers()
                                                if not name.endswith('quantizer.step')]
        fp = tuple((id(t), t._version, t.data_ptr()) for t in held) + (getattr(self.model, '_b2y_epoch', 0),)
        return held, fp

    def forward(self, x):
        """Eval forward of the INT8 graph; after one eager call the static launch sequence replays from a CUDA graph
        (the quantiser state is frozen in eval; call plan.invalidate() after re-calibrating)."""
        if self.q1:
            held, fp = self._state_fingerprint()
            if fp != self.param_version:
                # trained since the plan was packed: re-fold, re-pack and re-capture
                self.invalidate()
                self._held, self.param_version = held, fp
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

    def _qshortcut(self, i, m, xv, sx_in, av, sa_in, ov, c):
        """shortcut layer i (module m) over c channels of the int8 addends xv (scale sx_in) and av (scale sa_in) into ov"""
        scale_x, scale_a, scale_sum, clamp = self.sc_scales[i]
        lo, hi = -(1 << (m.bits - 1)), (1 << (m.bits - 1)) - 1
        pixels = xv.shape[0] * xv.shape[1] * xv.shape[2]
        if clamp:
            # the addends are clamped onto their grid too: requantise them first, then the shortcut's roundings are
            # identities
            tmp = self._scratch.get(i)
            if tmp is None:
                tmp = self._scratch[i] = torch.empty((2,) + tuple(xv.shape[:3]) + (c,), dtype=torch.int8,
                                                     device=self.device)
            for t, s_in, s_out, q in ((xv, sx_in, scale_x, tmp[0]), (av, sa_in, scale_a, tmp[1])):
                call("b2y_requant_i8", ptr(t), ops._pitch(t), ptr(q), ops._pitch(q), pixels, c, s_in, s_out, float(lo),
                     float(hi), stream_ptr())
            xv, sx_in, av, sa_in = tmp[0], scale_x, tmp[1], scale_a
        call("b2y_qshortcut_i8", ptr(xv), ops._pitch(xv), ptr(av), ops._pitch(av), ptr(ov), ops._pitch(ov), pixels, c,
             sx_in, scale_x, sa_in, scale_a, scale_sum, float(lo), float(hi), stream_ptr())

    def _forward_eager(self, x):
        B = self.B
        sc = self.scale_of
        if self.q_steps:
            torch._foreach_add_(self.q_steps, 1)
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
                        # and the bias in the two fp16 terms it is split into; codes x 2^-n below fp16's subnormal
                        # grid (tiny weight scales) would be rounded
                        fits = self.stem_fused and _stem_fp16_exact(wq, bq)
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
                scale_x, scale_a, scale_sum, clamp = self.sc_scales[isc]
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
                                       float((1 << (bits - 1)) - 1), OUT_I8, 1, clamp)
                    try:
                        call("b2y_qconv2d_shortcut_fwd", C.byref(qd), ptr(xv), ptr(w8), ptr(bq), ptr(av), ops._pitch(av),
                             sc[id(at)], scale_x, scale_a, scale_sum, float(slo), float(shi), ptr(ov), stream_ptr())
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
                    self._qshortcut(isc, m, wv, s_a, av, sc[id(at)], ov, wv.shape[3])
            elif kind == 'shortcut':
                _, i, xt, at, out, m = st
                self._qshortcut(i, m, xt.view(), sc[id(xt)], at.view(), sc[id(at)], out.view(), out.C)
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
            elif kind == 'maxpool':
                _, i, src, out, k, s, tiny = st
                sv, ov = src.view(), out.view()
                call("b2y_maxpool_i8", ptr(sv), ops._pitch(sv), ptr(ov), ops._pitch(ov), B, src.H, src.W, src.C, int(k),
                     int(s), 1 if tiny else 0, stream_ptr())
        no = self.yolo[0][0].no
        io = torch.empty((B, self.total_rows, no), dtype=torch.float32, device=self.device)
        p_out = []
        for (m, raw, row_off, rows), anc in zip(self.yolo, self.anchors_px):
            _, p = ops.yolo_decode(raw.buf, m.na, m.no, anc, m.stride, io=io, row_offset=row_off)
            m.nx, m.ny = raw.W, raw.H
            p_out.append(p)
        return io, tuple(p_out), []
