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
import collections
import ctypes as C
import os

import torch

from . import ops
from .engine import MaxpoolStep, UpsampleStep
from .layout import _Tensor, infer_shapes, pair_form, sources, stem_path
from .lib import OUT_F32, OUT_I8, WLAYOUT_S2_PAIRS, B2YError, call, ptr, stream_ptr

_GOOGLE_SHORTCUTS = ('QuantizedShortcut_min', 'QuantizedShortcut_max')
_Q1_LAYERS = ('convolutional', 'shortcut', 'route', 'upsample', 'maxpool', 'yolo')

# ---- launch list vocabulary: field 0 is the step's kind; src / out / x / addend / own are layout._Tensor; upsample and
# max-pool steps are engine.UpsampleStep / engine.MaxpoolStep
# conv: src is None for the stem (it reads the image); a head writes fp32 fake-quant values for the decode; form is the
# pixel-pair form (layout.pair_form: 's1', 's2' or None); shortcut is a FusedShortcut or None
QConvStep = collections.namedtuple('QConvStep', 'kind i src out conv head form shortcut')
# shortcut layer i (module) folded into the epilogue of the conv before it, which then writes the shortcut's tensor: own
# is the conv's own output, materialised only when the fused launch is refused
FusedShortcut = collections.namedtuple('FusedShortcut', 'i addend module own')
# out = x + addend, both rounded onto the shortcut's scales
QShortcutStep = collections.namedtuple('QShortcutStep', 'kind i x addend out module')
# every source requantised onto the concat's scale, into its channel slot of out
QConcatStep = collections.namedtuple('QConcatStep', 'kind i srcs out module')

# packed weights of a body conv: int8 codes in the step's form, bias, acc_scale = s_in * s_w, s_a the output scale
QConvPack = collections.namedtuple('QConvPack', 'w8 bias acc_scale s_a act slope bits')
# the fp32 stem: fake-quantised weights and bias (the fused fp16 copy of the weights is made at the first launch)
QStemPack = collections.namedtuple('QStemPack', 'w bias s_a act slope bits')
ShortcutScales = collections.namedtuple('ShortcutScales', 'scale_x scale_a scale_sum clamp_addends')


def _late_readers(defs):
    """layer -> the layers that read it through a route or a shortcut"""
    readers = {}
    for j, dj in enumerate(defs):
        rel = dj.get('layers', []) if dj['type'] == 'route' else dj.get('from', []) if dj['type'] == 'shortcut' else []
        for s in sources(j, rel):
            readers.setdefault(s, []).append(j)
    return readers


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
    late_readers = _late_readers(defs)
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
    def __init__(self, model, x_shape, device, *, pair_forms=True, fuse_shortcuts=True):
        """pair_forms / fuse_shortcuts = False build the plain graph (dense weights everywhere, every shortcut a launch
        of its own), the one the tests compare the pixel-pair forms and the fused shortcut epilogue against."""
        self.model, self.device = model, device
        self.B, self.Cin, self.H, self.W = x_shape
        self.steps = []
        self.prepared = False
        self.runs = 0
        self.graph = None
        self._fusable = {}
        self._scratch = {}
        # quantized=1: the QAT state the plan was packed from (see _state_fingerprint); Engine.weights_changed() clears it
        self.q1 = model.quantized == 1
        self.param_version = None
        self._build(pair_forms, fuse_shortcuts)

    def _build(self, pair_forms, fuse_shortcuts):
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
        readers = _late_readers(defs)

        def codes(C, H, W):
            t = _Tensor(C, H, W, torch.int8)
            t.buf = torch.empty((B, H, W, C), dtype=torch.int8, device=dev)
            return t

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
                form = None
                if pair_forms and src is not None and not head:
                    form = pair_form(conv.kernel_size[0], conv.stride[0], conv.padding[0], conv.in_channels,
                                     conv.out_channels, src.W)
                self.steps.append(QConvStep('conv', i, src, out, conv, head, form, None))
                tens[i] = out
            elif t == 'shortcut':
                kinds = _GOOGLE_SHORTCUTS if self.q1 else ('COSPTQuantizedShortcut_min', 'COSPTQuantizedShortcut_max')
                if m.__class__.__name__ not in kinds:
                    raise RuntimeError("quantized=%d needs shortcut_way 1 or 2 (the reference silently drops the "
                                       "residual adds otherwise, models.py:275-305)" % model.quantized)
                if len(d['from']) != 1 or getattr(m, 'weight', False):
                    raise NotImplementedError("weighted / multi-source quantised shortcut")
                src = tens[sources(i, d['from'])[0]]
                out = codes(Cc, H, W)
                prev = self.steps[-1] if self.steps else None
                if (fuse_shortcuts and prev is not None and prev.kind == 'conv' and prev.i == i - 1
                        and prev.src is not None and not prev.head and (i - 1) not in readers and src is not tens[i - 1]):
                    # the conv writes the shortcut's result; its own output tensor is never materialised
                    self.steps[-1] = prev._replace(out=out, shortcut=FusedShortcut(i, src, m, tens[i - 1]))
                    tens[i - 1].buf = None
                else:
                    self.steps.append(QShortcutStep('shortcut', i, tens[i - 1], src, out, m))
                tens[i] = out
            elif t == 'route':
                srcs = sources(i, d['layers'])
                if 'groups' in d:
                    raise NotImplementedError("grouped route in the int8 graph")
                if len(srcs) == 1:
                    tens[i] = tens[srcs[0]]
                else:
                    tens[i] = codes(Cc, H, W)
                    self.steps.append(QConcatStep('concat', i, [tens[s] for s in srcs], tens[i], m))
            elif t == 'upsample':
                tens[i] = codes(Cc, H, W)
                self.steps.append(UpsampleStep('upsample', tens[i - 1], tens[i], d['stride']))
            elif t == 'maxpool':
                tens[i] = codes(Cc, H, W)
                k, s = d['size'], d['stride']
                self.steps.append(MaxpoolStep('maxpool', tens[i - 1], tens[i], k, s, k == 2 and s == 1))
            elif t == 'yolo':
                raw = tens[i - 1]
                rows = m.na * raw.H * raw.W
                self.yolo.append((m, raw, row_off, rows))
                row_off += rows
        self.total_rows = row_off
        self.anchors_px = [m.anchors.to(dev).float().contiguous() for (m, _, _, _) in self.yolo]

    def _pack_qconv(self, st, qw, bias, s_w):
        """(int8 weight codes [O][kh][kw][I], bias) of a body conv step in its form: 's1' = ops.s1_pair_weights (the
        tensors viewed as [B,H,W/2,2C], doubled output channels), 's2' = B2Y_WLAYOUT_S2_PAIRS, None = dense with zero
        columns up to the input's stored width.  q_weight holds code * s_w exactly, so the codes are recovered without
        rounding."""
        conv = st.conv
        if st.form == 's1':
            w2 = ops.s1_pair_weights(qw)
            return ops.pack_qconv_weights(w2, s_w, conv.w_bits), torch.cat([bias, bias]).contiguous()
        if st.form == 's2':
            lo, hi = -(1 << (conv.w_bits - 1)), (1 << (conv.w_bits - 1)) - 1
            return (ops.s2_pair_weights(qw) / s_w).round().clamp(lo, hi).to(torch.int8).contiguous(), bias
        if st.src.Cp != conv.in_channels:
            qw = torch.nn.functional.pad(qw, (0, 0, 0, 0, 0, st.src.Cp - conv.in_channels))
        return ops.pack_qconv_weights(qw, s_w, conv.w_bits), bias

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
        """ShortcutScales of a quantised shortcut (module eval forwards)"""
        name = m.__class__.__name__
        if name == 'QuantizedShortcut_min':
            v = ShortcutScales(_s(m.input_scale), _s(m.input_scale), _s(m.scale), 0)
        elif name == 'QuantizedShortcut_max':
            v = ShortcutScales(_s(m.scale), _s(m.scale), _s(m.scale), 1)
        else:
            v = ShortcutScales(_s(m.scale_x), _s(m.scale_a), _s(m.scale_sum), 0)
        if self.q1 and min(v.scale_x, v.scale_a, v.scale_sum) <= 0:
            raise RuntimeError("shortcut %s is not calibrated (scale == 0): load a calibrated state_dict" % m.name)
        return v

    def prepare(self):
        """fold BN + quantise weights (reference first-call behaviour), pack int8 weights, resolve tensor scales."""
        scale_of = {}
        self.packed = {}
        self.sc_scales = {}
        self.q_steps = []
        for st in self.steps:
            if st.kind == 'conv':
                conv, sc = st.conv, st.shortcut
                qw, qb, s_w, s_a = self._quantised_conv(st.i, conv)
                act, slope, bits_a = conv.activate, 0.25 if conv.maxabsscaler else 0.1, conv.a_bits
                if st.src is None:
                    self.packed[st.i] = QStemPack(qw, qb, s_a, act, slope, bits_a)
                else:
                    w8, bq = self._pack_qconv(st, qw, qb, s_w)
                    self.packed[st.i] = QConvPack(w8, bq, scale_of[id(st.src)] * s_w, s_a, act, slope, bits_a)
                if self.q1:
                    # the quantisers count their forwards in eval too (quantized_google.py Quantizer.forward)
                    self.q_steps += [conv.weight_quantizer.step, conv.bias_quantizer.step,
                                     conv.activation_quantizer.step]
                if sc is None:
                    scale_of[id(st.out)] = s_a
                else:
                    self.sc_scales[sc.i] = self._shortcut_scales(sc.module)
                    scale_of[id(sc.own)] = s_a
                    scale_of[id(st.out)] = self.sc_scales[sc.i].scale_sum
            elif st.kind == 'shortcut':
                self.sc_scales[st.i] = self._shortcut_scales(st.module)
                scale_of[id(st.out)] = self.sc_scales[st.i].scale_sum
            elif st.kind == 'concat':
                scale_of[id(st.out)] = _s(st.module.scale)
            else:       # upsample, maxpool: the codes keep their grid
                scale_of[id(st.out)] = scale_of[id(st.src)]
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

    def invalidate(self):
        self.graph = None
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

    def _launch_stem(self, st, x):
        """layer 0: the fp32 conv of the float image on the fake-quantised weights, int8 out"""
        pk, conv = self.packed[st.i], st.conv
        lo, hi = -(1 << (pk.bits - 1)), (1 << (pk.bits - 1)) - 1
        d = ops.make_conv_desc((self.B, self.H, self.W, self.Cin), self.Cin, conv.out_channels, conv.kernel_size[0],
                               conv.stride[0], conv.padding[0], ops._pitch(st.out.view()), pk.act, pk.slope, OUT_I8)
        ws = self.stem_w.get(st.i)
        if ws is None:
            # fused tensor-core stem when the fake-quantised weights (int8 code x 2^-n) are exact in fp16 and the bias in
            # the two fp16 terms it is split into; codes x 2^-n below fp16's subnormal grid (tiny weight scales) would be
            # rounded
            fits = self.stem_fused and _stem_fp16_exact(pk.w, pk.bias)
            ws = self.stem_w[st.i] = ops.pack_stem_weights(pk.w) if fits else False
        if ws is not False:
            call("b2y_stem_conv_fwd_fused_q", C.byref(d), ptr(x), 0, 1.0, ptr(ws), ptr(pk.bias), ptr(st.out.buf), pk.s_a,
                 float(lo), float(hi), stream_ptr())
        else:
            call("b2y_stem_conv_fwd_q", C.byref(d), ptr(x), ptr(pk.w), ptr(pk.bias), ptr(st.out.buf), pk.s_a, float(lo),
                 float(hi), stream_ptr())

    def _launch_conv(self, st):
        """A body conv step: the int8 conv, with its folded shortcut in the epilogue.  When the fused launch is refused
        as unsupported (e.g. a scale that is not a power of two) the conv writes its own output and the shortcut runs as
        a launch of its own, for this layer from then on."""
        pk, conv, sc = self.packed[st.i], st.conv, st.shortcut
        k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
        view = _pairs if st.form == 's1' else _Tensor.view
        w_layout = WLAYOUT_S2_PAIRS if st.form == 's2' else 0
        xv, ov = view(st.src), view(st.out)
        if sc is not None:
            av, s_addend, scales = view(sc.addend), self.scale_of[id(sc.addend)], self.sc_scales[sc.i]
            slo, shi = -(1 << (sc.module.bits - 1)), (1 << (sc.module.bits - 1)) - 1
            if self._fusable.get(st.i, True):
                cd = ops.make_conv_desc(xv.shape, ops._pitch(xv), pk.w8.shape[0], k, s, p, ops._pitch(ov), pk.act,
                                        pk.slope, OUT_I8, 0, w_layout)
                qd = ops.QConvDesc(cd, float(pk.acc_scale), float(pk.s_a), float(-(1 << (pk.bits - 1))),
                                   float((1 << (pk.bits - 1)) - 1), OUT_I8, 1, scales.clamp_addends)
                try:
                    call("b2y_qconv2d_shortcut_fwd", C.byref(qd), ptr(xv), ptr(pk.w8), ptr(pk.bias), ptr(av),
                         ops._pitch(av), s_addend, scales.scale_x, scales.scale_a, scales.scale_sum, float(slo),
                         float(shi), ptr(ov), stream_ptr())
                    return
                except B2YError as e:
                    if 'unsupported' not in str(e).lower():
                        raise
                    self._fusable[st.i] = False
            if sc.own.buf is None:
                sc.own.buf = torch.empty((self.B, sc.own.H, sc.own.W, sc.own.C), dtype=torch.int8, device=self.device)
        yv = ov if sc is None else view(sc.own)
        ops.qconv2d(xv, pk.w8, pk.bias, k, s, p, pk.acc_scale, pk.s_a, act=pk.act, slope=pk.slope, bits=pk.bits, out=yv,
                    out_kind=OUT_F32 if st.head else OUT_I8, w_layout=w_layout)
        if sc is not None:
            self._qshortcut(sc.i, sc.module, yv, pk.s_a, av, s_addend, ov, yv.shape[3])

    def _forward_eager(self, x):
        B = self.B
        sc = self.scale_of
        if self.q_steps:
            torch._foreach_add_(self.q_steps, 1)
        for st in self.steps:
            if st.kind == 'conv':
                if st.src is None:
                    self._launch_stem(st, x)
                else:
                    self._launch_conv(st)
            elif st.kind == 'shortcut':
                self._qshortcut(st.i, st.module, st.x.view(), sc[id(st.x)], st.addend.view(), sc[id(st.addend)],
                                st.out.view(), st.out.C)
            elif st.kind == 'concat':
                lo, hi = -(1 << (st.module.bits - 1)), (1 << (st.module.bits - 1)) - 1
                off = 0
                for t in st.srcs:
                    tv = t.view()
                    ov = st.out.buf[..., off:off + t.C]
                    call("b2y_requant_i8", ptr(tv), ops._pitch(tv), ptr(ov), ops._pitch(ov), B * t.H * t.W, t.C,
                         sc[id(t)], sc[id(st.out)], float(lo), float(hi), stream_ptr())
                    off += t.C
            elif st.kind == 'upsample':
                src, sv, ov = st.src, st.src.view(), st.out.view()
                call("b2y_upsample_nearest_i8", ptr(sv), ops._pitch(sv), ptr(ov), ops._pitch(ov), B, src.H, src.W,
                     src.C, int(st.stride), stream_ptr())
            elif st.kind == 'maxpool':
                src, sv, ov = st.src, st.src.view(), st.out.view()
                call("b2y_maxpool_i8", ptr(sv), ops._pitch(sv), ptr(ov), ops._pitch(ov), B, src.H, src.W, src.C,
                     int(st.k), int(st.s), 1 if st.tiny_pad else 0, stream_ptr())
        no = self.yolo[0][0].no
        io = torch.empty((B, self.total_rows, no), dtype=torch.float32, device=self.device)
        p_out = []
        for (m, raw, row_off, rows), anc in zip(self.yolo, self.anchors_px):
            _, p = ops.yolo_decode(raw.buf, m.na, m.no, anc, m.stride, io=io, row_offset=row_off)
            m.nx, m.ny = raw.W, raw.H
            p_out.append(p)
        return io, tuple(p_out), []
