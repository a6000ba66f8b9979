"""Graph executor for Darknet models on sm_90a.

Replaces the reference's per-module Python loop (models.py:508-561, ~250-520 ATen/cuDNN launches per forward)
by a static plan over NHWC fp16 buffers:

  * conv + folded BN + activation (+ the following Shortcut) = one wgmma implicit-GEMM launch,
  * route/concat is zero-copy: producers write straight into their channel slot of the concat buffer,
  * the stem reads the NCHW fp32 image directly, the head convs emit fp32 for the decode kernel,
  * the launch sequence is captured once into a CUDA graph per input shape and replayed.

Parameters stay in the nn.Module tree (fp32, NCHW) and are folded/packed on the device whenever they change.
Shapes, folded shortcuts and the concat placement come from layout.py, which the training plan shares.  Every fp16
tensor is stored in whole 8-channel groups (layout.phys_width): a channel-pruned width such as 37 runs on the same
kernels as 40, with zero weight rows and bias for the pad outputs and zero weight columns wherever an input channel is
a pad or a gap between concat sources.
"""
import collections
import os

import torch
import torch.nn as nn

from . import ops
from .layout import _block_parts, build_layout, feature_slots, infer_shapes, pair_form, pitch, sources, stem_path
from .lib import WLAYOUT_S2_PAIRS


# ---- launch list vocabulary: field 0 is the step's kind; src / out / res / dst are layout._Tensor -------------------
# conv: src is None for the stem (it reads the image), res is the source of the shortcut folded into the conv, or None;
# form is its pixel-pair form (layout.pair_form: 's1', 's2' or None)
ConvStep = collections.namedtuple('ConvStep', 'kind i src out res conv bn act slope form')
DwStep = collections.namedtuple('DwStep', 'kind i src out conv bn act slope')
SeStep = collections.namedtuple('SeStep', 'kind i src out fc1 fc2 ws')
# out = first + others[0] + ...; widths may differ (layers.py:57-72): a sum covers the first min(nx, na) channels, the
# rest of x passes through
AddStep = collections.namedtuple('AddStep', 'kind first others out')
# a concat source that could not be placed inside the concat buffer `dst`: copied to channel offset `off`
CopyStep = collections.namedtuple('CopyStep', 'kind src dst off')
UpsampleStep = collections.namedtuple('UpsampleStep', 'kind src out stride')
# tiny_pad: k = 2, s = 1 (yolov3-tiny), padded on the right / bottom only
MaxpoolStep = collections.namedtuple('MaxpoolStep', 'kind src out k s tiny_pad')


def pointwise_steps(lay, i, d, m, alloc):
    """The steps of layer i when it is a shortcut, route, up-sample or max-pool (the same in inference and training);
    `alloc(tensor, i)` binds the plan's buffer of a tensor that has none yet and returns the tensor."""
    t, tens = d['type'], lay.tens
    if t == 'shortcut':
        if lay.fused_into[i] is not None:
            return []
        if getattr(m, 'weight', False):
            raise NotImplementedError("weighted shortcut is not supported by the sm_90a engine yet")
        return [AddStep('add', tens[i - 1], [tens[s] for s in sources(i, d['from'])], alloc(tens[i], i))]
    if t == 'route':
        if i in lay.grouped:
            tens[i].buf = lay.grouped[i].buf
        return [CopyStep('copy', st, tens[i], off) for st, off, placed in lay.concats.get(i, ()) if not placed]
    if t == 'upsample':
        return [UpsampleStep('upsample', tens[i - 1], alloc(tens[i], i), d['stride'])]
    if t == 'maxpool':
        k, s = d['size'], d['stride']
        return [MaxpoolStep('maxpool', tens[i - 1], alloc(tens[i], i), k, s, k == 2 and s == 1)]
    return []


def launch_pointwise(st):
    """Forward launches of an add / copy / upsample / maxpool step."""
    if st.kind == 'add':
        cur, ov = st.first, st.out.view()
        for a in st.others:
            xv, av = cur.view(), a.view()
            n = min(xv.shape[3], av.shape[3])
            ops.add(xv[..., :n], av[..., :n], out=ov[..., :n])
            if xv.shape[3] > n and cur is not st.out:
                ops.copy_channels(xv[..., n:], ov[..., n:])
            cur = st.out
    elif st.kind == 'copy':
        ops.copy_channels(st.src.view(), st.dst.buf[..., st.off:st.off + st.src.Cp])
    elif st.kind == 'upsample':
        ops.upsample(st.src.view(), st.stride, out=st.out.view())
    elif st.kind == 'maxpool':
        ops.maxpool(st.src.view(), st.k, st.s, tiny_pad=st.tiny_pad, out=st.out.view())


def _whole(t):
    """t is an fp16 tensor that fills its buffer, which the pixel-pair views reshape"""
    return t.c0 == 0 and t.buf.shape[3] == t.C == t.Cp and t.dtype == torch.float16


def _pad_rows(t, n, fill=0.0):
    """t with n - len(t) entries of `fill` appended along dim 0 (the pad output channels of a weight)."""
    if t is None or t.shape[0] == n:
        return t
    return torch.cat([t, t.new_full((n - t.shape[0],) + tuple(t.shape[1:]), fill)])


def _scatter(t, dim, cmap, n):
    """t with entry j along `dim` moved to position cmap[j] of a zero tensor of length n there (layout.Layout.chmap)."""
    if t is None:
        return None
    shape = list(t.shape)
    shape[dim] = n
    return t.new_zeros(shape).index_copy_(dim, torch.as_tensor(cmap, device=t.device), t).contiguous()


def fold_bn(conv, bn):
    """Eval-mode BatchNorm (+ conv bias) as a per-channel (scale, bias) in fp32: y = conv * scale + bias with
    scale = gamma / sqrt(var + eps), bias = beta - mean * scale (+ conv.bias * scale).  Without a BatchNorm the scale is
    None and the bias is the conv's (None when it has none)."""
    if bn is None:
        return None, conv.bias.detach().float() if conv.bias is not None else None
    sc = (bn.weight.detach() / torch.sqrt(bn.running_var + bn.eps)).float()
    bi = (bn.bias.detach() - bn.running_mean * sc).float()
    if conv.bias is not None:
        bi = bi + conv.bias.detach().float() * sc
    return sc, bi


class LazyFeatures(list):
    """feature_out of the reference API (models.py:542-543): one entry per conv block that does not feed a YOLO layer.
    Entries are materialised (NHWC fp16 -> NCHW fp32) on access; they alias engine buffers and are only valid
    until the next forward.  An entry is the NHWC view of the logical channels, or (physical view, logical channel
    index) for a tensor whose channels a concat placed with gaps."""

    def __init__(self, views):
        super().__init__([None] * len(views))
        self._views = views

    def __getitem__(self, i):
        if isinstance(i, slice):
            return [self[j] for j in range(*i.indices(len(self)))]
        v = self._views[i]
        if v is None:
            raise RuntimeError("feature_out[%d] was not kept: set model.keep_features = True before the forward" % i)
        if isinstance(v, tuple):
            return ops.nhwc_to_nchw(v[0]).index_select(1, v[1])
        return ops.nhwc_to_nchw(v)

    def __iter__(self):
        return (self[i] for i in range(len(self)))


class SlotStore:
    """Device storage that the plans of one model share across input shapes.

    A slot is named by what a buffer is (layer index, role, channel pitch, dtype), never by its shape; its capacity is
    the largest request made so far.  A plan's tensor is a prefix of its slot: with the pitch fixed by the channel count,
    pixel n of a smaller plan sits on pixel n of a larger one, so pad channels land on pad channels and stay zero (slots
    are zero-filled when allocated and nobody writes pad channels).  Slot bases come straight from the caching allocator
    (512-byte aligned).  A request above a slot's capacity reallocates that slot and bumps its version: every plan that
    took the old slot still points at the old memory (tensor views, tensor maps, CUDA graphs) and is dropped by the
    engine, which frees the old slot.

    A training forward that waits for its backward pins the store (`pin`, a weak reference to the pin that the step's
    autograd node owns); the engine then builds plans of other shapes on private storage until the backward has run or
    the graph has been freed."""

    def __init__(self, device):
        self.device = device
        self.slots = {}
        self.versions = {}
        self.generation = 0     # bumped by every reallocation
        self.pin = None

    def take(self, name, shape, dtype):
        nbytes = 1
        for s in shape:
            nbytes *= int(s)
        nbytes *= torch.empty((), dtype=dtype).element_size()
        slot = self.slots.get(name)
        if slot is None or slot.numel() < nbytes:
            if slot is not None:
                self.generation += 1
                del self.slots[name], slot          # plans built on the old slot hold it until they are dropped
            slot = self.slots[name] = torch.zeros(max(nbytes, 1), dtype=torch.uint8, device=self.device)
            self.versions[name] = self.versions.get(name, -1) + 1
        return slot[:nbytes].view(dtype).view(shape)

    def pinned_by(self):
        """The plan whose pending backward holds the store, or None."""
        pin = self.pin() if self.pin is not None else None
        return pin.plan if pin is not None else None

    def stale(self, held):
        """held: {slot name: version} of one plan.  True when one of those slots has been reallocated since."""
        return any(self.versions[n] != v for n, v in held.items())


class EvalWeights:
    """Packed inference weights of one model, shared by its eval plans of every shape and re-packed once per parameter
    version.  Entries are keyed (layer index, form): the pixel-pair forms depend on the plan (an odd width rules them
    out), the dense one (form None) does not."""

    def __init__(self):
        self.version = None
        self.packs = {}


class Plan:
    def __init__(self, model, x_shape, device, keep_features=False, store=None, shared_weights=None):
        self.model = model
        self.keep_features = bool(keep_features)
        self.device = device
        self.B, self.Cin, self.H, self.W = x_shape
        self.store = store if store is not None else SlotStore(device)
        self.shared_weights = shared_weights if shared_weights is not None else EvalWeights()
        self.held = {}          # slot name -> version taken
        self.steps = []
        self.wkey = {}          # layer index -> key (layer index, form or kind) of its pack in shared_weights.packs
        self.param_version = None
        self.graph = None
        self.runs = 0
        self.static_x = None
        self._build()

    def _take(self, name, shape, dtype=torch.float16):
        t = self.store.take(name, shape, dtype)
        self.held[name] = self.store.versions[name]
        return t

    def _new_act(self, name, C, H, W):
        """fp16 NHWC activation buffer; widths that are not a multiple of 16 get a zero pad (see _Tensor.view_k)."""
        pc = pitch(C, torch.float16)
        return self._take(('act', name, pc, torch.float16), (self.B, H, W, pc))

    def _w(self, i):
        return self.shared_weights.packs[self.wkey[i]]

    # ---------------------------------------------------------------------------------------------------------
    def _build(self):
        model, B = self.model, self.B
        defs, mods = model.module_defs, model.module_list
        n = len(defs)
        shapes = infer_shapes(model, (self.Cin, self.H, self.W))
        # inference folds a shortcut into the residual epilogue of the conv before it; the epilogue reads whole
        # 8-channel groups, which every physical width is
        lay = build_layout(model, shapes, self.keep_features, lambda i: True)
        tens, fused_into = lay.tens, lay.fused_into
        self.chmap = lay.chmap

        # multi-source routes are buffers their producers write into; a conv reads a placed source through view_k, up to
        # its next 16-channel boundary, which may lie past the concat's own width
        for i, parts in lay.concats.items():
            dst = tens[i]
            width = max([dst.Cp] + [off + (st.Cp + 15) // 16 * 16 for st, off, placed in parts if placed])
            dst.buf = self._new_act(('cat', i), width, dst.H, dst.W)
            for st, off, placed in parts:
                if placed:
                    st.buf = dst.buf

        # allocate what is left and emit the launch list
        def alloc(t, i):
            if t.buf is None:
                if t.dtype == torch.float16:
                    t.buf = self._new_act(i, t.Cp, t.H, t.W)
                else:
                    pc = pitch(t.Cp, t.dtype)
                    t.buf = self._take(('head', i, pc, t.dtype), (B, t.H, t.W, pc), t.dtype)
            return t

        self.yolo = []
        row_off = 0
        for i, (d, m) in enumerate(zip(defs, mods)):
            t = d['type']
            if t == 'depthwise':
                conv, bn, act, slope = _block_parts(m)
                if conv.groups != conv.in_channels or conv.out_channels != conv.in_channels:
                    raise NotImplementedError("only channel-multiplier-1 depthwise convolutions are supported")
                self.steps.append(DwStep('dw', i, tens[i - 1], alloc(tens[i], i), conv, bn, act, slope))
            elif t == 'se':
                fc = m[0].fc if isinstance(m, nn.Sequential) else m.fc
                src = tens[i - 1]
                ws = self._take(('se_ws', i), (B, 3 * src.Cp + fc[0].out_features), torch.float32)
                self.steps.append(SeStep('se', i, src, alloc(tens[i], i), fc[0], fc[2], ws))
            elif t == 'convolutional':
                conv, bn, act, slope = _block_parts(m)
                if conv.groups != 1:
                    raise NotImplementedError("grouped convolution is not supported by the sm_90a engine yet")
                out = alloc(tens[i], i)
                res = None
                if i + 1 < n and fused_into[i + 1] == i:
                    res = tens[sources(i + 1, defs[i + 1]['from'])[0]]
                src = None if i == 0 else tens[i - 1]
                k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
                form = None
                if src is None:
                    self.stem = stem_path(conv.in_channels, k, out.Cp)
                    if self.stem == 'im2col':
                        d = ops.make_conv_desc((B, self.H, self.W, conv.in_channels), conv.in_channels, out.Cp, k, s,
                                               p, out.Cp)
                        self.stem_ws = self._take(('stem_ws',), (ops.stem_workspace_bytes(d) // 2,))
                else:
                    form = pair_form(k, s, p, conv.in_channels, conv.out_channels, src.W)
                    if form == 's1' and not all(_whole(t) for t in (src, out, res) if t is not None):
                        form = None
                    elif form == 's2' and not (_whole(src) and out.C == out.Cp):
                        form = None
                self.steps.append(ConvStep('conv', i, src, out, res, conv, bn, act, slope, form))
            elif t == 'yolo':
                raw = tens[i - 1]
                rows = m.na * raw.H * raw.W
                self.yolo.append((m, raw, row_off, rows))
                row_off += rows
            else:
                self.steps += pointwise_steps(lay, i, d, m, alloc)
        self.total_rows = row_off
        self.feature_views = [self._logical(tens[i], lay.chmap[i]) if self.keep_features else None
                              for i in feature_slots(model)]
        self.anchors_px = [m.anchors.to(self.device).float().contiguous() for (m, _, _, _) in self.yolo]

    def _logical(self, t, cmap):
        """(tensor, None) when its logical channels are the first C physical ones (the map is strictly increasing, so
        it is the identity when it ends at C - 1), else (tensor, device index of its logical channels)."""
        if cmap[-1] == t.C - 1:
            return t, None
        return t, torch.as_tensor(cmap, device=self.device)

    # ---------------------------------------------------------------------------------------------------------
    def _params_version(self):
        # tensor versions catch optimiser steps and copy_(); the data pointers catch re-assigned `.data` (nn.Module.to /
        # half, FlatDataParallel); the model-level epoch is bumped by the training plan, whose kernels update the
        # BatchNorm running statistics through raw pointers (no version bump, invisible under CUDA-graph replay).
        # Edits through `.data` that keep the storage (w.data.mul_()) are invisible: call model.engine().invalidate().
        v = getattr(self.model, '_b2y_epoch', 0)
        for t in list(self.model.parameters()) + list(self.model.buffers()):
            v += t._version + (t.data_ptr() & 0xffff)
        return v

    def _pack_weights(self, ver):
        """Look up (and pack on first use at this parameter version) the weights of every layer in the engine-wide
        EvalWeights; the plan keeps only the keys, so it never holds packed weights of an outdated version."""
        sw = self.shared_weights
        if sw.version != ver:
            sw.packs = {}
            sw.version = ver
        packs = sw.packs
        for st in self.steps:
            if st.kind in ('dw', 'se'):
                # channel by channel over the input's physical channels: zero weights, scale and bias (squeeze-excite:
                # zero fc1 columns and fc2 rows) for its pad and gap channels
                key = self.wkey[st.i] = (st.i, st.kind)
                if key not in packs:
                    cmap, cp = self.chmap[st.i - 1], st.src.Cp
                    if st.kind == 'dw':
                        sc, bi = fold_bn(st.conv, st.bn)
                        packs[key] = (_scatter(st.conv.weight.detach().float(), 0, cmap, cp),
                                      _scatter(sc, 0, cmap, cp), _scatter(bi, 0, cmap, cp))
                    else:
                        packs[key] = (_scatter(st.fc1.weight.detach(), 1, cmap, cp),
                                      _scatter(st.fc2.weight.detach(), 0, cmap, cp))
                continue
            if st.kind != 'conv':
                continue
            i, conv, bn = st.i, st.conv, st.bn
            key = self.wkey[i] = (i, st.form)
            if key in packs:
                continue
            bnp = None
            eps = 1e-5
            if bn is not None:
                bnp = (bn.weight.detach(), bn.bias.detach(), bn.running_mean, bn.running_var)
                eps = bn.eps
            base = packs.get((i, None))
            if base is None:
                stem = st.src is None
                # [Cp_out][K][kh][kw]: zero rows, bias and BatchNorm scale for the pad outputs (BatchNorm padded with
                # gamma = beta = mean = 0, var = 1); the input columns go through the source's channel map, with zero
                # columns for its pad and gap channels and up to the MMA K granule (view_k)
                cp = st.out.Cp
                wsrc = _pad_rows(conv.weight.detach(), cp)
                if not stem:
                    wsrc = _scatter(wsrc, 1, self.chmap[i - 1], (st.src.Cp + 15) // 16 * 16)
                bnp_p = None if bnp is None else tuple(_pad_rows(t, cp, f) for t, f in zip(bnp, (0.0, 0.0, 0.0, 1.0)))
                wp, bias, w32 = ops.pack_conv_weights(wsrc, _pad_rows(conv.bias.detach(), cp) if conv.bias is not None
                                                      else None, bnp_p, eps, want_fp32=stem)
                wstem = ops.pack_stem_weights(w32) if stem and self.stem != 'direct' else None
                base = packs[(i, None)] = (wp, bias, w32, wstem)
            if st.form == 's1':
                packs[key] = base + (self._pair_pack(conv, bnp, eps),)
            elif st.form == 's2':
                _, bias_f, w32f = ops.pack_conv_weights(conv.weight.detach(), conv.bias.detach() if conv.bias is not None
                                                        else None, bnp, eps, want_fp32=True)
                packs[key] = base + ((ops.s2_pair_weights(w32f).half(), bias_f),)

    # ---- pixel-pair packing of the Cin = 32 3x3 layers (layout.pair_form) ------------------------------------------
    # With 32 input channels a tap of the im2col gather is a 64-byte row: one TMA request per pixel per tap, and the
    # layer is bound by the TMA request rate (0.16 of the tensor peak, 31-46 % of HBM in round 1), not by HBM.  The NHWC
    # tensor [B,H,W,32] is the same memory as [B,H,W/2,64]: viewed as pixel PAIRS the same convolution is a 3x3 conv
    # with 64 input and 2*Cout output channels whose weights are the original taps placed at
    # s = 2(kwp-1) + i_sub - o_sub + 1 (zero elsewhere).  Half of the MACs multiply zeros, but the rows are 128 bytes,
    # the tile count halves and N = 128 brings the CTA-pair path in -- no new kernel, only a weight layout.  Stride 2
    # reads the input as pixel pairs through B2Y_WLAYOUT_S2_PAIRS: a 3 x 2 window with stride 2 x 1 over 128-byte rows
    # (6 im2col boxes, not 9 halves).
    def _pair_pack(self, conv, bnp, eps):
        _, bias, w32 = ops.pack_conv_weights(conv.weight.detach(), conv.bias.detach() if conv.bias is not None else None,
                                             bnp, eps, want_fp32=True)
        wp2, _, _ = ops.pack_conv_weights(ops.s1_pair_weights(w32))
        return wp2, torch.cat([bias, bias]).contiguous()

    def _launch_conv(self, st, x):
        src, out, res, conv, act, slope = st.src, st.out, st.res, st.conv, st.act, st.slope
        wp, bias, w32, wstem = self._w(st.i)[:4]
        k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
        if src is None:
            if self.stem == 'fused':
                # the fused kernel builds the im2col tile in smem (no workspace)
                ops.stem_conv_fused(x, wstem, bias, k, s, p, act=act, slope=slope, out=out.view(),
                                    x_div=256.0 if x.dtype == torch.uint8 else 1.0)
                return
            if x.dtype != torch.float32:
                x = x.float() / 256.0 if x.dtype == torch.uint8 else x.float()
            if self.stem == 'im2col':
                ops.stem_conv_tc(x, wstem, bias, conv.in_channels, k, s, p, act=act, slope=slope,
                                 out=out.view(), workspace=self.stem_ws)
            else:
                ops.stem_conv(x, w32, bias, k, s, p, act=act, slope=slope, out=out.view())
        elif st.form == 's2':
            wps2, bias_s2 = self._w(st.i)[4]
            ops.conv2d(src.view(), wps2, bias_s2, k, s, p, act=act, slope=slope,
                       residual=res.view() if res is not None else None, out=out.view(), w_layout=WLAYOUT_S2_PAIRS)
        elif st.form == 's1':
            wp2, bias2 = self._w(st.i)[4]
            pairs = lambda t: t.buf.view(t.buf.shape[0], t.H, t.W // 2, 2 * t.C)
            ops.conv2d(pairs(src), wp2, bias2, 3, 1, 1, act=act, slope=slope,
                       residual=pairs(res) if res is not None else None, out=pairs(out))
        else:
            ops.conv2d(src.view_k(), wp, bias, k, s, p, act=act, slope=slope,
                       residual=res.view() if res is not None else None, out=out.view())

    def _launch_all(self, x):
        for st in self.steps:
            if st.kind == 'conv':
                self._launch_conv(st, x)
            elif st.kind == 'dw':
                conv = st.conv
                w, sc, bi = self._w(st.i)
                ops.dwconv2d(st.src.view(), w, conv.kernel_size[0], conv.stride[0], conv.padding[0], scale=sc, bias=bi,
                             act=st.act, slope=st.slope, out=st.out.view())
            elif st.kind == 'se':
                w1, w2 = self._w(st.i)
                ops.se_fwd(st.src.view(), w1, w2, out=st.out.view(), ws=st.ws)
            else:
                launch_pointwise(st)
        for (m, raw, row_off, rows), anc in zip(self.yolo, self.anchors_px):
            _, p = ops.yolo_decode(raw.buf, m.na, m.no, anc, m.stride, io=self.io, row_offset=row_off)
            self.p_out.append(p)

    def forward(self, x):
        model = self.model
        ver = self._params_version()
        if ver != self.param_version:
            self._pack_weights(ver)
            self.param_version = ver
            self.graph = None
        # fp32 / fp16 images go to the stem as they are; uint8 images (the reference's dataloader output before
        # test.py:95 / train.py:348 "imgs.float() / 256.0") are normalised inside the stem kernel
        x = x.contiguous()
        if x.dtype not in (torch.float32, torch.float16, torch.uint8):
            x = x.float()
        no = self.yolo[0][0].no
        use_graph = getattr(model, 'use_cuda_graph', os.environ.get('B2Y_NO_GRAPH', '0') != '1')
        if not use_graph or self.runs < 1:
            self.io = torch.empty((self.B, self.total_rows, no), dtype=torch.float32, device=self.device)
            self.p_out = []
            self._launch_all(x)
            self.runs += 1
            io, p = self.io, tuple(self.p_out)
        else:
            if self.graph is None:
                self.static_x = self._take(('x', x.dtype), tuple(x.shape), x.dtype)
                self.static_x.copy_(x)
                self.io = torch.empty((self.B, self.total_rows, no), dtype=torch.float32, device=self.device)
                g = torch.cuda.CUDAGraph()
                torch.cuda.synchronize()
                with torch.cuda.graph(g):
                    self.p_out = []
                    self._launch_all(self.static_x)
                self.graph = g
                self.static_p = tuple(self.p_out)
            if x.data_ptr() != self.static_x.data_ptr():
                self.static_x.copy_(x)
            self.graph.replay()
            if getattr(model, 'static_outputs', False):
                io, p = self.io, self.static_p
            else:
                io, p = self.io.clone(), tuple(t.clone() for t in self.static_p)
        for (m, raw, _, _) in self.yolo:
            m.nx, m.ny = raw.W, raw.H
        feats = LazyFeatures([None if f is None else f[0].buf[..., f[0].c0:f[0].c0 + f[0].C] if f[1] is None
                              else (f[0].view(), f[1]) for f in self.feature_views])
        return io, p, feats


class Engine:
    def __init__(self, model):
        self.model = model
        self.plans = {}
        self._reset_shared()

    def _reset_shared(self):
        # shape-dependent buffers: one slot store for the training plans, one for the eval plans (created on the
        # model's device at first use); shape-independent state: packed weights, gradient outputs, side stream
        self.train_store = self.eval_store = None
        self.eval_weights = EvalWeights()
        self.train_shared = None

    def invalidate(self):
        self.plans.clear()
        self._reset_shared()

    def weights_changed(self):
        """The parameters were written in place without a version bump (fused optimiser on the flat buffers): every
        plan re-packs its weights on its next forward."""
        self.eval_weights.version = None
        for plan in self.plans.values():
            plan.param_version = None

    def _drop_stale(self):
        """Drop the plans whose slots were reallocated by a larger request (their graphs point at the old memory)."""
        for store in (self.train_store, self.eval_store):
            if store is None:
                continue
            for k in [k for k, p in self.plans.items() if getattr(p, 'store', None) is store and store.stale(p.held)]:
                del self.plans[k]

    def _forward_quantized(self, x):
        model = self.model
        if model.quantized in (1, 2):
            # QAT graphs (google / TPSQ): the module forwards themselves, over NHWC fp32 tensors (b200yolo/qat.py)
            from .qat import QatRunner
            if model.training:
                return QatRunner(model).forward(x)
            if model.quantized == 1:
                # eval of a google-QAT model whose structure qengine.int8_graph_refusal accepts: the integer network,
                # bit-identical to the module forwards; the plan re-packs itself when training has moved the QAT state
                key = (tuple(x.shape), 'q1', x.device.index)
                plan = self.plans.get(key)
                if plan is None:
                    from .qengine import QPlan, int8_graph_refusal
                    if int8_graph_refusal(model) is None:
                        plan = self.plans[key] = QPlan(model, tuple(x.shape), x.device)
                if plan is not None:
                    return plan.forward(x)
            with torch.no_grad():
                return QatRunner(model).forward(x)
        if model.quantized != 3:
            raise NotImplementedError("quantized=%d is not a mode of the reference" % model.quantized)
        if model.training:
            # calibration forward (PTQ.py:76-88): votes / bias correction mutate the quantiser state, so every cached
            # INT8 eval plan (packed int8 weights, scales baked into its CUDA graph) is stale afterwards
            from .qcalib import QCalibPlan
            for k in [k for k in self.plans if len(k) == 3 and k[1] == 'q3']:
                del self.plans[k]
            with torch.no_grad():
                return QCalibPlan(model, tuple(x.shape), x.device).forward(x)
        key = (tuple(x.shape), 'q3', x.device.index)
        plan = self.plans.get(key)
        if plan is None:
            from .qengine import QPlan
            plan = QPlan(model, tuple(x.shape), x.device)
            self.plans[key] = plan
        return plan.forward(x)

    def plan_for(self, x):
        self.forward(x)
        return self.last_plan

    def _check_device(self, x):
        """One engine serves ONE device: the packed weights, plans and CUDA graphs live where the parameters are.
        nn.DataParallel replicas (test.py:55-56 wraps the model when several GPUs are visible) share this object and
        would read device-0 weight pointers from other devices -- refuse instead of computing garbage.  Multi-GPU =
        one process per GPU (b200yolo.parallel.FlatDataParallel / torchrun); for test.py use --device 0."""
        p = next(self.model.parameters(), None)
        if p is not None and p.device != x.device:
            raise RuntimeError(
                "b200yolo: input on %s but the model's parameters are on %s. Single-process multi-GPU "
                "(nn.DataParallel) is not supported by the sm_90a engine: run one process per GPU "
                "(CUDA_VISIBLE_DEVICES / --device 0, or torchrun + FlatDataParallel)." % (x.device, p.device))

    def forward(self, x):
        self._check_device(x)
        with torch.cuda.device(x.device):       # kernels go to the current stream OF THE INPUT'S DEVICE
            return self._forward(x)

    def _forward(self, x):
        model = self.model
        if model.quantized != -1:
            return self._forward_quantized(x)
        if getattr(model, 'accurate', False) and not model.training:
            # fp32-accurate verification mode (split-fp16 tensor-core convs, fp32 activations): accurate.py
            if getattr(self, '_accurate', None) is None:
                from .accurate import AccurateRunner
                self._accurate = AccurateRunner(model)
            return self._accurate.forward(x)
        keep = bool(model.keep_features)
        # a train-mode forward that records no graph (torch.no_grad(), or frozen parameters) only needs the batch
        # statistics and the running-statistics update: the forward-only plan, which runs channel-pruned widths too
        # (adaptive BatchNorm recalibration of pruned candidates, EagleEye_*_prune.py)
        fwd_only = model.training and not (torch.is_grad_enabled() and any(p.requires_grad for p in model.parameters()))
        key = (tuple(x.shape), bool(model.training), x.device.index, keep, x.dtype) + (('stats',) if fwd_only else ())
        if model.training:
            from .train_engine import TrainPlan, TrainShared
            if self.train_store is None:
                self.train_store, self.train_shared = SlotStore(x.device), TrainShared(x.device)
            store = self.train_store
        else:
            if self.eval_store is None:
                self.eval_store = SlotStore(x.device)
            store = self.eval_store
        plan = self.plans.get(key)
        owner = None if fwd_only else store.pinned_by()      # the forward-only plan's slots are its own
        if owner is not None and owner is not plan:
            # a training forward of another shape still waits for its backward and owns the shared slots: this step
            # runs on a plan with private storage, which is not cached
            plan = TrainPlan(model, tuple(x.shape), x.device, keep, SlotStore(x.device), self.train_shared)
        elif plan is None:
            # bounded plan cache: a cached plan holds its tensor maps, CUDA graphs and caller-visible outputs, while the
            # activation / gradient buffers are slots shared by every shape; least recently used plans are dropped
            # beyond B2Y_MAX_PLANS (default 32: 11 multi-scale training sizes plus a rectangular evaluation set)
            limit = int(os.environ.get('B2Y_MAX_PLANS', '32'))
            while len(self.plans) >= limit > 0:
                self.plans.pop(next(iter(self.plans)))
            gen = store.generation
            if model.training:
                plan = TrainPlan(model, tuple(x.shape), x.device, keep, store, self.train_shared, forward_only=fwd_only)
            else:
                plan = Plan(model, tuple(x.shape), x.device, keep, store, self.eval_weights)
            self.plans[key] = plan
            if store.generation != gen:
                self._drop_stale()
        else:
            self.plans[key] = self.plans.pop(key)      # move to the most-recently-used end
        self.last_plan = plan
        gen = store.generation
        out = plan.run(x) if model.training else plan.forward(x)
        if store.generation != gen:                 # a slot taken on first use grew
            self._drop_stale()
        return out
